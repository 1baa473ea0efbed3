#!/usr/bin/env python3
"""Golden case O: the uint8 images free_viewpoint_rendering.py saves for rendered frames (:615-766), on seeded inputs
(tests/frame_images_reference.seeded_inputs: 3 frames of 24 x 32), with the imports and shims of make_golden.py:
    python tests/golden/make_golden_frame_images.py
Writes tests/golden/caseO_frame_images.npz: the inputs, and every image.

to8b, visualize_disparity_with_jet_color_scheme and visualize_disparity_with_blinn_phong are EXECUTED from the
unmodified reference (run_nerf_helpers.py).  matplotlib is replaced by a stub whose cm.jet(i) returns
tests/eval_reference.jet_lut()[i], the table tests/test_evaluation_cpu.py checks against matplotlib's segment data.
The correspondence arithmetic (:640-644) and the convert_* helpers (:346-378) live inside free_viewpoint_rendering()
and cannot be called on their own: for the images they make (disp, disp_video, correspondences, rigidity) the fixture
stores to8b of tests/frame_images_reference.py's values, so it pins that restatement rather than checking it.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden as G  # noqa: E402
from tests import eval_reference as E  # noqa: E402
from tests import frame_images_reference as R  # noqa: E402

SEED, F, H, W = 1500, 3, 24, 32


def main():
    rt, rh = G.import_reference()
    lut = E.jet_lut()
    cm = types.ModuleType("matplotlib.cm")
    cm.jet = lambda i: tuple(lut[int(i)]) + (1.0,)
    sys.modules["matplotlib.cm"] = cm
    sys.modules["matplotlib"].cm = cm

    rgbs, disps, pts, rig, lo, hi = R.seeded_inputs(F, H, W, SEED)
    with np.errstate(invalid="ignore"):
        out = {
            "rgb": rh.to8b(rgbs),
            "disp": np.stack([rh.to8b(R.normalized(d)) for d in disps]),
            "disp_video": rh.to8b(R.normalized(disps)),
            "disp_jet": np.stack([rh.to8b(rh.visualize_disparity_with_jet_color_scheme(R.normalized(d))) for d in disps]),
            "disp_phong": np.stack([rh.to8b(rh.visualize_disparity_with_blinn_phong(R.normalized(d))) for d in disps]),
            "correspondences": rh.to8b(R.correspondence_rgb(pts.reshape(F, H, W, 3), lo, hi)),
            "rigidity": rh.to8b(rig.reshape(F, H, W).copy()),
            "rigidity_jet": np.stack([rh.to8b(rh.visualize_disparity_with_jet_color_scheme(r.copy())) for r in rig.reshape(F, H, W)]),
        }
    ref = R.frame_images(rgbs, disps, pts, rig, lo, hi)
    for k, v in out.items():
        d = np.abs(v.astype(np.int16) - ref[k].astype(np.int16))
        print(f"{k:16s} {str(v.shape):16s} restatement: {int((d != 0).sum())} values differ, at most by {int(d.max())}")
    np.savez_compressed(os.path.join(HERE, "caseO_frame_images.npz"), seed=SEED, rgbs=rgbs, disps=disps, surface_pts=pts,
                        surface_rigidity=rig, min_point=lo, max_point=hi, **out)


if __name__ == "__main__":
    main()
