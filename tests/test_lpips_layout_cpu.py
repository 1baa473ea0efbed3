"""The LPIPS workspace layout that tests/lpips_layout.py mirrors, pinned to the library's workspace sizes and to the
constants of csrc/lpips.cuh and lpips.cu.  No kernel is launched here."""
import os
import re

import pytest

from tests import lpips_layout as L
from tests import lpips_stages as S


def _src(name):
    from nonrigid_nerf_b200 import _lib
    return open(os.path.join(os.path.dirname(_lib.__file__), "csrc", name)).read()


def _ints(text):
    return [int(t) for t in re.findall(r"-?\d+", text)]


def test_mirror_constants_are_the_headers():
    h = _src("lpips.cuh")
    arr = lambda name: _ints(re.search(name + r"\[[^\]]*\]\s*=\s*\{(.*?)\};", h, re.S).group(1))
    const = lambda name: re.search(r"constexpr\s+\w+\s+" + name + r"\s*=\s*([^;]*);", h).group(1)
    assert tuple(arr("kLpipsStageChannels")) == L.STAGE_CHANNELS
    assert tuple(arr("kLpipsTapStage")) == L.TAP_STAGES
    convs = arr("kLpipsConv")
    assert tuple(tuple(convs[i:i + 7]) for i in range(0, 35, 7)) == L.CONVS and len(convs) == 35
    assert int(const("kLpipsTaps")) == L.TAPS and int(const("kLpipsStages")) == L.STAGES
    assert int(const("kLpipsDistPixels")) == L.DIST_PIXELS and int(const("kLpipsSlabChunks")) == L.SLAB_CHUNKS
    assert int(const("kLpipsMaxChunk")) == L.MAX_CHUNK
    assert int(const("kLpipsMinSide")) == L.MIN_SIDE and int(const("kLpipsMaxSide")) == L.MAX_SIDE
    assert const("kLpipsChunkBudget").replace(" ", "") == "256ull<<20" and L.CHUNK_BUDGET == 256 << 20
    assert float(const("kLpipsHalfMax").rstrip("f")) == S.F16_MAX == 65504.0
    # the stage each convolution reads (launch_conv_layer's kInStage)
    assert tuple(_ints(re.search(r"kInStage\[kLpipsTaps\]\s*=\s*\{(.*?)\}", _src("lpips.cu")).group(1))) == L.IN_STAGE


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_mirror_sizes_are_the_librarys(shape):
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    h, w = S.SHAPES[shape]
    for hh, ww in ((h, w), (w, h)):
        base = lib.nrn_lpips_workspace_bytes(0, hh, ww)
        assert base == L.mask_bytes(hh, ww) == L.workspace_bytes(0, hh, ww)
        assert lib.nrn_lpips_workspace_bytes(1, hh, ww) - base == L.frame_bytes(hh, ww)
        for fc in (1, 2, 37):
            assert lib.nrn_lpips_workspace_bytes(fc, hh, ww) == L.workspace_bytes(fc, hh, ww), (hh, ww, fc)
            c = L.chunk(fc, hh, ww)
            # every stage 256-byte aligned and in order, the partials and words after them, all inside the chunk's share
            assert all(o % 256 == 0 for o in c["act"]) and c["act"] == sorted(c["act"])
            assert c["partials"] % 256 == 0 and c["sat"] % 8 == 0
            assert c["end"] <= L.mask_bytes(hh, ww) + fc * L.frame_bytes(hh, ww), (hh, ww, fc)


def test_stage_geometry():
    assert L.dims(31, 31)[5:] == [(1, 1)] * 3
    assert L.px(35, 35, 1) == 64 and L.px(35, 67, 1) == 128 and L.px(47, 143, 1) == 385
    assert L.px(63, 71, 1) == 255 and L.px(63, 191, 1) == 705
    assert L.px(71, 135, 2) == L.px(71, 135, 3) == 128 and L.px(127, 143, 3) == 255
    assert L.dims(31, 1000)[7][0] == 1 and L.dims(1000, 31)[7][1] == 1
    # the chunk of 180 frames at 1008 x 756 that tests/test_lpips_stages_gpu.py reads: its input stage passes 2^32
    # bytes and its conv1 stage 2^31
    c = L.chunk(180, 756, 1008)
    assert c["act"][1] - c["act"][0] > 2 ** 32 and c["act"][2] - c["act"][1] > 2 ** 31
    assert 359 * L.image_bytes(756, 1008, 0) > 2 ** 32 and 359 * L.image_bytes(756, 1008, 1) > 2 ** 31
