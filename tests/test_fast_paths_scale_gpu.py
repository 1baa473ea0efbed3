"""The inference-only render passes (occupancy grids, early ray termination, baked radiance grids and baked per-frame
deformation grids) at the render workload's chunk and past 2^31 bytes of their workspaces, bit for bit against their
definitions: raw equals the exact fused pass where a pass evaluates the network, and the numpy restatements of
tests/occupancy_reference.py, tests/termination_reference.py, tests/baked_reference.py and
tests/baked_deformation_reference.py where it looks a value up.  Every output and workspace is filled with 0xFF before
a pass is called through its C entry point, so a slot that nobody writes cannot pass; the autograd entry points must
give the same bits.

  render chunk   65,536 rays, 64 + 64 samples, perturb 0, no noise (4.2 M coarse and 8.4 M fine samples per pass):
                 configurations that change nothing render identically to render(); partial ones are checked per pass
                 on every sample; the fine compositing of sampled rays (first and last, the rays of each launch's first
                 and last persistent sweep, and rays at the stride boundaries of the capped grid-stride kernels) holds
                 the fp64 bounds of tests/ray_reference.py; chunk = 65,536 and chunk = 4,096 render the same frame
  past 2^31      one pass per path, called directly without details: the rays whose samples hold byte 2^31 (and 2^32)
                 of each named buffer, their neighbours, the first and last rays and random rays equal a separate small
                 call on those rays, and that call its definition.  Kept and fallback sets follow from an exact GPU
                 restatement of the rule, because compaction is in order; the workspace's kept indices must equal it.

Each test asserts its premise first (kept and fallback counts against two strides of the capped kernels, which run
16 blocks of 256 threads per SM; buffer sizes against 2^31 / 2^32 from nrn_*_workspace_bytes and c_abi.cu's layout),
and prints it with `pytest -s`, with the worst compositing c_obs and each case's run time and peak memory.

Measured on one H100 80GB HBM3 (700 W power limit, 132 SMs; one stride of the capped kernels is 540,672 items), printed
with `pytest -s`; the file runs in about 5 minutes, most of it the numpy restatements of the deformation tests.
  render chunk   identities 0.3 to 1.4 s each, peak 3.5 GiB allocated; the all-fallback deformation pass gathers and
                 scatters over 8 / 16 strides (coarse / fine) and runs field_bend_rays_kernel over 32,768 / 65,536 tiles.
                 Partial passes 3.5 to 46 s, peak 6.3 GiB: the 30 % grid keeps 1.27 M / 5.0 M samples (3 / 10 scatter
                 strides, 4 / 8 scan chunks), the half box sends 2.1 M / 4.2 M to the trunk (4 / 8 strides), the half
                 deformation box lets 19,492 rays fall back (3 / 5 gather and scatter strides); opaque densities kill
                 every ray without a grid and 90 % with one keeping 80 %.  Worst compositing c_obs 14.6 of c = 400
                 (weights), rgb 4.5, acc 5.0
  past 2^31      1.5 M x 128 with a bender (occupancy and baked, 97 % kept): ws 1.46, raw 1.83, craw 1.78 and kept_xyz
                 1.07 x 2^31 bytes, 353 scatter strides, 188 scan chunks; 17.5 GiB peak, under 1 s each.
                 Termination 6.8 M x 32: ws 1.62, raw 2.03 and one round's craw 1.01 x 2^31, 202 scatter strides;
                 12.8 GiB.  Deformation 8.65 M x 16, 99 % falling back: deform_rays_kernel 2 strides of 2^23 rays, the
                 fallback scan 8,448 block counts (9 chunks), gather 507 and scatter 254 strides, ws 1.03, raw 1.29, bw
                 1.02 and craw 1.16 x 2^31; 16.3 GiB, 1.3 s.  Baked without a bender 2.15 M x 128: baked_rays_kernel 2
                 strides of 2^28 samples, raw 2.56 x 2^31; 21.1 GiB.  Each case is skipped with the GiB it needs when
                 the device has less free.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import baked_deformation_reference as D
from tests import baked_reference as BR
from tests import occupancy_reference as OR
from tests import ray_reference as RR
from tests import stash_layout as SL
from tests import termination_reference as TR
from tests.parity import DEV, Report, poison_bytes, poison_f32
from tests.test_baked_deformation_gpu import DETAILS, _box, _cut_box, _lats
from tests.test_baked_gpu import _bits_equal, _point_raw
from tests.test_ray_kernels_parity_gpu import UNDERFLOW, c_scan
from tests.test_scale_gpu import f32_bits_equal

pytestmark = pytest.mark.gpu
N = 65536            # rays of the render workload's chunk
NS, NI = 64, 64      # coarse and importance samples
CHUNK = 1 << 20      # points per chunk of the numpy restatements
LIMITS = (2 ** 31, 2 ** 32)


@pytest.fixture(autouse=True)
def _time_and_memory(request):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"  [{request.node.name}] {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB "
          f"allocated")


def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L


def _G():
    from nonrigid_nerf_b200 import geometry
    return geometry


def _np(t):
    return t.detach().cpu().numpy()


def _stride():
    """Items per stride of the capped grid-stride kernels (occ_scatter_kernel, deform_gather_kernel,
    deform_scatter_kernel): 16 blocks of 256 threads per SM."""
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 16 * 256


def _ceil(a, b):
    return -(-int(a) // int(b))


def _strides(k):
    return _ceil(k, _stride())


def _scan_chunks(n):
    """Chunks of 1,024 block counts occ_scan_kernel carries its total across, for n items in blocks of 1,024."""
    return _ceil(_ceil(n, 1024), 1024)


def _align(b):
    return (b + 255) // 256 * 256


def _has_bender(net):
    return net.ray_bender[0] is not None


def _models(bender, boost=30.0):
    coarse, fine, b, _ = helpers.build_models(O, 900, DEV, with_bender=bender, density_boost=boost)
    return coarse, fine, b


# ---- one pass through its C entry point, outputs and workspace poisoned -------------------------------------------------
def direct(path, net, rays, z, lat, details=True, grid=None, frame=None, t=None):
    """One pass of `path` (occupancy, terminate, baked, deformed) with raw, the details, termination_index and the
    workspace filled with 0xFF first.  Returns (raw, details, termination_index or None, workspace)."""
    from nonrigid_nerf_b200 import autograd as A, ops
    L = _lib()
    lib = L.load()
    bend = _has_bender(net)
    out_ch = net.output_linear.weight.shape[0]
    bp = ops.pack_bender(net.ray_bender[0]) if bend else None
    a, _, _, keep = ops._field_args(rays, z, None, 1, lat if bend else None, ops.pack_nerf(net), bp, out_ch, A._knobs(net), False, False)
    n, S = a.n_rays, a.n_samples
    raw = poison_f32(n, S, out_ch)
    a.raw = raw.data_ptr()
    det = {}
    if details:
        for k in ("initial_input_pts", "input_pts") + (DETAILS[2:] if bend else ()):
            det[k] = poison_f32(n, S, 1 if k == "rigidity_mask" else 3)
            setattr(a, k, det[k].data_ptr())
    term = None
    if path == "occupancy":
        nbytes = lib.nrn_occupancy_workspace_bytes(n, S, out_ch, int(bend))
        ws, g = poison_bytes(nbytes), grid.c_struct(DEV)
        rc = lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws.data_ptr(), nbytes)
    elif path == "terminate":
        nbytes = lib.nrn_termination_workspace_bytes(n, S, out_ch, int(bend))
        ws, g = poison_bytes(nbytes), grid.c_struct(DEV) if grid is not None else None
        term = torch.full((n,), -1, dtype=torch.int32, device=DEV)
        ta = L.NrnTerminationArgs()
        ta.threshold, ta.termination_index = float(t), term.data_ptr()
        rc = lib.nrn_field_forward_terminate(C.byref(a), C.byref(g) if g is not None else None, C.byref(ta), ws.data_ptr(), nbytes)
    elif path == "baked":
        nbytes = lib.nrn_baked_workspace_bytes(n, S, out_ch, int(bend))
        ws, g = poison_bytes(nbytes), grid.c_struct(DEV)
        rc = lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws.data_ptr(), nbytes)
    else:
        nbytes = lib.nrn_deformed_workspace_bytes(n, S, out_ch, int(details))
        ws, g, d = poison_bytes(nbytes), grid.c_struct(DEV), frame.c_struct(DEV)
        rc = lib.nrn_field_forward_deformed(C.byref(a), C.byref(g), C.byref(d), ws.data_ptr(), nbytes)
    L.check(rc, path)
    L.device_error_check()
    del keep
    return raw, det, term, ws


def via_autograd(path, net, rays, z, lat, grid=None, frame=None, t=None):
    """The same pass through the autograd entry point (details on)."""
    from nonrigid_nerf_b200 import autograd as A
    with torch.no_grad():
        if path == "occupancy":
            return A.field_occupancy(net, rays, z, lat, True, grid) + (None,)
        if path == "terminate":
            return A.field_terminate(net, rays, z, lat, True, t, grid, None)
        return A.field_baked(net, rays, z, lat if _has_bender(net) else None, True, grid, frame) + (None,)


def _exact(net, rays, z, lat, details=False):
    from nonrigid_nerf_b200 import autograd as A
    with torch.no_grad():
        return A.field_rays(net, rays, z, lat if _has_bender(net) else None, details)


def _same_bits(got, want, what):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} words differ, first at flat index {np.flatnonzero(bad)[:8].tolist()}"


def _lookup(pts, grid):
    """baked_reference.lookup in chunks of CHUNK points."""
    vals = _np(grid.values)
    ins, out = [], []
    for s in range(0, pts.shape[0], CHUNK):
        i, v = BR.lookup(pts[s:s + CHUNK], vals, grid.min_point, grid.max_point)
        ins.append(i)
        out.append(v)
    return (np.concatenate(ins), np.concatenate(out)) if ins else (np.zeros(0, bool), np.zeros((0, 4), np.float32))


def _bend(x, frame, b):
    """baked_deformation_reference.bend in chunks of CHUNK points."""
    g = frame.grid
    vals = _np(g.values[frame.index])
    parts = [D.bend(x[s:s + CHUNK], vals, g.min_point, g.max_point, b.rigidity_test_time_cutoff, b.test_time_scaling)
             for s in range(0, x.shape[0], CHUNK)]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def _removal(net, w, rigidity):
    thr = getattr(net, "test_time_nonrigid_object_removal_threshold", None)
    if thr is not None:
        w[:, 3] = np.where(rigidity >= np.float32(thr), w[:, 3] * np.float32(0), w[:, 3])
    return w


# ---- the definitions of each pass ----------------------------------------------------------------------------------------
def define_occupancy(net, rays, z, lat, raw, det, grid, occ):
    """raw = where(kept, exact raw, 0), kept from the numpy lookup of the pass's own (bent) points; the details equal the
    exact pass's.  Returns the keep mask [n * S]."""
    full, det_full = _exact(net, rays, z, lat, True)
    kept = OR.keep(_np(det["input_pts"]).reshape(-1, 3), occ, grid.min_point, grid.max_point)
    f = _np(full).reshape(kept.size, -1)
    _same_bits(_np(raw).reshape(f.shape), np.where(kept[:, None], f, np.float32(0)), "occupancy raw")
    for k in det_full:
        assert _bits_equal(_np(det[k]), _np(det_full[k])), k
    return kept


def define_terminate(net, rays, z, lat, raw, det, idx, t, grid=None, occ=None):
    """raw = where(i < termination_index (and kept), exact raw, 0); termination_index from the pass's own alphas.
    Returns the evaluated mask [n * S]."""
    from nonrigid_nerf_b200 import autograd as A
    full, det_full = _exact(net, rays, z, lat, True)
    n, S = z.shape
    i = _np(idx)
    keep = (np.arange(S)[None, :] < i[:, None]).reshape(-1)
    if grid is not None:
        keep &= OR.keep(_np(det["input_pts"]).reshape(-1, 3), occ, grid.min_point, grid.max_point)
    f = _np(full).reshape(keep.size, -1)
    _same_bits(_np(raw).reshape(f.shape), np.where(keep[:, None], f, np.float32(0)), "termination raw")
    for k in det_full:
        assert _bits_equal(_np(det[k]), _np(det_full[k])), k
    with torch.no_grad():
        c = A.composite(raw, z, rays[:, 3:6], None, False)
    assert np.array_equal(i, TR.termination_index(_np(c["alpha"]), _lib().load().nrn_termination_segment(), t))
    return keep


def define_baked(net, rays, z, lat, raw, det, grid):
    """raw = where(inside, lookup of the pass's own points (object removal applied, raw[4] = 0), exact raw).  Returns the
    inside mask [n * S]."""
    full, _ = _exact(net, rays, z, lat)
    pts = _np(det["input_pts"]).reshape(-1, 3)
    inside, look = _lookup(pts, grid)
    if "rigidity_mask" in det:
        look = _removal(net, look, _np(det["rigidity_mask"]).reshape(-1))
    f = _np(full).reshape(pts.shape[0], -1)
    if f.shape[1] == 5:
        look = np.concatenate([look, np.zeros((look.shape[0], 1), np.float32)], 1)
    assert _bits_equal(_np(raw).reshape(f.shape), np.where(inside[:, None], look, f))
    return inside


def define_deformed(net, rays, z, lat, raw, det, rgrid, frame):
    """Deformed rays: the restatement's bend, then the radiance lookup at c (the trunk at c outside the radiance box),
    every detail included; fallback rays: the baked pass without a deformation grid.  Returns the deformed-ray mask [n]."""
    b = net.ray_bender[0]
    g = frame.grid
    x = D.sample_points(_np(rays), _np(z))
    ok = D.deformed_rays(x, g.min_point, g.max_point)
    n_ch = raw.shape[-1]
    got = {k: _np(det[k]) for k in DETAILS}
    if (~ok).any():
        base_raw, base_det, _, _ = direct("baked", net, rays, z, lat, True, grid=rgrid)
        for k in DETAILS:
            assert _bits_equal(got[k][~ok], _np(base_det[k])[~ok]), k
        assert _bits_equal(_np(raw)[~ok], _np(base_raw)[~ok])
        define_baked(net, rays, z, lat, base_raw, base_det, rgrid)
    if ok.any():
        want = _bend(x[ok].reshape(-1, 3), frame, b)
        for k in DETAILS:
            assert _bits_equal(got[k][ok].reshape(want[k].shape), want[k]), k
        c = want["input_pts"]
        inside, look = _lookup(c, rgrid)
        if n_ch == 5:
            look = np.concatenate([look, np.zeros((look.shape[0], 1), np.float32)], 1)
        trunk = np.zeros((c.shape[0], n_ch), np.float32)
        if (~inside).any():
            trunk[~inside] = _np(_point_raw(net, torch.from_numpy(np.ascontiguousarray(c[~inside])).to(DEV)))
        w = _removal(net, np.where(inside[:, None], look, trunk), want["rigidity_mask"])
        assert _bits_equal(_np(raw)[ok].reshape(-1, n_ch), w)
    return ok


def run_pass(path, net, rays, z, lat, cfg):
    """The pass through its C entry point (poisoned) and its autograd entry point, equal bit for bit, checked against its
    definition on every sample.  Returns (raw, details, termination_index, mask): mask is the kept [n * S] mask of the
    samples the trunk evaluated (occupancy, terminate, baked) or the deformed rays [n]."""
    raw, det, idx, ws = direct(path, net, rays, z, lat, True, cfg.get("grid"), cfg.get("frame"), cfg.get("t"))
    del ws
    a_raw, a_det, a_idx = via_autograd(path, net, rays, z, lat, cfg.get("grid"), cfg.get("frame"), cfg.get("t"))
    assert f32_bits_equal(raw, a_raw) and set(det) == set(a_det)
    assert all(f32_bits_equal(det[k], a_det[k]) for k in det)
    assert idx is None or torch.equal(idx, a_idx)
    if path == "occupancy":
        mask = define_occupancy(net, rays, z, lat, raw, det, cfg["grid"], cfg["occ"])
    elif path == "terminate":
        mask = define_terminate(net, rays, z, lat, raw, det, idx, cfg["t"], cfg.get("grid"), cfg.get("occ"))
    elif path == "baked":
        mask = ~define_baked(net, rays, z, lat, raw, det, cfg["grid"])
    else:
        mask = define_deformed(net, rays, z, lat, raw, det, cfg["grid"], cfg["frame"])
    return raw, det, idx, mask


# ---- rendering at the render chunk ---------------------------------------------------------------------------------------
def _render(coarse, fine, r, chunk=N, **kw):
    from nonrigid_nerf_b200 import train as T
    n = r["rays_o"].shape[0]
    args = dict(network_query_fn=None, perturb=0.0, N_importance=NI, network_fine=fine, N_samples=NS, network_fn=coarse,
                use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    args.update(kw)
    with torch.no_grad():
        rgb, disp, acc, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, near=r["near"], far=r["far"],
                                      additional_pixel_information={"ray_bending_latents": r["latents"][:n].to(DEV)},
                                      detailed_output=True, retraw=True, **args)
    _lib().device_error_check()
    out = dict(ex)
    out.update(rgb_map=rgb, disp_map=disp, acc_map=acc)
    return out


def _assert_same(a, b, skip=()):
    ka, kb = set(a) - set(skip), set(b) - set(skip)
    assert ka == kb, ka ^ kb
    for k in ka:
        x, y = a[k], b[k]
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if x.is_floating_point():
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), k   # bit for bit
        else:
            assert torch.equal(x, y), k


def _chunk_independent(coarse, fine, r, got, **kw):
    _assert_same(got, _render(coarse, fine, r, chunk=4096, **kw))
    print(f"  chunk = {N} and chunk = 4096 render the same frame bit for bit ({len(got)} outputs)")


def _rays_of_kept(mask, S, ks):
    """The rays that hold kept samples number ks (compaction is in order)."""
    nz = np.flatnonzero(mask)
    return {int(nz[k]) // S for k in ks if 0 <= k < nz.size}


def _sweep_items(total, per):
    """First and last items of the persistent CTAs' first and last sweep over `total` items in tiles of `per`."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    T = -(-total // per)
    return [t * per + o for t in (sms - 1, sms, T - sms - 1, T - sms) if 0 <= t < T for o in (0, per - 1)]


def _stride_items(total):
    s = _stride()
    return [j * s + o for j in range(1, -(-total // s)) for o in (-1, 0)]


def composite_sampled(got, tag, extra_rays):
    """The fine compositing of sampled rays of a render against the fp64 bounds of tests/ray_reference.py on the kernel's
    own raw and alpha: the first and last rays, those of the field launches' first and last sweeps, and `extra_rays`."""
    S = NS + NI
    rays = {0, 1, N - 2, N - 1} | set(extra_rays)
    for s_pass in (NS, S):
        rays.update(i // s_pass for i in _sweep_items(N * s_pass, SL.TILE_M))
    sel = torch.tensor(sorted(r for r in rays if 0 <= r < N), device=DEV)
    rep = Report(f"{tag}: {sel.numel()} sampled rays", quiet=True)
    raw, alpha = got["raw"][sel], got["fine_opacity_alpha"][sel]
    ref = RR.composite_ref(alpha, raw, torch.zeros_like(alpha))
    for k, g in (("weights", got["fine_visibility_weights"][sel]), ("rgb", got["rgb_map"][sel]), ("acc", got["acc_map"][sel])):
        rep.check(f"fine {k}", g, *ref[k], c_scan(S), floor=UNDERFLOW)
    rep.worst()


def _passes(path, coarse, fine, r, cfg_c, cfg_f):
    """Both passes of the render, the fine one on the depths the coarse pass's compositing resamples, each checked on
    every sample (run_pass).  Returns (raw_c, det_c, mask_c, idx_c, c0, raw_f, det_f, mask_f, idx_f, c1)."""
    from nonrigid_nerf_b200 import autograd as A, ops
    rays, lat = helpers.rays8(r, DEV), r["latents"].to(DEV)
    with torch.no_grad():
        z = ops.sample_coarse(rays, NS, None, False)
        raw_c, det_c, idx_c, mask_c = run_pass(path, coarse, rays, z, lat, cfg_c)
        c0 = A.composite(raw_c, z, rays[:, 3:6], None, False, NI, None)
        z_f = c0["z_vals_out"]
        raw_f, det_f, idx_f, mask_f = run_pass(path, fine, rays, z_f, lat, cfg_f)
        c1 = A.composite(raw_f, z_f, rays[:, 3:6], None, False)
    return raw_c, det_c, mask_c, idx_c, c0, raw_f, det_f, mask_f, idx_f, c1


def _render_equals_passes(got, raw_f, c0, c1, det_c, det_f):
    assert f32_bits_equal(got["input_pts"], det_c["input_pts"]) and f32_bits_equal(got["fine_input_pts"], det_f["input_pts"])
    for k, v in (("raw", raw_f), ("rgb_map", c1["rgb_map"]), ("disp_map", c1["disp_map"]), ("acc_map", c1["acc_map"]),
                 ("rgb0", c0["rgb_map"])):
        assert f32_bits_equal(got[k], v), k


def _scatter_premise(tag, kept):
    k = int(kept.sum())
    print(f"  [{tag}] kept {k} of {kept.size} samples: occ_scatter_kernel runs {_strides(k)} strides of {_stride()}, "
          f"occ_scan_kernel {_scan_chunks(kept.size)} chunks of 1024 block counts, field_fwd_kept_kernel "
          f"{-(-k // SL.TILE_M)} tiles")
    return k


def _occ_grid(pts, frac, seed, res=(24, 20, 28)):
    """A grid over the box of pts whose occupied cells, taken in random order, hold about `frac` of pts."""
    lo = (pts.min(0) - np.float32(0.01)).astype(np.float32)
    hi = (pts.max(0) + np.float32(0.01)).astype(np.float32)
    per_cell = np.bincount(OR.cells(pts, res, lo, hi), minlength=res[0] * res[1] * res[2])
    order = np.random.RandomState(seed).permutation(per_cell.size)
    take = order[:np.searchsorted(np.cumsum(per_cell[order]), frac * pts.shape[0]) + 1]
    occ = np.zeros(per_cell.size, bool)
    occ[take] = True
    occ = occ.reshape(res[2], res[1], res[0])
    return _G().OccupancyGrid(torch.from_numpy(OR.pack(occ)).to(DEV), lo, hi, res), occ


def _half_box(net, pts, res=(33, 29, 31)):
    """A radiance grid baked over the box of pts, cut at the median x: about half of them inside."""
    lo, hi = pts.min(0).astype(np.float32), pts.max(0).astype(np.float32)
    hi[0] = np.float32(np.median(pts[:, 0]))
    return _G().bake_radiance(net, lo, hi, res)


def _far_grid(net):
    return _G().bake_radiance(net, [50.0] * 3, [51.0] * 3, 2)


def _opaque(nets, r, cross):
    """The sigma bias that makes T cross 1e-4 about `cross` of the way along [near, far] (test_termination_gpu)."""
    import math
    d = float(r["rays_d"].norm(dim=-1).median())
    sigma = math.log(1e4) / (cross * (float(r["far"]) - float(r["near"])) * d)
    with torch.no_grad():
        for net in nets:
            net.output_linear.bias[3] += sigma


# ---- part 1: identity at the render chunk ---------------------------------------------------------------------------------
IDENTITY = [("occupancy", True), ("occupancy", False), ("terminate", True), ("terminate", False), ("baked", True),
            ("baked", False), ("deformed", True)]


@pytest.mark.parametrize("path,bender", IDENTITY)
def test_identity_configurations_render_as_without(path, bender):
    """An all-occupied grid, early_termination = 0 and a radiance box holding no sample render as render(); a deformation
    box holding no ray whole renders as the baked render without it, every ray through gather, field_bend_rays_kernel and
    scatter.  Every output with detailed_output, bit for bit, and chunk independent."""
    coarse, fine, b = _models(bender)
    r = O.make_rays(9101, N)
    skip = ()
    if path == "terminate":
        _opaque((coarse, fine), r, 0.5)
    base = _render(coarse, fine, r)
    if path == "occupancy":
        res = (8, 8, 8)
        occ = np.ones(res[::-1], bool)
        kw = {"occupancy": _G().OccupancyGrid(torch.from_numpy(OR.pack(occ)).to(DEV), np.float32([-0.2, -0.2, -0.7]),
                                              np.float32([0.3, 0.2, 0.45]), res)}
        print(f"  [{path}] every sample kept: {N * NS} coarse, {N * (NS + NI)} fine; occ_scatter_kernel "
              f"{_strides(N * NS)} / {_strides(N * (NS + NI))} strides")
        assert N * NS > 2 * _stride()
    elif path == "terminate":
        kw = {"early_termination": 0.0}
        skip = ("termination_index", "termination_index0")
    elif path == "baked":
        kw = {"baked": _G().BakedScene(_far_grid(coarse), _far_grid(fine))}
    else:
        pts = base["input_pts"].reshape(-1, 3).cpu().numpy()
        scene = _G().BakedScene(_half_box(coarse, pts), _half_box(fine, pts))
        base = _render(coarse, fine, r, baked=scene)
        frame = _G().bake_deformation(b, _lats(2, 4), [50.0] * 3, [51.0] * 3, 2).frame(1)
        kw = {"baked": _G().BakedScene(scene.coarse, scene.fine, frame)}
        for s_pass in (NS, NS + NI):
            assert N * s_pass > 2 * _stride()
            print(f"  [{path}] S = {s_pass}: all {N} rays fall back; deform_gather_kernel / deform_scatter_kernel run "
                  f"{_strides(N * max(s_pass, 32))} / {_strides(N * s_pass)} strides, field_bend_rays_kernel "
                  f"{N * s_pass // SL.TILE_M} tiles")
    got = _render(coarse, fine, r, **kw)
    _assert_same(base, got, skip)
    if path == "terminate":
        assert torch.all(got["termination_index0"] == NS) and torch.all(got["termination_index"] == NS + NI)
    _chunk_independent(coarse, fine, r, got, **kw)


def test_deformation_box_holding_every_ray():
    """Fallback count 0: gather, field_bend_rays_kernel and scatter run with a device count of zero.  Per pass, every
    sample is the restatement's bend followed by the lookup, or the trunk at c outside the radiance box."""
    coarse, fine, b = _models(True)
    r = O.make_rays(9102, N)
    o = r["rays_o"].numpy()
    d = r["rays_d"].numpy()
    ends = np.concatenate([o + d * np.float32(r["near"]), o + d * np.float32(r["far"])])
    lo, hi = _box(ends, 0.01)
    frame = _G().bake_deformation(b, _lats(3, 2), lo, hi, (21, 17, 19)).frame(2)
    base = _render(coarse, fine, r)
    pts = base["input_pts"].reshape(-1, 3).cpu().numpy()
    rc, rf = _half_box(coarse, pts), _half_box(fine, pts)
    scene = _G().BakedScene(rc, rf, frame)
    got = _render(coarse, fine, r, baked=scene)
    raw_c, det_c, ok_c, _, c0, raw_f, det_f, ok_f, _, c1 = _passes("deformed", coarse, fine, r, {"grid": rc, "frame": frame},
                                                                    {"grid": rf, "frame": frame})
    assert ok_c.all() and ok_f.all()
    print(f"  [deformed, every ray inside] fallback rays 0 of {N} in both passes")
    _render_equals_passes(got, raw_f, c0, c1, det_c, det_f)
    composite_sampled(got, "deformed, every ray inside", ())
    _chunk_independent(coarse, fine, r, got, baked=scene)


# ---- part 1: partial configurations on every sample -----------------------------------------------------------------------
@pytest.mark.parametrize("bender", [True, False])
def test_occupancy_grid_keeping_30_percent(bender):
    coarse, fine, b = _models(bender)
    if bender:
        coarse.test_time_nonrigid_object_removal_threshold = fine.test_time_nonrigid_object_removal_threshold = 0.6
    r = O.make_rays(9103, N)
    base = _render(coarse, fine, r)
    grid, occ = _occ_grid(base["input_pts"].reshape(-1, 3).cpu().numpy(), 0.3, 7)
    cfg = {"grid": grid, "occ": occ}
    raw_c, det_c, kept_c, _, c0, raw_f, det_f, kept_f, _, c1 = _passes("occupancy", coarse, fine, r, cfg, cfg)
    k_c, k_f = _scatter_premise("occupancy coarse", kept_c), _scatter_premise("occupancy fine", kept_f)
    assert abs(k_c / kept_c.size - 0.3) < 0.1 and k_c > 2 * _stride() and k_f > 2 * _stride()
    got = _render(coarse, fine, r, occupancy=grid)
    _render_equals_passes(got, raw_f, c0, c1, det_c, det_f)
    S = NS + NI
    extra = _rays_of_kept(kept_f, S, _stride_items(k_f) + _sweep_items(k_f, SL.TILE_M))
    composite_sampled(got, f"occupancy bender={bender}", extra)
    _chunk_independent(coarse, fine, r, got, occupancy=grid)


@pytest.mark.parametrize("with_grid", [False, True])
def test_early_termination_opaque(with_grid):
    coarse, fine, b = _models(True, boost=0.0)
    r = O.make_rays(9104, N)
    _opaque((coarse, fine), r, 0.5)
    t = 1e-4
    cfg, kw = {"t": t}, {"early_termination": t}
    if with_grid:
        base = _render(coarse, fine, r)
        cfg["grid"], cfg["occ"] = _occ_grid(base["input_pts"].reshape(-1, 3).cpu().numpy(), 0.8, 9)
        kw["occupancy"] = cfg["grid"]
    raw_c, det_c, ev_c, idx_c, c0, raw_f, det_f, ev_f, idx_f, c1 = _passes("terminate", coarse, fine, r, cfg, cfg)
    died = float((idx_c < NS).float().mean())
    print(f"  [terminate grid={with_grid}] coarse: {died:.2f} of the rays die, {int(ev_c.sum())} of {ev_c.size} samples "
          f"evaluated; fine: {int(ev_f.sum())} of {ev_f.size}; a round's scatter runs at most {_strides(N * 16)} strides")
    assert died > 0.05   # rounds after the first compact fewer slots than there are rays (skipped samples have alpha 0)
    got = _render(coarse, fine, r, **kw)
    _render_equals_passes(got, raw_f, c0, c1, det_c, det_f)
    assert torch.equal(got["termination_index0"], idx_c) and torch.equal(got["termination_index"], idx_f)
    composite_sampled(got, f"terminate grid={with_grid}", _rays_of_kept(ev_f, NS + NI, _sweep_items(int(ev_f.sum()), SL.TILE_M)))
    _chunk_independent(coarse, fine, r, got, **kw)


@pytest.mark.parametrize("bender", [True, False])
def test_baked_half_box(bender):
    coarse, fine, b = _models(bender)
    if bender:
        coarse.test_time_nonrigid_object_removal_threshold = fine.test_time_nonrigid_object_removal_threshold = 0.6
    r = O.make_rays(9105, N)
    base = _render(coarse, fine, r)
    rc = _half_box(coarse, base["input_pts"].reshape(-1, 3).cpu().numpy())
    rf = _half_box(fine, base["fine_input_pts"].reshape(-1, 3).cpu().numpy())
    raw_c, det_c, out_c, _, c0, raw_f, det_f, out_f, _, c1 = _passes("baked", coarse, fine, r, {"grid": rc}, {"grid": rf})
    k_c, k_f = _scatter_premise("baked coarse", out_c), _scatter_premise("baked fine", out_f)
    assert 0.3 < k_c / out_c.size < 0.7 and k_c > 2 * _stride() and k_f > 2 * _stride()
    scene = _G().BakedScene(rc, rf)
    got = _render(coarse, fine, r, baked=scene)
    _render_equals_passes(got, raw_f, c0, c1, det_c, det_f)
    extra = _rays_of_kept(out_f, NS + NI, _stride_items(k_f) + _sweep_items(k_f, SL.TILE_M))
    composite_sampled(got, f"baked bender={bender}", extra)
    _chunk_independent(coarse, fine, r, got, baked=scene)


@pytest.mark.parametrize("knob", [None, "cutoff", "scaling", "removal"])
def test_deformation_box_holding_half_the_rays(knob):
    from nonrigid_nerf_b200 import ops
    coarse, fine, b = _models(True)
    if knob == "cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif knob == "scaling":
        b.test_time_scaling = 1.7
    elif knob == "removal":
        coarse.test_time_nonrigid_object_removal_threshold = fine.test_time_nonrigid_object_removal_threshold = 0.5
    r = O.make_rays(9106, N)
    rays = helpers.rays8(r, DEV)
    with torch.no_grad():
        x = D.sample_points(_np(rays), _np(ops.sample_coarse(rays, NS, None, False)))
    lo, hi = _cut_box(x)
    frame = _G().bake_deformation(b, _lats(3, 6), lo, hi, (21, 17, 19)).frame(1)
    base = _render(coarse, fine, r)
    rc = _half_box(coarse, base["input_pts"].reshape(-1, 3).cpu().numpy())
    rf = _half_box(fine, base["fine_input_pts"].reshape(-1, 3).cpu().numpy())
    raw_c, det_c, ok_c, _, c0, raw_f, det_f, ok_f, _, c1 = _passes("deformed", coarse, fine, r, {"grid": rc, "frame": frame},
                                                                    {"grid": rf, "frame": frame})
    for tag, ok, S in (("coarse", ok_c, NS), ("fine", ok_f, NS + NI)):
        k = int((~ok).sum())
        print(f"  [deformed {knob} {tag}] {int(ok.sum())} rays deformed, {k} fall back: deform_gather_kernel / "
              f"deform_scatter_kernel run {_strides(k * max(S, 32))} / {_strides(k * S)} strides")
        assert 0.3 < ok.mean() < 0.85 and k * S > 2 * _stride()
    scene = _G().BakedScene(rc, rf, frame)
    got = _render(coarse, fine, r, baked=scene)
    _render_equals_passes(got, raw_f, c0, c1, det_c, det_f)
    S = NS + NI
    fb = np.flatnonzero(~ok_f)
    extra = {int(fb[q // S]) for q in _stride_items(fb.size * S) if q // S < fb.size}
    composite_sampled(got, f"deformed {knob}", extra)
    _chunk_independent(coarse, fine, r, got, baked=scene)


# ---- part 2: one pass past 2^31 bytes per path ------------------------------------------------------------------------------
def _need(gib):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib:.0f} GiB of device memory, {free / 2 ** 30:.1f} GiB free")


def _big_rays(seed, n, S):
    from nonrigid_nerf_b200 import ops
    rs = np.random.RandomState(seed)
    H, W, focal = 384, 512, 256.61   # oracle.make_rays' camera, without its per-ray targets
    px, py = rs.randint(0, W, size=n).astype(np.float32), rs.randint(0, H, size=n).astype(np.float32)
    r = O.make_rays(seed, 1)
    d = torch.from_numpy(np.stack([(px - W * 0.5) / focal, -(py - H * 0.5) / focal, -np.ones_like(px)], -1))
    ang = 0.2
    rot = torch.tensor([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], dtype=torch.float32)
    rays_d = (d @ rot.T).float()
    rays = torch.empty(n, 8)
    rays[:, 0:3] = r["rays_o"][0]
    rays[:, 3:6] = rays_d
    rays[:, 6], rays[:, 7] = float(r["near"]), float(r["far"])
    rays = rays.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    lat = torch.randn(n, 32, generator=g, device=DEV) * 0.1
    with torch.no_grad():
        z = ops.sample_coarse(rays, S, None, False)
    return rays, z, lat


def _byte_rays(buffers, S):
    """{buffer: rays} whose samples hold bytes 2^31 / 2^32 of each buffer, and their neighbours.  buffers: {name:
    (total bytes, bytes per item, item -> sample)}."""
    out = {}
    for name, (total, per, to_sample) in buffers.items():
        assert total > 2 ** 31, f"{name}: {total} bytes, not past 2^31"
        rays = set()
        for B in LIMITS:
            if B < total:
                ray = int(to_sample(B // per)) // S
                rays.update({ray - 1, ray, ray + 1})
        out[name] = rays
        print(f"    {name}: {total} bytes ({total / 2 ** 31:.2f} x 2^31); rays at the boundaries {sorted(rays)}")
    return out


def _sel(n, named, extra=(), seed=0):
    rays = {0, 1, n - 2, n - 1} | set(extra)
    for r in named.values():
        rays |= r
    rays |= set(np.random.RandomState(seed).randint(0, n, 16).tolist())
    return torch.tensor(sorted(x for x in rays if 0 <= x < n), device=DEV)


def _outside(pts, lo, hi):
    """[P] bool on the GPU: outside [lo, hi] or not finite, the rule of an empty occupancy grid and of a radiance box."""
    lo_t, hi_t = torch.tensor(lo, device=DEV), torch.tensor(hi, device=DEV)
    return ~((pts >= lo_t) & (pts <= hi_t)).all(1)


def _corner_box(pts, frac):
    """A box holding about `frac` of pts (the ones of least x): lo at their minimum, hi[0] at the frac quantile of x."""
    lo, hi = pts.min(0).astype(np.float32), pts.max(0).astype(np.float32)
    hi[0] = np.float32(np.quantile(pts[:, 0], frac))
    return lo, hi


@pytest.mark.parametrize("path", ["occupancy", "baked"])
def test_pass_past_2_31_with_bender(path):
    """1.5 M rays x 128 samples (196.6 M) with a bender, 97 % of the samples outside the grid's box (an empty occupancy
    grid, or a radiance grid): ws, raw, the kept points and their raw (craw) pass 2^31 bytes, and ws and raw 2^32."""
    n, S = 1_536_000, 128
    _need(26)
    t0 = time.perf_counter()
    coarse, _, _ = _models(True)
    L = _lib()
    lib = L.load()
    P, out_ch = n * S, 5
    rays, z, lat = _big_rays(9201, n, S)
    # the box from the bent points of a small call on every 64th ray
    probe = torch.arange(0, n, 64, device=DEV)
    _, pdet, _, _ = direct("occupancy", coarse, rays[probe], z[probe], lat[probe], True, grid=_empty_grid([0] * 3, [1] * 3))
    lo, hi = _corner_box(_np(pdet["input_pts"]).reshape(-1, 3), 0.03)
    if path == "occupancy":
        grid = _empty_grid(lo, hi)
        cfg = {"grid": grid, "occ": np.zeros((8, 8, 8), bool)}
    else:
        grid = _G().bake_radiance(coarse, lo, hi, (17, 19, 23))
        cfg = {"grid": grid}
    raw, _, _, ws = direct(path, coarse, rays, z, lat, False, grid=grid)
    bent = ws[:P * 16].view(torch.float32).view(P, 4)[:, :3]
    kept = _outside(bent, lo, hi)
    nz = torch.nonzero(kept).squeeze(1)
    K = nz.numel()
    off = _align(P * 16)
    off_idx = off + _align(P * 12)
    off_craw = off_idx + _align(P * 4)
    off_count = off_craw + _align(P * out_ch * 4)
    count = int(ws[off_count:off_count + 4].view(torch.int32)[0])
    assert count == K, (count, K)
    assert torch.equal(ws[off_idx:off_idx + 4 * K].view(torch.int32).long(), nz), "kept indices out of order"
    need = (lib.nrn_occupancy_workspace_bytes if path == "occupancy" else lib.nrn_baked_workspace_bytes)(n, S, out_ch, 1)
    assert ws.numel() == need >= off_count
    print(f"  [{path} {n} x {S}] {P} samples, {K} kept ({K / P:.3f}): occ_scatter_kernel {_strides(K)} strides, "
          f"occ_scan_kernel {_scan_chunks(P)} chunks, field_fwd_kept_kernel {-(-K // SL.TILE_M)} tiles")
    named = _byte_rays({"ws": (P * 16, 16, int), "raw": (P * out_ch * 4, out_ch * 4, int),
                        "craw": (K * out_ch * 4, out_ch * 4, lambda k: int(nz[k])), "kept_xyz": (K * 12, 12, lambda k: int(nz[k]))}, S)
    extra = [int(nz[k]) // S for k in _stride_items(K)[:4] + _stride_items(K)[-2:]]   # at the scatter's stride boundaries
    del nz, kept
    sel = _sel(n, named, extra, 1)
    sel_ws = ws[:P * 16].view(torch.float32).view(n, S, 4)[sel].clone()
    big = raw[sel].clone()
    del ws, raw, bent
    torch.cuda.empty_cache()
    s_raw, s_det, _, _ = direct(path, coarse, rays[sel], z[sel], lat[sel], True, grid=grid)
    assert f32_bits_equal(big, s_raw), f"{path}: the sampled rays of the large pass differ from a call on just those rays"
    assert f32_bits_equal(sel_ws[..., :3].contiguous(), s_det["input_pts"])
    if path == "occupancy":
        define_occupancy(coarse, rays[sel], z[sel], lat[sel], s_raw, s_det, grid, cfg["occ"])
    else:
        define_baked(coarse, rays[sel], z[sel], lat[sel], s_raw, s_det, grid)
    print(f"  [{path} {n} x {S}] {sel.numel()} rays equal a small call and the definition; {time.perf_counter() - t0:.1f} s")


def _empty_grid(lo, hi, res=(8, 8, 8)):
    occ = np.zeros(res[::-1], bool)
    return _G().OccupancyGrid(torch.from_numpy(OR.pack(occ)).to(DEV), np.float32(lo), np.float32(hi), res)


def test_termination_past_2_31():
    """6.8 M rays x 32 samples with a bender and opaque densities: one round's craw (n x 16 slots x 20 bytes) passes
    2^31 bytes, ws passes 2^31 and raw 2^32."""
    n, S = 6_800_000, 32
    _need(24)
    t0 = time.perf_counter()
    coarse, _, _ = _models(True, boost=0.0)
    K = _lib().load().nrn_termination_segment()
    P, out_ch = n * S, 5
    rays, z, lat = _big_rays(9202, n, S)
    _opaque((coarse,), {"rays_d": rays[:4096, 3:6].cpu(), "near": rays[0, 6].item(), "far": rays[0, 7].item()}, 0.5)
    t = 1e-4
    raw, _, idx, ws = direct("terminate", coarse, rays, z, lat, False, t=t)
    del ws
    died = float((idx < S).float().mean())
    print(f"  [terminate {n} x {S}] {died:.2f} of the rays die; round 0 keeps {n * K} slots: occ_scatter_kernel "
          f"{_strides(n * K)} strides, occ_scan_kernel {_scan_chunks(n * K)} chunks")
    assert 0.05 < died
    named = _byte_rays({"ws": (P * 16, 16, int), "raw": (P * out_ch * 4, out_ch * 4, int),
                        "craw (round 0)": (n * K * out_ch * 4, out_ch * 4, lambda q: (q // K) * S + q % K)}, S)
    sel = _sel(n, named, [q // K for q in _stride_items(n * K)[:4]], 2)
    big, big_idx = raw[sel].clone(), idx[sel].clone()
    del raw, idx
    torch.cuda.empty_cache()
    s_raw, s_det, s_idx, _ = direct("terminate", coarse, rays[sel], z[sel], lat[sel], True, t=t)
    assert f32_bits_equal(big, s_raw) and torch.equal(big_idx, s_idx)
    define_terminate(coarse, rays[sel], z[sel], lat[sel], s_raw, s_det, s_idx, t)
    print(f"  [terminate {n} x {S}] {sel.numel()} rays equal a small call and the definition; {time.perf_counter() - t0:.1f} s")


def test_deformed_past_2_31():
    """8.65 M rays x 16 samples, 99 % of them falling back: deform_rays_kernel runs past its 2^23-ray stride, the
    fallback scan over 8,448 block counts, and ws, bw (the gathered rays' bend workspace), raw and craw pass 2^31 bytes."""
    n, S = 8_650_000, 16
    _need(30)
    t0 = time.perf_counter()
    coarse, _, b = _models(True)
    lib = _lib().load()
    P, out_ch = n * S, 5
    rays, z, lat = _big_rays(9203, n, S)
    x = rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]     # multiply, then add: the kernel's points, exactly
    xmax = x[..., 0].amax(1)
    lo = x.reshape(-1, 3).amin(0).cpu().numpy() - np.float32(0.01)
    hi = x.reshape(-1, 3).amax(0).cpu().numpy() + np.float32(0.01)
    hi[0] = np.float32(torch.quantile(xmax[::97].float(), 0.01).item())
    lo, hi = lo.astype(np.float32), hi.astype(np.float32)
    fallback = _outside(x.reshape(-1, 3), lo, hi).view(n, S).any(1)
    del x, xmax
    Kf = int(fallback.sum())
    frame = _G().bake_deformation(b, _lats(2, 3), lo, hi, (13, 11, 9)).frame(0)
    probe = torch.arange(0, n, 256, device=DEV)
    _, pdet, _, _ = direct("baked", coarse, rays[probe], z[probe], lat[probe], True, grid=_far_grid(coarse))
    rlo, rhi = _corner_box(_np(pdet["input_pts"]).reshape(-1, 3), 0.1)
    rgrid = _G().bake_radiance(coarse, rlo, rhi, (15, 13, 11))
    raw, _, _, ws = direct("deformed", coarse, rays, z, lat, False, grid=rgrid, frame=frame)
    base = lib.nrn_baked_workspace_bytes(n, S, out_ch, 1)
    flag = ws[base:base + n]
    assert torch.equal(flag.bool(), fallback), "fallback flags differ from the restatement"
    off_f = base + _align(n)
    off_count = off_f + _align(4 * (-(-n // 1024) + 1))
    assert int(ws[off_count:off_count + 4].view(torch.int32)[0]) == Kf
    off_idx = off_count + 256
    fb = torch.nonzero(fallback).squeeze(1)
    assert torch.equal(ws[off_idx:off_idx + 4 * Kf].view(torch.int32).long(), fb), "fallback rays out of order"
    bent = ws[:P * 16].view(torch.float32).view(P, 4)[:, :3]
    kept = _outside(bent, rlo, rhi)
    nz = torch.nonzero(kept).squeeze(1)
    K = nz.numel()
    print(f"  [deformed {n} x {S}] {n - Kf} rays deformed, {Kf} fall back: deform_rays_kernel {-(-n // (1 << 23))} strides "
          f"of 2^23 rays, the fallback scan {_ceil(n, 1024)} block counts ({_scan_chunks(n)} chunks), "
          f"deform_gather_kernel {_strides(Kf * 32)} and deform_scatter_kernel {_strides(Kf * S)} strides, "
          f"field_bend_rays_kernel {-(-Kf * S // SL.TILE_M)} tiles; {K} samples outside the radiance box: occ_scatter_kernel "
          f"{_strides(K)} strides")
    assert n > 1 << 23 and -(-n // 1024) > 1024 and Kf * S > 2 * _stride()
    named = _byte_rays({"ws": (P * 16, 16, int), "raw": (P * out_ch * 4, out_ch * 4, int),
                        "bw": (Kf * S * 16, 16, lambda q: int(fb[q // S]) * S + q % S),
                        "craw": (K * out_ch * 4, out_ch * 4, lambda k: int(nz[k]))}, S)
    extra = [(1 << 23) - 1, 1 << 23, (1 << 23) + 1] + [int(fb[q // S]) for q in _stride_items(Kf * S)[:4]]
    dr = torch.nonzero(~fallback).squeeze(1)   # deformed rays: the first and last, random ones, and those past 2^23
    past = dr[dr >= 1 << 23]
    assert past.numel() > 0
    pick = torch.randint(0, dr.numel(), (8,), generator=torch.Generator().manual_seed(3)).tolist()
    extra += [int(dr[0]), int(dr[-1]), int(past[0])] + [int(dr[i]) for i in pick]
    sel = _sel(n, named, extra, 3)
    big = raw[sel].clone()
    del ws, raw, bent, kept, nz, flag
    torch.cuda.empty_cache()
    s_raw, s_det, _, _ = direct("deformed", coarse, rays[sel], z[sel], lat[sel], True, grid=rgrid, frame=frame)
    assert f32_bits_equal(big, s_raw), "the sampled rays of the large pass differ from a call on just those rays"
    ok = define_deformed(coarse, rays[sel], z[sel], lat[sel], s_raw, s_det, rgrid, frame)
    assert np.array_equal(ok, ~_np(fallback[sel])) and ok.sum() >= 4
    print(f"  [deformed {n} x {S}] {sel.numel()} rays ({int(ok.sum())} deformed) equal a small call and the definition; "
          f"{time.perf_counter() - t0:.1f} s")


def test_baked_without_bender_past_2_28_samples():
    """2.15 M rays x 128 samples (275 M > 2^28) without a bender: baked_rays_kernel runs a second stride; raw passes
    2^32 bytes.  95 % of the samples inside the box."""
    n, S = 2_150_000, 128
    _need(30)
    t0 = time.perf_counter()
    coarse, _, _ = _models(False)
    P, out_ch = n * S, 5
    assert P > 1 << 28
    rays, z, lat = _big_rays(9204, n, S)
    x = (rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    lo, hi = _corner_box(_np(x[::4099]), 0.95)
    grid = _G().bake_radiance(coarse, lo, hi, (19, 17, 15))
    raw, _, _, ws = direct("baked", coarse, rays, z, lat, False, grid=grid)
    kept = _outside(x, lo, hi)
    del x
    K = int(kept.sum())
    off_count = _align(P * 12) + _align(P * 4) + _align(P * out_ch * 4)
    assert int(ws[off_count:off_count + 4].view(torch.int32)[0]) == K
    print(f"  [baked no bender {n} x {S}] {P} samples: baked_rays_kernel {-(-P // (1 << 28))} strides of 2^28; {K} outside "
          f"the box: occ_scatter_kernel {_strides(K)} strides")
    named = _byte_rays({"raw": (P * out_ch * 4, out_ch * 4, int)}, S)
    extra = [((1 << 28) + o) // S for o in (-1, 0, 1)]
    sel = _sel(n, named, extra, 4)
    big = raw[sel].clone()
    del ws, raw, kept
    torch.cuda.empty_cache()
    s_raw, s_det, _, _ = direct("baked", coarse, rays[sel], z[sel], lat[sel], True, grid=grid)
    assert f32_bits_equal(big, s_raw)
    define_baked(coarse, rays[sel], z[sel], lat[sel], s_raw, s_det, grid)
    print(f"  [baked no bender {n} x {S}] {sel.numel()} rays equal a small call and the definition; {time.perf_counter() - t0:.1f} s")
