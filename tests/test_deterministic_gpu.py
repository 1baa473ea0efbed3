"""Deterministic mode (torch.use_deterministic_algorithms(True)) on the H100.

  reduction rule  nrn_field_backward_det / nrn_divergence_forward_det: the per-ray results equal, bit for bit, a numpy
                  float32 sum of the kernels' own rows taken sequentially in the documented walk order; every other
                  output equals the atomic entry point's bit for bit; the atomic path and an fp64 sum of the same rows
                  agree within fp32 reassociation bounds derived from sum |row|.  S in {128, 64, 100, 24, 2}: uniform and
                  non-uniform warps, rays across tiles and CTAs, ragged last tiles, several waves of CTAs.
  end to end      training_wrapper_class with a bender and all three regularisers (perturb = 1, noise = 1 from a
                  seeded generator) and optim.Adam: two 5-step runs under the flag give bit-identical losses, .grad,
                  parameters and Adam moments; also the time-conditioned model.  The first step still meets golden case
                  H's bounds.
  graph replay    GraphedStep replays under the flag equal the eager deterministic steps bit for bit.
  flag off        the fixed-order reductions are never launched.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import stage_reference as SR
from tests.parity import DEV, poison_f32

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U32 = 2.0 ** -24   # unit roundoff of fp32


class deterministic:
    """torch.use_deterministic_algorithms(True) for the duration of a block."""

    def __enter__(self):
        self.prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev)


def walk_sum(rows, n, s):
    """The fixed-order per-ray sum of det_reduce.cu, in numpy float32: per ray, the points in increasing order; the first
    point 32k of a uniform block (32k + 31 < P, one ray) stands for the whole block.  rows: [P, c] float32.
    Returns (sum [n, c] float32, visited mask [P])."""
    P = n * s
    pos = np.arange(n, dtype=np.int64) * s
    end = pos + s
    acc = np.zeros((n, rows.shape[1]), dtype=np.float32)
    visited = np.zeros(P, dtype=bool)
    while True:
        live = pos < end
        if not live.any():
            break
        idx = pos[live]
        visited[idx] = True
        acc[live] = acc[live] + rows[idx]   # float32 + float32, one addition per ray and step
        uni = (idx % 32 == 0) & (idx + 31 < P) & (idx // s == (idx + 31) // s)
        pos[live] = idx + np.where(uni, 32, 1)
    return acc, visited


def fp64_bound(rows, visited, n, s, factor):
    """fp64 sum of the visited rows per ray and factor * (m - 1) * u * sum |row|, m = rows added per ray."""
    r = np.where(visited[:, None], rows.astype(np.float64), 0.0).reshape(n, s, -1)
    m = visited.reshape(n, s).sum(1)[:, None]
    return r.sum(1), factor * np.maximum(m - 1, 1) * U32 * np.abs(r).sum(1)


SHAPES = [(4099, 128), (2053, 64), (777, 100), (1601, 24), (20001, 2)]


def _bwd(cs, o, det):
    """nrn_field_backward (atomic) or nrn_field_backward_det into poisoned buffers."""
    L = SR._lib()
    lib = L.load()
    a = L.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = cs.n, cs.s, cs.out_ch
    a.d_raw, a.stash, a.relu_mask, a.nerf_packed = cs.d_raw.data_ptr(), o["stash"].data_ptr(), o["mask"].data_ptr(), o["npk"].data_ptr()
    b = {"gstash": SR.poison_bytes(lib.nrn_grad_stash_bytes(cs.n, cs.s)), "scratch": SR.poison_bytes(lib.nrn_wgrad_scratch_bytes()),
         "nerf_grad": poison_f32(lib.nrn_nerf_grad_floats(cs.out_ch)), "bender_grad": poison_f32(lib.nrn_bender_grad_floats()),
         "d_lat": poison_f32(cs.n, 32)}
    a.grad_stash, a.wgrad_scratch, a.nerf_grad = b["gstash"].data_ptr(), b["scratch"].data_ptr(), b["nerf_grad"].data_ptr()
    a.bender_packed = o["bpk"].data_ptr()
    a.unmasked_offsets, a.rigidity_mask = o["un"].data_ptr(), o["rig"].data_ptr()
    a.d_unmasked_offsets, a.d_rigidity_mask = SR.ptr(cs.d_un_up), SR.ptr(cs.d_rig_up)
    a.bender_grad, a.d_latents = b["bender_grad"].data_ptr(), b["d_lat"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    if det:
        b["rows"] = poison_f32(cs.P, 32)
        L.check(lib.nrn_field_backward_det(C.byref(a), b["rows"].data_ptr()), "field_backward_det")
    else:
        L.check(lib.nrn_field_backward(C.byref(a)), "field_backward")
    L.device_error_check()
    return b


@pytest.mark.parametrize("n,s", SHAPES, ids=[f"{n}x{s}" for n, s in SHAPES])
def test_latent_gradient_follows_the_walk_order_bit_for_bit(n, s):
    cs = SR.Case(n, s)
    o = SR.run_forward(cs)
    at, de = _bwd(cs, o, False), _bwd(cs, o, True)
    for k in ("nerf_grad", "bender_grad", "gstash"):
        assert torch.equal(de[k].view(torch.int32 if k != "gstash" else torch.uint8),
                           at[k].view(torch.int32 if k != "gstash" else torch.uint8)), f"{k} differs from the atomic path"
    rows = de["rows"].cpu().numpy()
    ref, visited = walk_sum(rows, n, s)
    got = de["d_lat"].cpu().numpy()
    assert np.isfinite(rows[visited]).all()
    assert np.array_equal(got.view(np.int32), ref.view(np.int32)), "d_latents is not the walk-order float32 sum of its rows"
    exact, bound = fp64_bound(rows, visited, n, s, 1.0)
    assert (np.abs(got - exact) <= bound).all()
    # the atomic path adds the same rows (its warps reduce exactly like the deterministic kernel's) in another order
    atom = at["d_lat"].cpu().numpy().astype(np.float64)
    assert (np.abs(atom - got) <= 2 * bound + 1e-38).all()
    print(f"  [{n}x{s}] rows added {int(visited.sum())} of {n * s}; max |det - atomic| {np.abs(atom - got).max():.3e}")


@pytest.mark.parametrize("n,s", SHAPES, ids=[f"{n}x{s}" for n, s in SHAPES])
def test_divergence_loss_follows_the_walk_order_bit_for_bit(n, s):
    L = SR._lib()
    lib = L.load()
    cs = SR.Case(n, s)
    o = SR.run_forward(cs)
    at = SR.run_divergence_forward(cs, o)
    de = {"tan": SR.poison_bytes(lib.nrn_div_stash_bytes(n, s)), "scal": poison_f32(4, cs.P), "loss": poison_f32(n),
          "rows": poison_f32(cs.P)}
    L.check(lib.nrn_divergence_forward_det(C.byref(SR._div_args(cs, o, de)), de["rows"].data_ptr()), "divergence_forward_det")
    L.device_error_check()
    assert torch.equal(de["tan"], at["tan"]) and torch.equal(de["scal"].view(torch.int32), at["scal"].view(torch.int32))
    rows = de["rows"].cpu().numpy()[:, None]
    ref, visited = walk_sum(rows, n, s)
    got = de["loss"].cpu().numpy()
    assert np.isfinite(rows[visited]).all()
    assert np.array_equal(got.view(np.int32), ref[:, 0].view(np.int32)), "loss is not the walk-order float32 sum of its rows"
    exact, bound = fp64_bound(rows, visited, n, s, 1.0)
    assert (np.abs(got - exact[:, 0]) <= bound[:, 0]).all()
    atom = at["loss"].cpu().numpy().astype(np.float64)
    assert (np.abs(atom - got) <= 2 * bound[:, 0] + 1e-38).all()


def test_empty_batch_launches_nothing():
    from nonrigid_nerf_b200 import _lib as L
    lib = L.load()
    cs = SR.Case(4, 64)
    o = SR.run_forward(cs)
    d = {"tan": SR.poison_bytes(16), "scal": poison_f32(4, 4), "loss": poison_f32(4)}
    a = SR._div_args(cs, o, d)
    a.n_rays = 0
    L.timing_enable(True)
    try:
        assert lib.nrn_divergence_forward_det(C.byref(a), None) == 0
        kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS
        assert all(c == 0 for _, c in L.timing_read(kinds).values())
    finally:
        L.timing_enable(False)
    assert torch.isnan(d["loss"]).all()


# ----------------------------------------------------------------------------------------------------------------------
# end to end
# ----------------------------------------------------------------------------------------------------------------------
def _setup(seed, n, s_c=64, n_imp=64, n_images=86):
    """training_wrapper_class with a bender and the offsets, rigidity and divergence terms, optim.Adam over an n_images-row
    latent table; every random draw (render_rays' four, the divergence probes) from one seeded generator."""
    import types
    from nonrigid_nerf_b200 import optim, parallel
    from tests import helpers
    torch.manual_seed(seed)   # the modules' dead weights (views_linears) keep nn.Linear's random initialisation
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, s_c, n_imp).items()}
    rnd["e"] = torch.randn(n, s_c, 3, generator=g).to(DEV)
    table = (torch.randn(n_images, 32, generator=g) * 0.1).to(DEV)
    pix = torch.stack([torch.randint(0, n_images, (n,), generator=g), torch.randint(0, 384, (n,), generator=g),
                       torch.randint(0, 512, (n,), generator=g)], 1).to(DEV)
    latents = [table[i].clone().requires_grad_(True) for i in range(n_images)]
    params = latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=5e-4)
    targs = types.SimpleNamespace(chunk=32768, N_samples=s_c, N_importance=n_imp, N_iters=200000, offsets_loss_weight=60.0,
                                  divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": n_imp, "network_fine": fine, "N_samples": s_c,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]
    extras = {"imageid_to_timestepid": list(range(n_images))}
    global_step = torch.zeros((), dtype=torch.float32, device=DEV)

    def step(rays_o, rays_d, target, pix):
        opt.zero_grad()
        losses = wrapper(targs, rays_o, rays_d, 100, kw, target, global_step, 0, extras, pix)
        (losses.sum() / n).backward()
        opt.step()
        global_step.add_(1.0)
        return losses.detach()

    return step, inputs, opt, params


def _setup_tc(seed, n):
    """The time-conditioned baseline (no bender) with a trainable latent table, optim.Adam."""
    from nonrigid_nerf_b200 import optim, parallel
    from tests import helpers, test_time_conditioned_gpu as TC
    g = TC._golden()
    r = O.make_rays(seed, n)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    gen = torch.Generator().manual_seed(seed)
    n_images = len(g["latent_table"])
    latents = [(torch.randn(32, generator=gen) * 0.1).to(DEV).requires_grad_(True) for _ in range(n_images)]
    pix = torch.stack([torch.randint(0, n_images, (n,), generator=gen), torch.randint(0, 384, (n,), generator=gen),
                       torch.randint(0, 512, (n,), generator=gen)], 1).to(DEV)
    torch.manual_seed(seed)
    coarse, fine, _ = helpers.tc_models(seed, DEV)
    params = latents + list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=5e-4)
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=None)
    kw = TC._kwargs(coarse, fine, r, rnd, 1.0, 1.0)
    extras = {"imageid_to_timestepid": list(range(n_images))}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]

    def step(rays_o, rays_d, target, pix):
        opt.zero_grad()
        loss = wrapper(TC._targs(), rays_o, rays_d, 100, kw, target, 50000, 0, extras, pix)
        loss.mean().backward()
        opt.step()
        return loss.detach()

    return step, inputs, opt, params


def _state(losses, opt, params):
    grads = [torch.zeros(0, device=DEV) if p.grad is None else p.grad.detach().clone() for p in params]
    return [losses.clone()] + grads + [opt._flat.clone(), opt._m.clone(), opt._v.clone(), opt._step.clone()]


def _run(make, steps=5):
    with deterministic():
        step, inputs, opt, params = make()
        out = []
        for _ in range(steps):
            out.append(_state(step(*inputs), opt, params))
        torch.cuda.synchronize()
    return out


def _bits_equal(a, b):
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _assert_runs_identical(r1, r2, label):
    for i, (s1, s2) in enumerate(zip(r1, r2)):
        for j, (a, b) in enumerate(zip(s1, s2)):
            assert _bits_equal(a, b), f"{label}: step {i + 1}, tensor {j} differs between two deterministic runs"
    assert not _bits_equal(r1[0][-3], r1[-1][-3]), f"{label}: the parameters did not move"


CASES = {
    "1024_64+64": lambda: _setup(8191, 1024),
    "cfg4_8192_64+64": lambda: _setup(8192, 8192),
    "1024_100+50": lambda: _setup(8193, 1024, 100, 50),
    "time_conditioned": lambda: _setup_tc(4100, 1024),
}


@pytest.mark.parametrize("case", list(CASES))
def test_two_deterministic_runs_are_bit_identical(case):
    r1, r2 = _run(CASES[case]), _run(CASES[case])
    _assert_runs_identical(r1, r2, case)


def test_first_deterministic_step_meets_golden_case_H():
    from tests import test_training_wrapper_gpu as TW
    g = np.load(os.path.join(GOLD, "caseH_training_wrapper.npz"))
    with deterministic():
        loss, coarse, fine, bender, latents, _ = TW._run_wrapper(g, True)
    d = float(np.abs(loss.numpy() - g["loss"]).max())
    rel = TW._rel(loss, torch.from_numpy(g["loss"]))
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()] + \
            [("bender." + k, v) for k, v in bender.named_parameters()]
    TW._golden_grad_check(g, named, 1.2e-1, "deterministic")
    e_lat = TW._rel(torch.stack([l.grad for l in latents]).cpu(), torch.from_numpy(g["latent_grads"]))
    assert e_lat <= 8e-2, e_lat


def test_graph_replay_equals_the_eager_deterministic_steps():
    """Six eager deterministic steps against 3 warm-up steps inside GraphedStep (captured under the flag) and 3 replays:
    steps 4..6 are bit-identical in every loss, parameter and Adam moment."""
    from nonrigid_nerf_b200.graphs import GraphedStep
    eager = _run(lambda: _setup(8191, 1024), steps=6)[3:]
    with deterministic():
        step, inputs, opt, params = _setup(8191, 1024)
        graphed = GraphedStep(step, inputs, warmup=3)
        replay = []
        for _ in range(3):
            losses = graphed(*inputs)
            torch.cuda.synchronize()
            st = _state(losses, opt, params)
            replay.append([st[0]] + st[-4:])
    for i, (e, r) in enumerate(zip(eager, replay)):
        for j, (a, b) in enumerate(zip([e[0]] + e[-4:], r)):
            assert _bits_equal(a, b), f"step {4 + i}: tensor {j} of the replay differs from the eager deterministic step"


def test_flag_off_launches_no_fixed_order_reduction():
    from nonrigid_nerf_b200 import _lib as L
    kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS
    counts = {}
    for det in (False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            step, inputs, opt, params = _setup(8191, 1024)
            L.timing_enable(True)
            step(*inputs)
            counts[det] = L.timing_read(kinds)
        finally:
            L.timing_enable(False)
            torch.use_deterministic_algorithms(prev)
    assert counts[False]["latent_reduce"][1] == 0 and counts[False]["div_loss_reduce"][1] == 0
    # with the flag: one latent reduction per field backward (coarse, fine), one loss reduction
    assert counts[True]["latent_reduce"][1] == 2 and counts[True]["div_loss_reduce"][1] == 1
    for k in L.KERNEL_KINDS:
        assert counts[True][k][1] == counts[False][k][1], k
