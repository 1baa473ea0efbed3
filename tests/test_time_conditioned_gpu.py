"""GPU tests of the time-conditioned baseline (NeRF(time_conditioned_baseline=True), no bender): the latent enters L0 and
L5 of the fused kernels as a per-ray bias (csrc/field_fwd.cu), and its gradients come from per-ray sums of the stashed
dY0 / dY5 (csrc/field_bwd.cu).

  * render() coarse + fine and point-mode NeRF.forward vs golden case L (executed reference) and the fp32 restatement;
  * a broadcast latent (stride 0) vs explicit rows, chunked vs un-chunked rendering;
  * each new kernel vs an fp64 reference of its own inputs: the ray bias; the per-ray sums, d z and the latent columns of
    dW0 / dW5 from the gradient stash (decoded with tests/stash_layout.py);
  * the training wrapper's loss and gradients vs golden case L, through fresh gradient buffers and optim.Adam's arena;
  * two backward passes bit-identical, and a CUDA-graph replay of a training step vs the eager step.

Tolerances follow the bending path's tests (fp16 tensor-core operands vs the fp32 reference)."""
import os

import numpy as np
import pytest
import torch

from tests import helpers, stash_layout as SL, tc_reference as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"
O = R.O


def _golden():
    return np.load(os.path.join(GOLD, "caseL_time_conditioned.npz"))


def _kwargs(coarse, fine, r, rnd=None, perturb=0.0, noise=0.0):
    kw = {"network_query_fn": None, "perturb": perturb, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": None, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": noise,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"]}
    if rnd is not None:
        kw["randomness"] = rnd
    return kw


def _render(coarse, fine, r, lat, chunk=32768):
    from nonrigid_nerf_b200 import train as T
    with torch.no_grad():
        rgb, disp, acc, extras = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, retraw=True,
                                          additional_pixel_information={"ray_bending_latents": lat}, **_kwargs(coarse, fine, r))
    return rgb, acc, extras


def test_render_and_point_mode_match_golden_and_oracle():
    from nonrigid_nerf_b200 import _lib
    g = _golden()
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, (cp, fp) = helpers.tc_models(seed, DEV)
    r = O.make_rays(seed, n)
    lat = torch.from_numpy(g["latents"])
    rgb, acc, extras = _render(coarse, fine, r, lat.to(DEV))
    _lib.device_error_check()
    with torch.no_grad():
        ora = R.render_rays(cp, fp, r["rays_o"], r["rays_d"], r["near"], r["far"], lat)
    for name, ours, ref in (("rgb_map", rgb, g["rgb_map"]), ("acc_map", acc, g["acc_map"]), ("rgb0", extras["rgb0"], g["rgb0"])):
        d = float(np.abs(ours.cpu().numpy() - ref).max())
        d_o = float(np.abs(ours.cpu().numpy() - ora[name].numpy()).max())
        print(f"{name}: max |ours - reference| {d:.3e}, |ours - oracle| {d_o:.3e}")
        assert d <= 5e-4 and d_o <= 5e-4, (name, d, d_o)
    e_raw = R.rel(extras["raw"][:16].cpu().numpy(), g["raw"])
    print(f"raw[:16] rel L2 vs reference {e_raw:.3e}")
    assert e_raw <= 1e-2, e_raw
    # point mode: NeRF.forward(x) with x = [xyz (63 columns, the kernel re-derives the encoding) | latent]
    pts, pts_lat = torch.from_numpy(g["pts"]), torch.from_numpy(g["pts_latents"])
    x = torch.zeros(pts.shape[0] * pts.shape[1], 63 + 32)
    x[:, :3] = pts.reshape(-1, 3)
    x[:, 63:] = pts_lat[:, None, :].expand(-1, pts.shape[1], -1).reshape(-1, 32)
    with torch.no_grad():
        raw_pts = coarse(x.to(DEV)).reshape(pts.shape[0], pts.shape[1], -1).cpu()
    e_pts = R.rel(raw_pts.numpy(), g["pts_raw"])
    print(f"point mode raw rel L2 vs reference {e_pts:.3e}")
    assert e_pts <= 1e-2, e_pts


def test_broadcast_latent_and_chunking_are_exact():
    g = _golden()
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, _ = helpers.tc_models(seed, DEV)
    r = O.make_rays(seed, n)
    row = torch.from_numpy(g["latents"][3]).to(DEV)
    rgb_b, acc_b, ex_b = _render(coarse, fine, r, row[None, :].expand(n, 32))        # stride 0: one ray-bias row
    rgb_e, acc_e, ex_e = _render(coarse, fine, r, row[None, :].repeat(n, 1))         # explicit rows
    assert torch.equal(rgb_b, rgb_e) and torch.equal(acc_b, acc_e) and torch.equal(ex_b["raw"], ex_e["raw"])
    lat = torch.from_numpy(g["latents"]).to(DEV)
    rgb_1, acc_1, ex_1 = _render(coarse, fine, r, lat)
    rgb_c, acc_c, ex_c = _render(coarse, fine, r, lat, chunk=37)
    d = max(float((rgb_1 - rgb_c).abs().max()), float((acc_1 - acc_c).abs().max()), float((ex_1["rgb0"] - ex_c["rgb0"]).abs().max()))
    print(f"chunk=37 vs one chunk: max difference {d:.3e}")
    assert d <= 1e-6, d


def test_ray_bias_matches_fp64():
    from nonrigid_nerf_b200 import ops
    coarse, _, _ = helpers.tc_models(R.SEED, DEV)
    lat = torch.randn(300, 32, generator=torch.Generator().manual_seed(3)).to(DEV)
    rb = ops.tc_ray_bias(coarse, lat, lat.stride(0))
    w0, b0 = coarse.pts_linears[0].weight.detach().double(), coarse.pts_linears[0].bias.detach().double()
    w5, b5 = coarse.pts_linears[5].weight.detach().double(), coarse.pts_linears[5].bias.detach().double()
    ref = torch.stack([b0 + lat.double() @ w0[:, 63:95].T, b5 + lat.double() @ w5[:, 63:95].T], 1)
    err = float((rb.double() - ref).abs().max())
    print(f"ray bias vs fp64: max abs err {err:.3e} (max |rb| {float(ref.abs().max()):.3f})")
    assert rb.shape == (300, 2, 256) and err <= 2e-6, err
    one = ops.tc_ray_bias(coarse, lat[:1], 0)
    assert one.shape == (1, 2, 256) and torch.equal(one[0], rb[0])


def test_per_ray_sums_latent_gradient_and_latent_columns_match_fp64():
    """nrn_field_backward_tc's per-ray sums of dY0 / dY5 vs an fp64 sum of the stashed (fp16, loss-scaled) dY images; d z and
    dW0 / dW5[:, 63:95] vs fp64 products of those sums.  S = 96: rays cross tile boundaries."""
    import ctypes as C
    from nonrigid_nerf_b200 import _lib, ops
    lib = _lib.load()
    coarse, _, _ = helpers.tc_models(R.SEED, DEV)
    n, s, out_ch = 40, 96, 5
    gen = torch.Generator().manual_seed(5)
    r = O.make_rays(7, n)
    rays = helpers.rays8(r, DEV)
    z = torch.sort(torch.rand(n, s, generator=gen), -1)[0].to(DEV) * 0.9 + 0.05
    lat = (torch.randn(n, 32, generator=gen) * 0.5).to(DEV)
    stash = torch.empty(lib.nrn_stash_bytes(n, s), dtype=torch.uint8, device=DEV)
    mask = torch.empty(lib.nrn_relu_mask_bytes(n, s), dtype=torch.uint8, device=DEV)
    ops.field_forward(rays, z, lat, ops.pack_nerf(coarse), None, out_ch, stash=stash, relu_mask=mask, tc_net=coarse)
    d_raw = (torch.randn(n, s, out_ch, generator=gen) * 1e-3).to(DEV)
    a = _lib.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = n, s, out_ch
    gstash = torch.empty(lib.nrn_grad_stash_bytes(n, s), dtype=torch.uint8, device=DEV)
    scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=DEV)
    grad = torch.empty(lib.nrn_nerf_tc_grad_floats(out_ch), dtype=torch.float32, device=DEV)
    a.d_raw, a.stash, a.relu_mask, a.grad_stash, a.wgrad_scratch = d_raw.data_ptr(), stash.data_ptr(), mask.data_ptr(), gstash.data_ptr(), scratch.data_ptr()
    a.nerf_packed, a.nerf_grad = ops.pack_nerf(coarse).data_ptr(), grad.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    t = _lib.NrnTcBwdArgs()
    ws = torch.empty(lib.nrn_tc_workspace_bytes(n) // 4, dtype=torch.float32, device=DEV)
    d_lat = torch.empty(n, 32, dtype=torch.float32, device=DEV)
    t.latents, t.latent_stride = lat.data_ptr(), 32
    t.w0, t.w5 = coarse.pts_linears[0].weight.data_ptr(), coarse.pts_linears[5].weight.data_ptr()
    t.d_latents, t.workspace = d_lat.data_ptr(), ws.data_ptr()
    _lib.check(lib.nrn_field_backward_tc(C.byref(a), C.byref(t)), "field_backward_tc")
    _lib.device_error_check()
    n_tiles = (n * s + 127) // 128
    scale = SL.loss_scale(float(d_raw[..., :4].abs().max()))
    ref = []
    for l in (0, 5):
        dy = SL.image(gstash, SL.GRAD_TILE, SL.GS_Y[l][0], 32, n_tiles)[:n * s].double() / scale
        ref.append(dy.view(n, s, 256).sum(1))
    ref = torch.stack(ref, 1)                                           # [n][2][256]
    sums = ws[:n * 512].view(n, 2, 256).double()
    e_s = R.rel(sums.cpu(), ref.cpu())
    print(f"per-ray sums vs fp64 of the stashed dY0 / dY5: rel L2 {e_s:.3e}")
    assert e_s <= 1e-6, e_s
    w0, w5 = coarse.pts_linears[0].weight.detach().double(), coarse.pts_linears[5].weight.detach().double()
    dz_ref = ref[:, 0] @ w0[:, 63:95] + ref[:, 1] @ w5[:, 63:95]
    e_z = R.rel(d_lat.double().cpu(), dz_ref.cpu())
    dw_ref = torch.stack([ref[:, 0].T @ lat.double(), ref[:, 1].T @ lat.double()])       # [2][256][32]
    flat = SL.split_flat(grad.cpu(), SL.nerf_param_shapes(out_ch, tc=True))
    e_w0 = R.rel(flat["w0"][:, 63:95].double(), dw_ref[0].cpu())
    e_w5 = R.rel(flat["w5"][:, 63:95].double(), dw_ref[1].cpu())
    print(f"d z vs fp64 {e_z:.3e}; dW0[:, 63:95] {e_w0:.3e}, dW5[:, 63:95] {e_w5:.3e}")
    assert e_z <= 1e-5 and e_w0 <= 1e-5 and e_w5 <= 1e-5, (e_z, e_w0, e_w5)
    # the embedding and h columns are WGRAD's, the same values the 63-input layout gets from the same stash
    assert float(flat["w5"][:, 95:].abs().sum()) > 0 and float(flat["b0"].abs().sum()) > 0


def _targs(**over):
    import types
    a = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=200000, offsets_loss_weight=0.0,
                              divergence_loss_weight=0.0, rigidity_loss_weight=0.0, ray_bending_latent_size=32)
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _run_wrapper(g, use_arena):
    from nonrigid_nerf_b200 import _lib, optim, parallel
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, _ = helpers.tc_models(seed, DEV)
    r = O.make_rays(seed, n)
    rnd = dict(O.make_randomness(seed, n, 64, 64))
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
    opt = optim.Adam(latents + list(coarse.parameters()) + list(fine.parameters()), lr=5e-4) if use_arena else None
    if opt is not None:
        opt.zero_grad()
        assert opt.grads_in_arena
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=None)
    loss = wrapper(_targs(), r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, _kwargs(coarse, fine, r, rnd, 1.0, 1.0),
                   r["target"].to(DEV), 50000, 0, {"imageid_to_timestepid": [int(v) for v in g["i2t"]]},
                   torch.from_numpy(g["pix"]).to(DEV))
    loss.mean().backward()
    _lib.device_error_check()
    if opt is not None:
        assert opt.grads_in_arena, "the backward must accumulate into the arena, not re-bind .grad"
    return loss.detach().cpu(), coarse, fine, latents


def test_training_wrapper_loss_and_gradients_match_golden_fresh_and_arena():
    g = _golden()
    results = {}
    for use_arena in (False, True):
        loss, coarse, fine, latents = _run_wrapper(g, use_arena)
        d, e_loss = float(np.abs(loss.numpy() - g["loss"]).max()), R.rel(loss.numpy(), g["loss"])
        print(f"[arena={use_arena}] per-ray loss vs executed reference: L-inf {d:.3e}, rel L2 {e_loss:.3e}")
        assert d <= 2e-3 and e_loss <= 2e-3, (d, e_loss)
        named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()]
        worst = 0.0
        for nm, t in named:
            if nm + ".val" not in g.files or t.grad is None:
                continue
            ours = t.grad.reshape(-1).cpu()[torch.from_numpy(g[nm + ".idx"])].double().numpy()
            err = R.rel(ours, g[nm + ".val"])
            nrm = abs(float(t.grad.norm()) - float(g[nm + ".norm"][0])) / (float(g[nm + ".norm"][0]) + 1e-30)
            worst = max(worst, err)
            assert err <= 1.2e-1 and nrm <= 1.2e-1, (nm, err, nrm)
        e_cols = []
        for nm, mod in (("coarse", coarse), ("fine", fine)):
            e_cols.append(R.rel(mod.pts_linears[0].weight.grad[:, 63:95].cpu().numpy(), g[nm + ".w0_latent_grad"]))
            e_cols.append(R.rel(mod.pts_linears[5].weight.grad[:, 63:95].cpu().numpy(), g[nm + ".w5_latent_grad"]))
        lg = torch.stack([l.grad for l in latents]).cpu()
        e_lat = R.rel(lg.numpy(), g["latent_grads"])
        print(f"[arena={use_arena}] worst sampled gradient error {worst:.3e}; latent columns of W0 / W5 {max(e_cols):.3e}; "
              f"latent table {e_lat:.3e}")
        assert max(e_cols) <= 1.2e-1 and e_lat <= 8e-2, (e_cols, e_lat)
        results[use_arena] = [p.grad.detach().clone() for nm, p in named if "views_linears" not in nm] + [lg]
        if use_arena:
            assert coarse.views_linears[0].weight.grad.abs().max() == 0
        else:
            assert coarse.views_linears[0].weight.grad is None
    for a, b in zip(results[False], results[True]):
        assert R.rel(b.cpu().numpy(), a.cpu().numpy()) <= 1e-5


def test_two_backward_passes_are_bit_identical():
    from nonrigid_nerf_b200 import autograd as ag, ops
    coarse, _, _ = helpers.tc_models(R.SEED, DEV)
    n, s = 50, 80
    gen = torch.Generator().manual_seed(9)
    rays = helpers.rays8(O.make_rays(11, n), DEV)
    z = (torch.sort(torch.rand(n, s, generator=gen), -1)[0] * 0.9 + 0.05).to(DEV)
    lat = (torch.randn(n, 32, generator=gen) * 0.5).to(DEV).requires_grad_(True)
    w = torch.randn(n, s, 5, generator=gen).to(DEV)
    grads = []
    for _ in range(2):
        coarse.zero_grad(set_to_none=True)
        lat.grad = None
        raw, _ = ag.field(coarse, rays, z, lat, False)
        (raw * w).sum().backward()
        grads.append([lat.grad.clone()] + [p.grad.clone() for p in ops.nerf_param_list(coarse)[0] + ops.nerf_param_list(coarse)[1]])
    assert float(grads[0][0].abs().sum()) > 0
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_cuda_graph_replay_matches_eager_training_step():
    """optim.Adam + GraphedStep: the 4th step replayed from the graph (3 warm-up steps, then capture) gives the loss the
    4th eager step gives, and the parameters move.  The latent table stays fixed so that no step uses atomics."""
    from nonrigid_nerf_b200 import optim, parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    g = _golden()
    seed, n = int(g["seed"]), int(g["n"])
    r = O.make_rays(seed, n)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    latents = [torch.from_numpy(row.copy()).to(DEV) for row in g["latent_table"]]
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), torch.from_numpy(g["pix"]).to(DEV)]
    i2t = {"imageid_to_timestepid": [int(v) for v in g["i2t"]]}
    losses = {}
    for mode in ("eager", "graph"):
        coarse, fine, _ = helpers.tc_models(seed, DEV)
        opt = optim.Adam(list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
        wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=None)
        kw = _kwargs(coarse, fine, r, rnd, 1.0, 1.0)
        w_before = coarse.pts_linears[0].weight.detach().clone()

        def step(rays_o, rays_d, target, pix):
            opt.zero_grad()
            loss = wrapper(_targs(), rays_o, rays_d, 100, kw, target, 50000, 0, i2t, pix)
            loss.mean().backward()
            opt.step()
            return loss.detach()

        if mode == "eager":
            for _ in range(4):
                out = step(*inputs)
        else:
            graphed = GraphedStep(step, inputs, warmup=3)
            out = graphed(*inputs)
        torch.cuda.synchronize()
        losses[mode] = out.clone().cpu()
        assert float((coarse.pts_linears[0].weight.detach() - w_before).abs().max()) > 0
    e = R.rel(losses["graph"].numpy(), losses["eager"].numpy())
    print(f"graph replay vs eager, 4th step per-ray loss: rel L2 {e:.3e}")
    assert e <= 1e-5, e
