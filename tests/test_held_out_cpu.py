"""Held-out rays on the CPU: the argument checks of the held-out entry points (each rejected before any CUDA call), their
declarations, the Python-side refusals of a bad held_out mask, and its sharding over two gloo ranks.  No kernel is
launched here."""
import ctypes
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_deterministic_cpu import _bwd_args
from tests.test_div_abi_cpu import _fake, _full_args
from tests.test_host_cpu import _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HELD_OUT_SYMBOLS = ("nrn_field_backward_held_out", "nrn_field_backward_det_held_out", "nrn_divergence_backward_held_out")


def test_held_out_entry_points_are_declared_bound_and_exported():
    from nonrigid_nerf_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nrnerf_b200.h")).read()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in HELD_OUT_SYMBOLS:
        assert f"int {name}(" in header, name
        assert name in _lib.SYMBOLS, name
        assert hasattr(lib, name), name
    assert _lib.load().nrn_abi_version() == 4 == _lib.ABI_VERSION
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
    assert len(kinds) == 15 and _lib.HELD_OUT_KERNEL_KINDS == ("field_dgrad_held_out", "div_bwd_held_out")


def test_field_backward_held_out_validates_its_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()

    def bad(a, held, msg, rows=None, det=False):
        if det:
            rc = lib.nrn_field_backward_det_held_out(ctypes.byref(a) if a is not None else None, rows, held)
        else:
            rc = lib.nrn_field_backward_held_out(ctypes.byref(a) if a is not None else None, held)
        assert rc == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    for det in (False, True):
        who = b"nrn_field_backward_det_held_out" if det else b"nrn_field_backward_held_out"
        bad(None, p, b"null args", p, det)
        a = _bwd_args(p); a.bender_packed = None
        bad(a, p, b"needs a bender", p, det)
        a = _bwd_args(p); a.d_latents = None
        bad(a, p, b"d_latents", p, det)
        bad(_bwd_args(p), None, who + b": null held_out_rays", p, det)
        a = _bwd_args(p); a.n_samples = 0
        bad(a, p, b"bad sizes", p, det)
        a = _bwd_args(p); a.n_rays = -1
        bad(a, p, b"bad sizes", p, det)
        for name in ("d_raw", "stash", "grad_stash", "wgrad_scratch", "nerf_packed", "nerf_grad", "unmasked_offsets",
                     "rigidity_mask", "bender_grad", "relu_mask"):
            a = _bwd_args(p); setattr(a, name, None)
            bad(a, p, b"null", p, det)
        for name in ("nerf_packed", "stash", "grad_stash", "relu_mask"):
            a = _bwd_args(p); setattr(a, name, p.value + 4)
            bad(a, p, b"16-byte aligned", p, det)
        a = _bwd_args(p); a.out_ch = 6
        bad(a, p, b"out_ch=6", p, det)
        a = _bwd_args(p); a.n_rays = a.n_samples = 0x7fffffff
        bad(a, p, who + b": too many points", p, det)
    # the per-ray bytes need no alignment; the deterministic variant's latent_rows do
    bad(_bwd_args(p), ctypes.c_void_p(p.value + 1), b"latent_rows", None, True)
    bad(_bwd_args(p), ctypes.c_void_p(p.value + 1), b"latent_rows", ctypes.c_void_p(p.value + 4), True)


def test_divergence_backward_held_out_validates_its_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()

    def bad(a, held, msg):
        assert lib.nrn_divergence_backward_held_out(ctypes.byref(a) if a is not None else None, held) == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    bad(None, p, b"null args")
    bad(_full_args(p), None, b"nrn_divergence_backward_held_out: null held_out_rays")
    a = _full_args(p); a.n_samples = 0
    bad(a, p, b"bad sizes")
    a = _full_args(p); a.relu_mask = None
    bad(a, p, b"relu_mask")
    a = _full_args(p); a.bender_packed = ctypes.c_void_p(p.value + 4)
    bad(a, p, b"aligned")
    for name in ("adjoint_stash", "wgrad_scratch", "d_unmasked_offsets", "d_rigidity_mask", "bender_grad"):
        a = _full_args(p); setattr(a, name, None)
        bad(a, p, b"nrn_divergence_backward_held_out: null argument")


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.ray_bender = (None,)


def test_bad_held_out_masks_are_refused_before_any_launch():
    from nonrigid_nerf_b200 import autograd as ag
    n = 6
    ok = torch.zeros(n, dtype=torch.bool)
    assert ag.check_held_out(None, n, "cpu") is None
    assert ag.check_held_out(ok, n, "cpu").dtype == torch.uint8
    assert ag.check_held_out(torch.ones(n, dtype=torch.uint8), n, "cpu").dtype == torch.uint8
    for bad, msg in ((torch.zeros(n, dtype=torch.float32), "bool or uint8"),
                     (torch.zeros(n, dtype=torch.int64), "bool or uint8"),
                     (torch.zeros(n + 1, dtype=torch.bool), rf"shape \[{n}\]"),
                     (torch.zeros(n, 1, dtype=torch.bool), rf"shape \[{n}\]"),
                     ([0] * n, "must be a tensor"),
                     (torch.zeros(n, dtype=torch.bool, device="meta"), "device")):
        with pytest.raises(RuntimeError, match=msg):
            ag.check_held_out(bad, n, "cpu")


def test_wrapper_and_render_refuse_a_bad_mask_first():
    """training_wrapper_class.forward and render check held_out before touching anything else (here: CPU tensors, where
    any later step would fail differently)."""
    from nonrigid_nerf_b200 import parallel, train as T
    n = 4
    rays_o, rays_d, tgt = torch.zeros(n, 3), torch.ones(n, 3), torch.zeros(n, 3)
    w = parallel.training_wrapper_class(_Net(), [torch.zeros(32)], ray_bender=None)
    with pytest.raises(RuntimeError, match="held_out must be bool or uint8"):
        w(None, rays_o, rays_d, 0, {}, tgt, 0, 0, {}, None, held_out=torch.zeros(n))
    with pytest.raises(RuntimeError, match=r"held_out must have shape \[4\]"):
        w(None, rays_o, rays_d, 0, {}, tgt, 0, 0, {}, None, held_out=torch.zeros(n + 2, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="rays must be CUDA tensors"):   # render's own first refusal, mask or not
        T.render(rays_o, rays_d, ndc=False, held_out=torch.zeros(n, dtype=torch.bool))


# ---- world_size-2 gloo: RayShardedFunction hands each rank its rows of held_out -------------------------------------
class _Echo(torch.nn.Module):
    def forward(self, rays, held_out=None):
        return torch.cat([rays[:, :1], held_out.to(rays.dtype)[:, None]], -1)


def _worker(rank, world, port, n, out_path, dtype):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from nonrigid_nerf_b200 import parallel as P
    seen = {}

    class Spy(_Echo):
        def forward(self, rays, held_out=None):
            seen["held"] = held_out.clone()
            return super().forward(rays, held_out)

    g = torch.Generator().manual_seed(11 + rank)          # ranks hold different inputs; rank 0's are broadcast
    rays = torch.randn(n, 8, generator=g)
    held = (torch.rand(n, generator=g) < 0.3).to(dtype)
    out = P.RayShardedFunction(Spy())(rays, held_out=held)
    lo, hi = P.shard_bounds(n, world, rank)
    torch.save({"rank": rank, "seen": seen["held"], "lo": lo, "hi": hi, "out": out.detach()}, out_path + f".{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8])
def test_held_out_is_sharded_with_the_rays(tmp_path, dtype):
    n, world = 11, 2
    out = str(tmp_path / "r")
    mp.spawn(_worker, args=(world, _free_port(), n, out, dtype), nprocs=world, join=True)
    g = torch.Generator().manual_seed(11)
    rays0 = torch.randn(n, 8, generator=g)
    held0 = (torch.rand(n, generator=g) < 0.3).to(dtype)
    for r in range(world):
        got = torch.load(out + f".{r}")
        assert got["seen"].dtype == dtype and got["seen"].shape == (got["hi"] - got["lo"],)
        assert torch.equal(got["seen"], held0[got["lo"]:got["hi"]])                      # rank 0's mask, this rank's rows
        assert torch.equal(got["out"][:, 1], held0.float()) and torch.equal(got["out"][:, 0], rays0[:, 0])
