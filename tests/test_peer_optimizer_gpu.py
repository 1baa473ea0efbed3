"""The peer-memory gradient reduce + Adam and row gather (csrc/peer.cu) on ONE GPU, and the benchmark's graph-replayed
bending step against eager execution.

The peer protocol does not care whether a rank's window is another process's CUDA-IPC mapping or a second buffer on the
same device, so k ranks are emulated in one process with plain torch-owned windows laid out like peer.py's
([1024 B flags | 2 row slots | gradient arena], tests/stash_layout.peer_window_layout).  Before each call as rank `me`,
the other ranks' flags in window `me` are preset to the epoch the call is about to use (they have "arrived" and
"finished reading"), so no kernel ever waits.  Checked, bit for bit:
  * reduce + Adam: the arena of `me` and the `reduced` workspace hold the fp32 left fold ((+0 + g_0) + g_1) + ... in rank
    order; parameters and moments equal nrn_adam_step (adam.cu) run on that folded gradient, and lie within the fp64
    bounds of test_ray_kernels_parity_gpu.py::test_adam (see check_adam_fp64); every step count advances; the epoch advances across the
    u32 wrap; only ARRIVE[me] / DONE[me] of every window and the arena of `me` change; every `me` ends bit-identical;
  * row gather: the rank-order concatenation, published into the parity of the NEXT gather epoch, the other parity
    untouched, its epoch independent of the reduce's;
  * the Python reducer at world = 1 (a one-rank gloo group): gradients live in the window, opt.step() equals plain
    optim.Adam on the same arena;
  * the step bench.py times (bending model, device-scalar global_step, set_lr between replays, optionally the peer
    reducer and its gather inside the graph): CUDA-graph replays against eager steps.
`pytest -s` prints c_obs for every fp64 Adam check.
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import ray_reference as R
from tests import stash_layout as SL
from tests.parity import DEV, F64, Report, poison_f32

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C_ADAM_UPD, C_ADAM_MOM = 16, 8           # as test_ray_kernels_parity_gpu.py::test_adam
B1, B2, EPS = 0.9, 0.999, 1e-8
SIZES = (1, 255, 2047, 2048, 2049, 4097, 256 * 319)   # ragged 2048-element Adam blocks and ragged 256-thread rows
ARRIVE, DONE, GATHER = SL.PEER_ARRIVE * SL.PEER_MAX_RANKS, SL.PEER_DONE * SL.PEER_MAX_RANKS, SL.PEER_GATHER * SL.PEER_MAX_RANKS


def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L, L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def n_diff(a, b):
    return int((bits(a) != bits(b)).sum())


def i32(x):
    """u32 value -> the int32 a torch int32 tensor stores for it"""
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def u32(x):
    return int(x) & 0xFFFFFFFF


def F32(x):
    """the ABI takes fp32 betas, eps and lr: the reference uses those values"""
    return float(np.float32(x))


def half_ulp32(x):
    """0.5 ulp of fp32 values x (float64 tensor)"""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=-126) - 24)


# ----------------------------------------------------------------------------------------------------------------------
# emulated ranks
# ----------------------------------------------------------------------------------------------------------------------
class Windows:
    """k ranks' windows as plain device buffers, the context state int32[4] (three epochs, then the block counter) and
    the `reduced` workspace.  Flags and slots start as random bytes, so a stray write anywhere shows up."""

    def __init__(self, k, arena_floats, slot_floats, seed=0, random_fill=True):
        self.k, self.total, self.slot_floats = k, arena_floats, slot_floats
        self.slot_off, self.slot_bytes, self.arena_off, nbytes = SL.peer_window_layout(arena_floats, slot_floats)
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.win = [torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device=DEV, generator=g) if random_fill
                    else torch.zeros(nbytes, dtype=torch.uint8, device=DEV) for _ in range(k)]
        self.state = torch.zeros(4, dtype=torch.int32, device=DEV)
        self.reduced = poison_f32(max(arena_floats, 1))

    def flags(self, r, win=None):
        return (win or self.win)[r][:SL.PEER_FLAG_BYTES].view(torch.int32)

    def arena(self, r, win=None):
        return (win or self.win)[r][self.arena_off:self.arena_off + 4 * self.total].view(torch.float32)

    def slot_bytes_of(self, r, parity, win=None):
        o = self.slot_off + parity * self.slot_bytes
        return (win or self.win)[r][o:o + self.slot_bytes]

    def slot(self, r, parity, win=None):
        return self.slot_bytes_of(r, parity, win)[:4 * self.slot_floats].view(torch.float32)

    def epochs(self):
        return [u32(v) for v in self.state.tolist()]

    def ctx(self, me):
        L, _ = _lib()
        c = L.NrnPeerCtx()
        for r in range(self.k):
            c.window[r] = self.win[r].data_ptr()
        c.world, c.rank, c.arena_floats, c.slot_floats = self.k, me, self.total, self.slot_floats
        c.state, c.reduced = self.state.data_ptr(), self.reduced.data_ptr()
        return c

    def snapshot(self):
        return [w.clone() for w in self.win]

    def assert_windows(self, expect, what):
        for r in range(self.k):
            assert torch.equal(self.win[r], expect[r]), f"{what}: window {r}: {int((self.win[r] != expect[r]).sum())} bytes differ"


class AdamState:
    """Flat parameters / moments / per-tensor steps / block table / device lr of a set of tensors, like optim.Adam's."""

    def __init__(self, sizes, steps, seed, loaded=True):
        g = torch.Generator().manual_seed(seed)
        self.sizes = list(sizes)
        self.offs = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        self.total = int(self.offs[-1])
        self.P = torch.randn(self.total, generator=g).to(DEV)
        self.M = (torch.randn(self.total, generator=g) * 0.05).to(DEV) if loaded else torch.zeros(self.total, device=DEV)
        self.V = (torch.rand(self.total, generator=g) * 1e-3).to(DEV) if loaded else torch.zeros(self.total, device=DEV)
        self.steps = torch.tensor(steps, dtype=torch.int64, device=DEV)
        blocks = [(i, s, min(2048, n - s), int(o) + s) for i, (n, o) in enumerate(zip(self.sizes, self.offs)) for s in range(0, n, 2048)]
        self.blocks = torch.tensor(blocks, dtype=torch.int32, device=DEV)
        self.lr = torch.zeros((), dtype=torch.float32, device=DEV)

    def clone(self):
        c = object.__new__(AdamState)
        c.__dict__.update(self.__dict__)
        for k in ("P", "M", "V", "steps", "lr"):
            setattr(c, k, getattr(self, k).clone())
        return c

    def slices(self):
        return [slice(int(o), int(o) + n) for n, o in zip(self.sizes, self.offs)]

    def args(self, grads=None):
        """grads: a flat gradient tensor (its per-tensor views become the pointer table), or None (the peer path)"""
        L, _ = _lib()
        a = L.NrnAdamArgs()
        a.params, a.exp_avg, a.exp_avg_sq = self.P.data_ptr(), self.M.data_ptr(), self.V.data_ptr()
        if grads is not None:
            self._gp = torch.tensor([grads.data_ptr() + 4 * int(o) for o in self.offs[:-1]], dtype=torch.int64, device=DEV)
            a.grad_ptrs = self._gp.data_ptr()
        a.blocks, a.n_tensors, a.n_blocks = self.blocks.data_ptr(), len(self.sizes), int(self.blocks.shape[0])
        a.lr, a.step, a.beta1, a.beta2, a.eps = self.lr.data_ptr(), self.steps.data_ptr(), B1, B2, EPS
        a.stream = _stream()
        return a


def rank_grads(k, total, seed):
    """Every rank's gradients.  Per element (flat index mod 4):
      0: rank r holds (1, 2^-24, -1)[r % 3] times a power of two: the left fold's bits differ from a fold that starts at
         another rank, and from a tree sum;
      1: -0.0 on every rank (the fold starts at +0, so the sum is +0);
      2: subnormals;
      3: magnitudes 1e-9 .. 1e3, random signs."""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(total)
    scale = torch.ldexp(torch.ones(total, dtype=F64), torch.randint(-20, 20, (total,), generator=g))
    out = []
    for r in range(k):
        trip = ((1.0, 2.0 ** -24, -1.0)[r % 3] * scale).float()
        sub = (torch.randint(-2 ** 20, 2 ** 20, (total,), generator=g).to(F64) * 2.0 ** -149).float()
        wide = (10.0 ** (torch.rand(total, generator=g, dtype=F64) * 12 - 9)
                * torch.where(torch.rand(total, generator=g) < 0.5, -1.0, 1.0).to(F64)).float()
        x = torch.where(i % 4 == 0, trip, torch.where(i % 4 == 1, torch.full((total,), -0.0), torch.where(i % 4 == 2, sub, wide)))
        out.append(x.to(DEV))
    return out


def left_fold(grads):
    acc = torch.zeros_like(grads[0])       # +0
    for g in grads:
        acc = acc + g
    return acc


def check_adam_fp64(tag, before, after, fold, lr):
    """test_adam's bounds against the fp64 reference, fed with the folded fp32 gradient.  Two differences, both forced by
    the gradient patterns here rather than by the kernel:
      * the moments get an absolute floor of C_ADAM_MOM half-spacings of fp32's subnormal range (2^-150 each): a
        subnormal gradient gives a subnormal m, whose roundings are absolute, not relative;
      * the update is checked for the kernel's own new moments (read back from exp_avg / exp_avg_sq), the moments on their
        own.  With gradients up to 1e3 against a loaded m, m + (g - m)(1 - b1) cancels (|m_new| ~ M_m / 190 observed), so
        m_new's own rounding alone exceeds 16 ulp of |update| at a few elements of any fp32 evaluation."""
    floor_mom = C_ADAM_MOM * 2.0 ** -150
    for i, sl in enumerate(before.slices()):
        t = int(after.steps[i])
        rep = Report(f"{tag} size={before.sizes[i]} step={t} lr={lr:g}")
        _, _, m_new, M_m, v_new, M_v = R.adam_ref(before.P[sl], before.M[sl], before.V[sl], fold[sl], t, F32(lr), F32(B1),
                                                  F32(B2), F32(EPS))
        mk, vk = after.M[sl].to(F64), after.V[sl].to(F64)
        upd = -(F32(lr) / (1.0 - F32(B1) ** t)) * mk / (vk.sqrt() / (1.0 - F32(B2) ** t) ** 0.5 + F32(EPS))
        got = after.P[sl].to(F64) - before.P[sl].to(F64)
        rep.check("update", got, upd, upd.abs(), C_ADAM_UPD, floor=half_ulp32(after.P[sl].to(F64)))
        rep.check("exp_avg", after.M[sl], m_new, M_m, C_ADAM_MOM, floor=floor_mom)
        rep.check("exp_avg_sq", after.V[sl], v_new, M_v, C_ADAM_MOM, floor=floor_mom)


def reduce_call(W, me, st, grads, lr, fp64_tag=None):
    """One nrn_peer_reduce_adam as rank `me` with the other ranks emulated, and every check of that call."""
    L, lib = _lib()
    k, e = W.k, u32(W.state[0]) + 1
    for r in range(k):
        W.arena(r).copy_(grads[r])
    fl = W.flags(me)
    for r in range(k):
        if r != me:
            fl[ARRIVE + r] = i32(e)
            fl[DONE + r] = i32(e)
    st.lr.fill_(lr)
    fold = left_fold(grads)
    before, state0, win0 = st.clone(), W.state.clone(), W.snapshot()
    twin = st.clone()
    L.check(lib.nrn_peer_reduce_adam(C.byref(W.ctx(me)), C.byref(st.args())), "peer_reduce_adam")
    L.check(lib.nrn_adam_step(C.byref(twin.args(fold))), "adam_step")
    L.device_error_check()
    what = f"k={k} me={me} epoch={e:#x}"

    expect = win0
    for r in range(k):
        W.flags(r, expect)[ARRIVE + me] = i32(e)
        W.flags(r, expect)[DONE + me] = i32(e)
    W.arena(me, expect).copy_(fold)
    W.assert_windows(expect, what)        # own arena = fold; other arenas, slots and every other flag word untouched
    assert same_bits(W.reduced[:W.total], fold), f"{what}: reduced workspace: {n_diff(W.reduced[:W.total], fold)} differ"
    want_state = state0.clone()
    want_state[0], want_state[3] = i32(e), 0
    assert torch.equal(W.state, want_state), f"{what}: state {W.epochs()} (expected {[u32(v) for v in want_state.tolist()]})"
    assert torch.equal(st.steps, before.steps + 1), f"{what}: step counts"
    assert torch.equal(st.steps, twin.steps)
    for name in ("P", "M", "V"):
        a, b = getattr(st, name), getattr(twin, name)
        assert same_bits(a, b), f"{what}: {name} differs from nrn_adam_step in {n_diff(a, b)} of {a.numel()} elements"
    if lr == 0.0:
        assert same_bits(st.P, before.P), f"{what}: lr = 0 moved parameters"
    if fp64_tag is not None:
        check_adam_fp64(fp64_tag, before, st, fold, lr)


# steps the loaded state starts from: around 10^6 (double-precision bias correction) and a few small counts, where the
# bias correction is far from 1
LOADED_STEPS = [10 ** 6, 3, 999_999, 1 << 20, 10 ** 6 + 17, 40, 10 ** 6 - 1]
LRS_A = [5e-4, 0.0, 2e-3]


@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_peer_reduce_adam_emulated_ranks(k):
    """Three calls from a loaded state, the epoch preset to 0xFFFFFFFE (the calls use 0xFFFFFFFF, 0, 1), the lr changed
    between calls (the second is 0); run as every rank in turn, every rank must end bit-identical."""
    finals = []
    total = sum(SIZES)
    for me in range(k):
        W = Windows(k, total, 300, seed=k)
        W.state.copy_(torch.tensor([i32(0xFFFFFFFE), 12345, i32(0x80000001), 0], dtype=torch.int32))
        st = AdamState(SIZES, LOADED_STEPS, seed=1)
        per_call = []
        for call, lr in enumerate(LRS_A):
            reduce_call(W, me, st, rank_grads(k, total, seed=100 * k + call), lr,
                        fp64_tag=f"peer k={k} call={call}" if me == 0 else None)
            per_call.append(torch.cat([st.P, st.M, st.V]))
        assert W.epochs()[0] == 1
        finals.append(per_call)
    for me in range(1, k):
        for call in range(len(LRS_A)):
            assert same_bits(finals[me][call], finals[0][call]), f"rank {me} diverged from rank 0 after call {call}"


def test_peer_reduce_adam_one_rank_real_protocol():
    """k = 1 from a zero window, zero state and zero moments, nothing preset: the whole protocol runs (tick, wait on its
    own flag, reduce + Adam, DONE, finish) over 5 calls, bit-identical to nrn_adam_step from the first step on."""
    total = sum(SIZES)
    W = Windows(1, total, 256, random_fill=False)
    st = AdamState(SIZES, [0] * len(SIZES), seed=2, loaded=False)
    for call, lr in enumerate([1e-3, 5e-4, 0.0, 1e-2, 3e-4]):
        reduce_call(W, 0, st, rank_grads(1, total, seed=700 + call), lr, fp64_tag=f"peer k=1 fresh call={call}")
    assert W.epochs() == [5, 0, 0, 0]
    assert st.steps.tolist() == [5] * len(SIZES)


# ----------------------------------------------------------------------------------------------------------------------
# row gather
# ----------------------------------------------------------------------------------------------------------------------
GATHER_SLOT = 65537            # 262,148 bytes round up to 262,400: the arena sits 2 x 252 bytes further back
GATHER_SIZES = (2049, 5)


def gather_rows(W, me, rows):
    L, lib = _lib()
    return lib.nrn_peer_gather_rows(C.byref(W.ctx(me)), C.c_void_p(rows[me].data_ptr()), rows[me].numel(),
                                    C.c_void_p(W._out.data_ptr()), C.c_void_p(_stream()))


def gather_call(W, me, rows):
    """One nrn_peer_gather_rows as rank `me`: the other ranks' rows in slot[(epoch + 1) & 1] of their windows, 0xFF in the
    other parity, GATHER[r] of window `me` preset; every slot of window `me` starts as 0xFF."""
    L, _ = _lib()
    k, n = W.k, rows[0].numel()
    e = u32(W.state[2]) + 1
    par = e & 1
    for r in range(k):
        W.slot_bytes_of(r, 1 - par).fill_(0xFF)
        if r == me:
            W.slot_bytes_of(r, par).fill_(0xFF)
        else:
            W.slot(r, par)[:n].copy_(rows[r])
            W.flags(me)[GATHER + r] = i32(e)
    W._out = poison_f32(k * n)
    state0, win0 = W.state.clone(), W.snapshot()
    L.check(gather_rows(W, me, rows), "peer_gather_rows")
    L.device_error_check()
    what = f"gather k={k} me={me} n={n} epoch={e:#x}"
    want = torch.cat(rows)
    assert same_bits(W._out, want), f"{what}: out: {n_diff(W._out, want)} of {want.numel()} differ"
    expect = win0
    W.slot(me, par, expect)[:n].copy_(rows[me])
    for r in range(k):
        W.flags(r, expect)[GATHER + me] = i32(e)
    W.assert_windows(expect, what)        # own slot of this parity = local; the other parity and everything else untouched
    want_state = state0.clone()
    want_state[2] = i32(e)
    assert torch.equal(W.state, want_state), f"{what}: state {W.epochs()}"


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4099, GATHER_SLOT])
def test_peer_gather_rows_emulated_ranks(n):
    """k = 8 (at n >= 4097 the 8 n outputs exceed one pass of the 128 x 256 collect grid): 4 gathers from the gather epoch
    0xFFFFFFFE (parities 1, 0, 1, 0 across the wrap), each followed by a reduce + Adam call whose epoch runs separately."""
    k = 8
    total = sum(GATHER_SIZES)
    for me in range(k):
        W = Windows(k, total, GATHER_SLOT, seed=n)
        W.state.copy_(torch.tensor([7, 0, i32(0xFFFFFFFE), 0], dtype=torch.int32))
        st = AdamState(GATHER_SIZES, [10, 10], seed=3)
        g = torch.Generator(device=DEV).manual_seed(1000 * n + me)
        for call in range(4):
            rows = [torch.randn(n, device=DEV, generator=g) for _ in range(k)]
            rows[call % k][0] = -0.0
            gather_call(W, me, rows)
            reduce_call(W, me, st, rank_grads(k, total, seed=call), 1e-3)
        assert W.epochs() == [11, 0, 2, 0]


def test_peer_gather_rows_rejects_more_than_a_slot():
    L, lib = _lib()
    k, n = 3, 1000
    W = Windows(k, 16, n - 1, seed=5)
    rows = [torch.randn(n, device=DEV) for _ in range(k)]
    W._out = poison_f32(k * n)
    state0, win0 = W.state.clone(), W.snapshot()
    assert gather_rows(W, 1, rows) != 0
    assert b"exceed the slot" in lib.nrn_last_error()
    L.device_error_check()
    W.assert_windows(win0, "rejected gather")
    assert torch.equal(W.state, state0) and bool((bits(W._out) == -1).all())


# ----------------------------------------------------------------------------------------------------------------------
# the Python reducer at world = 1, and the benchmark's step under CUDA-graph replay
# ----------------------------------------------------------------------------------------------------------------------
def _golden():
    return np.load(os.path.join(GOLD, "caseH_training_wrapper.npz"))


def _build(g, n_iters=None):
    """caseH models, latents, rays and injected random draws (as tests/test_multigpu_gpu.py builds them), optim.Adam"""
    import types
    from nonrigid_nerf_b200 import optim
    seed, n = int(g["seed"]), int(g["n"])
    torch.manual_seed(seed)
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    rnd["e"] = torch.from_numpy(g["e"]).to(DEV).view(n, 64, 3)
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
    params = latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=5e-4)
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=int(n_iters or g["N_iters"]),
                                  offsets_loss_weight=float(g["offsets_w"]), divergence_loss_weight=float(g["divergence_w"]),
                                  rigidity_loss_weight=float(g["rigidity_w"]), ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64, "network_fn": coarse,
          "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0, "ndc": False, "lindisp": False,
          "near": r["near"], "far": r["far"], "randomness": rnd}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), torch.from_numpy(g["pix"]).to(DEV)]
    extras = {"imageid_to_timestepid": [int(v) for v in g["i2t"]]}
    return coarse, fine, bender, latents, opt, targs, kw, inputs, extras


@contextlib.contextmanager
def _world_one(tmp_path):
    """A one-rank gloo process group over a FileStore (no TCP)."""
    import torch.distributed as dist
    dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def _peer_reducer(opt):
    from nonrigid_nerf_b200 import parallel, peer
    try:
        red = peer.PeerArenaReducer(opt)
    except RuntimeError as exc:
        if "cudaIpcGetMemHandle" in str(exc):
            pytest.skip(f"CUDA IPC is not available here: {exc}")
        raise
    parallel.attach_optimizer(opt, red)
    return red


def test_peer_reducer_world_one_matches_plain_adam(tmp_path):
    """PeerArenaReducer + attach_optimizer at world = 1: every p.grad is a view of the window's arena and the backward
    kernels write there; opt.step() equals plain optim.Adam stepped on a copy of that arena (copying it sidesteps the
    latent gradient's fp32-atomic order); the arena then holds the reduced gradient (+0 + g); gather_rows is the identity."""
    from nonrigid_nerf_b200 import _lib as L, optim, parallel
    coarse, fine, bender, latents, opt, targs, kw, inputs, extras = _build(_golden())
    wrapper = parallel.get_parallelized_training_function(coarse, latents, fine_model=fine, ray_bender=bender)
    params = opt.param_groups[0]["params"]
    twin = optim.Adam([p.detach().clone() for p in params], lr=5e-4)
    with _world_one(tmp_path):
        red = _peer_reducer(opt)
        try:
            arena = opt.gradient_arena()
            arena_off = SL.peer_window_layout(opt._total, red.slot_floats)[2]
            assert arena.data_ptr() == red._own + arena_off
            opt.zero_grad()
            losses = wrapper(targs, *inputs[:2], 100, kw, inputs[2], int(_golden()["global_step"]), 0, extras, inputs[3])
            losses.mean().backward()
            for p, o in zip(params, opt._offs):
                assert p.grad is not None and p.grad.data_ptr() == arena.data_ptr() + 4 * int(o), "a gradient lives outside the window"
            for name, p in (("fine L3", fine.pts_linears[3].weight), ("coarse L0", coarse.pts_linears[0].weight),
                            ("bender", bender.network[0].weight), ("latent", latents[int(_golden()["i2t"][int(inputs[3][0, 0])])])):
                assert float(p.grad.abs().max()) > 0, f"{name}: no gradient reached the window"
            g_arena = arena.clone()
            opt.step()
            L.device_error_check()
            twin.gradient_arena().copy_(g_arena)
            twin.step()
            for name, a, b in (("params", opt._flat, twin._flat), ("exp_avg", opt._m, twin._m), ("exp_avg_sq", opt._v, twin._v)):
                assert same_bits(a, b), f"{name}: {n_diff(a, b)} of {a.numel()} differ from plain optim.Adam"
            assert torch.equal(opt._step, twin._step)
            assert same_bits(arena, torch.zeros_like(g_arena) + g_arena), "the arena does not hold the reduced gradient"
            got = red.gather_rows(losses)
            assert same_bits(got, losses.detach())
        finally:
            red.close()


N_ITERS_D = 8                              # 0.01^(1 - step / 8): the regularisers' weights change strongly per step
LRS_D = [5e-4, 5e-4, 5e-4, 2e-3, 0.0, 1e-3]   # steps 1..6; the graph's 3 warm-up steps run at the first value
LOSS_REL_D = 1e-5


def _bending_run(mode, reducer):
    """Six steps of bench.py's local_step on the caseH bending model (divergence, offsets and rigidity terms on).
    mode: "eager"; "graph" (3 warm-up steps inside GraphedStep, then 3 replays); "graph_after_forward" (3 eager steps,
    a no-grad validation render that leaves every packed-weight cache valid, then capture without warm-up and 3 replays).
    After a warm-up step the caches are stale anyway (its opt.step() invalidated them), so only the second capture shows
    that GraphedStep puts the weight packing into the graph even when the caches are valid (ops.FORCE_PACK).
    Returns per step (losses, gathered losses, parameters before, parameters after) for steps 4..6 (all 6 eagerly)."""
    from nonrigid_nerf_b200 import parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    coarse, fine, bender, latents, opt, targs, kw, inputs, extras = _build(_golden(), n_iters=N_ITERS_D)
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    red = _peer_reducer(opt) if reducer == "peer" else None
    global_step = torch.zeros((), dtype=torch.float32, device=DEV)
    n = inputs[0].shape[0]

    def local_step(rays_o, rays_d, target, pix):
        opt.zero_grad()
        losses = wrapper(targs, rays_o, rays_d, 100, kw, target, global_step, 0, extras, pix)
        (losses.sum() / n).backward()
        opt.step()
        gathered = red.gather_rows(losses) if red is not None else losses.detach()
        global_step.add_(1.0)
        return losses.detach(), gathered

    out = []
    try:
        if mode == "eager":
            first = 0
            run = local_step
        else:
            first = 3
            if mode == "graph":
                opt.set_lr(LRS_D[0])
                graphed = GraphedStep(local_step, inputs, warmup=3)
            else:
                for i in range(3):
                    opt.set_lr(LRS_D[i])
                    local_step(*inputs)
                with torch.no_grad():       # a validation render: packs the current weights of all three networks
                    from nonrigid_nerf_b200 import train as T
                    i2t = torch.tensor(extras["imageid_to_timestepid"], device=DEV)
                    lat = torch.stack(latents)[i2t[inputs[3][:, 0]]]
                    T.render(inputs[0], inputs[1], chunk=targs.chunk, additional_pixel_information={"ray_bending_latents": lat}, **kw)
                graphed = GraphedStep(local_step, inputs, warmup=0)
            run = graphed
        assert float(global_step) == first
        for i in range(first, 6):
            opt.set_lr(LRS_D[i])
            p0 = opt._flat.clone()
            losses, gathered = run(*inputs)
            torch.cuda.synchronize()
            out.append((losses.clone(), gathered.clone(), p0, opt._flat.clone()))
        from nonrigid_nerf_b200 import _lib as L
        L.device_error_check()
        assert float(global_step) == 6
    finally:
        if red is not None:
            red.close()
    return out[-3:] if mode == "eager" else out, [o[0] for o in out]


def _rel(a, b):
    return float((a.to(F64) - b.to(F64)).norm() / b.to(F64).norm())


@pytest.mark.parametrize("reducer,mode", [("adam", "graph"), ("peer", "graph"), ("adam", "graph_after_forward")])
def test_graphed_bending_step_matches_eager(tmp_path, reducer, mode):
    """bench.py's step -- zero_grad, training_wrapper_class with a device-scalar global_step, (sum / n).backward(),
    opt.step(), [gather_rows], global_step.add_(1) -- replayed from a CUDA graph with set_lr between replays (one replay
    at lr = 0) against eager steps 4..6 from the same initial state: per-ray losses within a relative L2 of LOSS_REL_D,
    the lr = 0 step leaves the parameters bit-unchanged, and the gathered losses equal the losses bit for bit.
    Two eager runs of this step differ by the latent gradient's and the divergence loss's fp32 atomics; their spread over
    the 6 steps is printed and held to the same bound."""
    ctx = _world_one(tmp_path) if reducer == "peer" else contextlib.nullcontext()
    with ctx:
        eager, eager_all = _bending_run("eager", reducer)
        _, eager2_all = _bending_run("eager", reducer)
        graph, _ = _bending_run(mode, reducer)
    spread = max(_rel(a, b) for a, b in zip(eager2_all, eager_all))
    print(f"[{reducer} {mode}] eager vs eager over 6 steps: max rel L2 {spread:.3e}")
    assert spread <= LOSS_REL_D, spread
    for j, ((le, ge, pe0, pe1), (lg, gg, pg0, pg1)) in enumerate(zip(eager, graph)):
        step = 4 + j
        d = _rel(lg, le)
        print(f"[{reducer} {mode}] step {step} lr {LRS_D[step - 1]:g}: graph replay vs eager per-ray loss rel L2 {d:.3e}")
        assert d <= LOSS_REL_D, (step, d)
        assert same_bits(gg, lg) and same_bits(ge, le), f"step {step}: gathered losses differ from the losses"
        if LRS_D[step - 1] == 0.0:
            assert same_bits(pg1, pg0), f"step {step}: the lr = 0 replay moved {n_diff(pg1, pg0)} parameters"
            assert same_bits(pe1, pe0), f"step {step}: the lr = 0 eager step moved {n_diff(pe1, pe0)} parameters"
        else:
            assert not same_bits(pg1, pg0), f"step {step}: the replay did not move the parameters"
