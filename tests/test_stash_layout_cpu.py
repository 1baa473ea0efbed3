"""The stash, mask and gradient layouts that tests/stash_layout.py mirrors, pinned to the library's own sizes, and a round
trip of the documented ReLU mask bit layout.  No kernel is launched here."""
import math
import os
import re

import pytest
import torch

from tests import stash_layout as SL


def _contiguous(images, tile_bytes, unit):
    o = 0
    for off, n in images:
        assert off == o, (off, o)
        o += n * unit
    assert o == tile_bytes


def test_image_offsets_tile_the_library_buffers():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    _contiguous(SL.STASH_IMAGES, SL.STASH_TILE, SL.CHUNK)
    _contiguous(SL.GRAD_IMAGES, SL.GRAD_TILE, SL.CHUNK)
    o = 0
    for off, ncols in SL.MASK_IMAGES:
        assert off == o
        o += SL.TILE_M * (32 if ncols > 128 else 16)
    assert o == SL.MASK_TILE
    _contiguous([SL.T_E, SL.T_1, SL.T_2, SL.T_3, SL.T_4], SL.TAN_TILE, SL.CHUNK)
    _contiguous([SL.A_4, SL.A_3, SL.A_2, SL.A_1, SL.A_0], SL.ADJ_TILE, SL.CHUNK)
    # the compact divergence stashes are the bender sections of the field stashes, in the same order
    assert SL.TAN_TILE == SL.STASH_TILE - SL.ST_BIN[0] and SL.ADJ_TILE == SL.GRAD_TILE - SL.GS_YB4[0]
    # the field stashes and masks hold an even number of tiles, the divergence stashes exactly the point tiles
    for n, s in ((1, 7), (2, 64), (3, 100), (11, 100), (1023, 64), (1024, 128)):
        tiles = -(-n * s // SL.TILE_M)
        even = tiles + (tiles & 1)
        assert lib.nrn_stash_bytes(n, s) == even * SL.STASH_TILE
        assert lib.nrn_grad_stash_bytes(n, s) == even * SL.GRAD_TILE
        assert lib.nrn_relu_mask_bytes(n, s) == even * SL.MASK_TILE
        assert lib.nrn_div_stash_bytes(n, s) == tiles * SL.TAN_TILE
        assert lib.nrn_div_grad_stash_bytes(n, s) == tiles * SL.ADJ_TILE


def test_view_stash_images_tile_the_library_buffers():
    """The view stash [Dir | F | Hv], the view gradient stash [dYv | dF] and the Hv mask, against the library's sizes (an
    even tile count, as the trunk's stashes), and the views gradient layout against nrn_nerf_views_grad_floats."""
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    _contiguous([SL.VS_DIR, SL.VS_F, SL.VS_HV], SL.V_STASH_TILE, SL.CHUNK)
    _contiguous([SL.VG_YV, SL.VG_F], SL.V_GRAD_TILE, SL.CHUNK)
    assert SL.VS_DIR[1] * 8 == 32 and SL.VS_F[1] * 8 == 256 and SL.VS_HV[1] * 8 == 128
    assert SL.VG_YV[1] * 8 == 128 and SL.VG_F[1] * 8 == 256 and SL.HV_MASK_TILE == SL.TILE_M * 16
    for n, s in ((1, 7), (2, 64), (3, 100), (11, 100), (1023, 64), (1024, 128), (22528, 128)):
        tiles = -(-n * s // SL.TILE_M)
        even = tiles + (tiles & 1)
        assert lib.nrn_views_stash_bytes(n, s) == even * SL.V_STASH_TILE
        assert lib.nrn_views_grad_stash_bytes(n, s) == even * SL.V_GRAD_TILE
        assert lib.nrn_hv_mask_bytes(n, s) == even * SL.HV_MASK_TILE
    shapes = SL.views_param_shapes()
    assert sum(math.prod(s) for _, s in shapes[:16]) == SL.TRUNK_FLOATS == lib.nrn_nerf_grad_floats(4) - 4 * 257
    assert sum(math.prod(s) for _, s in shapes) == lib.nrn_nerf_views_grad_floats() == 595844


@pytest.mark.parametrize("out_ch", [4, 5])
def test_gradient_parameter_maps_match_the_library(out_ch):
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert sum(math.prod(s) for _, s in SL.nerf_param_shapes(out_ch)) == lib.nrn_nerf_grad_floats(out_ch)
    assert sum(math.prod(s) for _, s in SL.nerf_param_shapes(out_ch, tc=True)) == lib.nrn_nerf_tc_grad_floats(out_ch)
    assert sum(math.prod(s) for _, s in SL.bender_param_shapes()) == lib.nrn_bender_grad_floats()


def test_peer_window_layout_matches_the_library():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert SL.PEER_FLAG_BYTES >= 4 * 3 * SL.PEER_MAX_RANKS
    for arena, slot in ((0, 0), (1, 1), (63, 64), (64, 65), (1_143_357, 1 << 16), (1_143_357, 65537), (2049, 8192)):
        slot_off, slot_bytes, arena_off, nbytes = SL.peer_window_layout(arena, slot)
        assert lib.nrn_peer_window_bytes(arena, slot) == nbytes, (arena, slot)
        assert slot_bytes % 256 == 0 and slot_bytes >= 4 * slot and arena_off % 256 == 0
        assert nbytes - arena_off >= 4 * arena
    assert SL.peer_window_layout(0, 65537)[1] == 262400     # 65537 floats round up: the arena moves by 2 x 252 bytes


def _encode_reference(bits):
    """The documented layout written out element by element (independent of stash_layout's vectorised code)."""
    rows, ncols = bits.shape
    kh = 2 if ncols > 128 else 1
    words = [[0] * (4 * kh) for _ in range(rows)]
    for r in range(rows):
        for c in range(ncols):
            if bits[r, c]:
                j, q = c // 8, (c % 8) // 2
                h, k = j // 16, j % 16
                words[r][q * kh + h] |= 1 << (k + 16 * (c % 2))
    out = bytearray()
    for r in range(rows):
        for w in words[r]:
            out += w.to_bytes(4, "little")
    return torch.frombuffer(out, dtype=torch.uint8).reshape(rows // SL.TILE_M, -1)


@pytest.mark.parametrize("ncols", [256, 96, 64])
def test_relu_mask_round_trip(ncols):
    g = torch.Generator().manual_seed(ncols)
    bits = torch.rand(2 * SL.TILE_M, ncols, generator=g) > 0.5
    ref = _encode_reference(bits)
    enc = SL.encode_relu_bits(bits)
    assert torch.equal(enc, ref)
    kh = 2 if ncols > 128 else 1
    assert enc.shape == (2, SL.TILE_M * 16 * kh)
    # decode from a mask buffer: the image sits at its offset inside each tile
    off = 8 * SL.MASK_H_BYTES if ncols < 128 else 3 * SL.MASK_H_BYTES
    buf = torch.zeros(2 * SL.MASK_TILE, dtype=torch.uint8)
    buf.view(2, SL.MASK_TILE)[:, off:off + enc.shape[1]] = enc
    assert torch.equal(SL.relu_bits(buf, off, ncols, 2), bits)
    # a single bit lands at the documented byte and bit: column 8 (16 h + k) + 2 q + 1 of row r
    one = torch.zeros(SL.TILE_M, ncols, dtype=torch.bool)
    r, c = 37, ncols - 5
    one[r, c] = True
    j, q = c // 8, (c % 8) // 2
    word = int.from_bytes(bytes(SL.encode_relu_bits(one)[0, r * 16 * kh + q * 4 * kh + 4 * (j // 16):][:4].tolist()), "little")
    assert word == 1 << (j % 16 + 16 * (c % 2))


def test_loss_scale_matches_the_kernels_rule():
    assert SL.loss_scale(0.0) == 1.0 and SL.loss_scale(float("inf")) == 1.0 and SL.loss_scale(float("nan")) == 1.0
    assert SL.loss_scale(3.1e38) == 1.0
    for amax in (1.0, 0.75, 1023.9, 1024.0, 3e-15, 2.5e10, 1e-30, 1e30):
        s = SL.loss_scale(amax)
        assert s == 2.0 ** round(math.log2(s))
        if 2.0 ** -60 <= s <= 2.0 ** 60 and 1e-17 < amax < 1e17:
            assert 512.0 <= amax * s < 1024.0, (amax, s)
    assert SL.loss_scale(1e-30) == 2.0 ** 60 and SL.loss_scale(1e30) == 2.0 ** -60


def test_boundary_tiles_hold_the_32_bit_limits_of_the_library_buffers():
    """The tiles tests/test_scale_gpu.py samples: per-tile sizes from the library, and the tile that holds byte 2^31 /
    2^32 of each buffer (the first byte a 32-bit signed / unsigned offset cannot address) with its neighbours."""
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    for (n, s), name, nbytes, expect in (
            ((8192, 128), "stash", lib.nrn_stash_bytes, [3381, 3382, 3383, 6764, 6765, 6766]),
            ((8192, 128), "grad stash", lib.nrn_grad_stash_bytes, [3471, 3472, 3473, 6943, 6944, 6945]),
            ((8192, 64), "stash", lib.nrn_stash_bytes, [3381, 3382, 3383]),
            ((53248, 128), "masks", lib.nrn_relu_mask_bytes, [52427, 52428, 52429]),
            ((53248, 128), "tangent", lib.nrn_div_stash_bytes, [22794, 22795, 22796, 45589, 45590, 45591]),
            ((53248, 128), "adjoint", lib.nrn_div_grad_stash_bytes, [23830, 23831, 23832, 47661, 47662, 47663])):
        T = -(-n * s // SL.TILE_M)
        n_buf = T + (T & 1) if name in ("stash", "grad stash", "masks") else T
        total = nbytes(n, s)
        tb = total // n_buf
        assert tb * n_buf == total, name
        got = SL.boundary_tiles(tb, T)
        assert got == [t for t in expect if t < T], (n, s, name, got)
        for lim in (2 ** 31, 2 ** 32):
            if lim < T * tb:
                t = lim // tb
                assert t in got and t * tb <= lim < (t + 1) * tb


@pytest.mark.parametrize("max_ctas", [132, 114, 66, 16])
def test_replicated_wgrad_plan_follows_the_job_cost_table_fits_the_scratch_and_covers_every_tile_once(max_ctas):
    """wgrad_plan / split_ranges restate launch_wgrad's plan: its per-job costs are the kJobCost table of wgrad.cu, its
    CTAs fit the device and the scratch partials (nrn_wgrad_scratch_bytes), and every job's splits own each tile exactly
    once.  The greedy rule itself is a copy: nothing the library exposes pins it."""
    from nonrigid_nerf_b200 import _lib
    from tests import stage_reference as SR
    lib = _lib.load()
    parts = lib.nrn_wgrad_scratch_bytes() // (4 * SR.WG_SCRATCH_FLOATS)
    assert parts * 4 * SR.WG_SCRATCH_FLOATS == lib.nrn_wgrad_scratch_bytes()
    src = open(os.path.join(os.path.dirname(_lib.__file__), "csrc", "wgrad.cu")).read()
    table = re.search(r"kJobCost\[16\]\s*=\s*\{([^}]*)\}", src).group(1)
    assert [sum(int(t) for t in x.split("+")) for x in table.split(",")] == SR._JOB_COST
    assert SR._JOB_COST[:12] == [46, 48, 48, 48, 48, 48, 48, 48, 32, 32, 54, 42]
    for T in (1, 9, 1024, 4096, 8192, 53248):
        for kw in (dict(has_bender=True), dict(has_bender=False), dict(compact=True)):
            plan = SR.wgrad_plan(T, max_ctas, **kw)
            halves = SR.wgrad_halves(**kw)
            used = sum(plan[j] * halves[j] for j in plan)
            assert used <= max(max_ctas, sum(halves.values())) and used <= parts, (T, kw, plan)
            for j, n_split in plan.items():
                ranges = SR.split_ranges(T, n_split)
                assert ranges[0][0] == 0 and ranges[-1][1] == T and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
                assert all(e > s for s, e in ranges) and len(ranges) <= n_split


@pytest.mark.parametrize("max_ctas", [132, 114, 66, 16])
def test_replicated_views_wgrad_plan_follows_the_job_cost_table_fits_the_scratch_and_covers_every_tile_once(max_ctas):
    """The same for launch_wgrad_views: its 14 jobs (the trunk's 0-9, then feature_linear 12, views_linears.0's feature
    columns 13, rgb_linear 14 and views_linears.0's direction columns 15) with their kJobCost costs; feature_linear
    takes two CTAs per split like a NeRF layer."""
    from nonrigid_nerf_b200 import _lib
    from tests import stage_reference as SR
    lib = _lib.load()
    parts = lib.nrn_wgrad_scratch_bytes() // (4 * SR.WG_SCRATCH_FLOATS)
    src = open(os.path.join(os.path.dirname(_lib.__file__), "csrc", "wgrad.cu")).read()
    table = re.search(r"kJobCost\[16\]\s*=\s*\{([^}]*)\}", src).group(1)
    assert [sum(int(t) for t in x.split("+")) for x in table.split(",")] == SR._JOB_COST
    assert [SR._JOB_COST[j] for j in (*range(10), 12, 13, 14, 15)] == [46, 48, 48, 48, 48, 48, 48, 48, 32, 32, 48, 48, 24, 20]
    halves = SR.wgrad_halves(views=True)
    assert list(halves) == [*range(10), 12, 13, 14, 15]
    assert [j for j, h in halves.items() if h == 2] == [*range(1, 10), 12]
    for T in (1, 9, 1024, 4096, 8192, 22528, 40960):
        plan = SR.wgrad_plan(T, max_ctas, views=True)
        used = sum(plan[j] * halves[j] for j in plan)
        assert used <= max(max_ctas, sum(halves.values())) and used <= parts, (T, plan)
        for j, n_split in plan.items():
            ranges = SR.split_ranges(T, n_split)
            assert ranges[0][0] == 0 and ranges[-1][1] == T and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
            assert all(e > s for s, e in ranges) and len(ranges) <= n_split
