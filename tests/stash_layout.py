"""Decoders of the buffers the fused kernels write, for tests that check each stage on its own.

The layouts are mirrored from csrc/nrn_common.cuh (forward stash kSt*, gradient stash kGs*, ReLU masks kMk*) and
csrc/div.cu (tangent stash kT*, adjoint stash kA*); tests/test_stash_layout_cpu.py pins them to the library's sizes.
Plain torch, CPU or CUDA tensors; no kernel code.
"""
import math

import torch

TILE_M = 128                 # points per tile
CHUNK = TILE_M * 16          # one 8-column fp16 chunk of a tile image
H_BYTES = 32 * CHUNK         # 256-column image
E_BYTES = 8 * CHUNK          # 64-column image

# forward (activation) stash, per tile: (offset, chunks)
ST_E = (0, 8)
ST_H = [(E_BYTES + l * H_BYTES, 32) for l in range(8)]          # H1..H8
ST_BIN = (E_BYTES + 8 * H_BYTES, 6)
ST_HB1 = (ST_BIN[0] + 6 * CHUNK, 12)
ST_HB2 = (ST_HB1[0] + 12 * CHUNK, 12)
ST_HB3 = (ST_HB2[0] + 12 * CHUNK, 8)
ST_HB4 = (ST_HB3[0] + 8 * CHUNK, 8)
STASH_TILE = ST_HB4[0] + 8 * CHUNK
STASH_IMAGES = [ST_E, *ST_H, ST_BIN, ST_HB1, ST_HB2, ST_HB3, ST_HB4]

# gradient stash, per tile
GS_RAW = (0, 2)
GS_Y = [(2 * CHUNK + l * H_BYTES, 32) for l in range(8)]        # dY0..dY7
GS_YB4 = (2 * CHUNK + 8 * H_BYTES, 2)
GS_YB3 = (GS_YB4[0] + 2 * CHUNK, 8)
GS_YB2 = (GS_YB3[0] + 8 * CHUNK, 10)                            # 64 + rigidity pre-activation (column 64) + pad
GS_YB1 = (GS_YB2[0] + 10 * CHUNK, 12)
GS_YB0 = (GS_YB1[0] + 12 * CHUNK, 12)
GRAD_TILE = GS_YB0[0] + 12 * CHUNK
GRAD_IMAGES = [GS_RAW, *GS_Y, GS_YB4, GS_YB3, GS_YB2, GS_YB1, GS_YB0]

# ReLU masks, per tile: (offset, columns)
MASK_H_BYTES, MASK_B_BYTES = TILE_M * 32, TILE_M * 16
MK_H = [(l * MASK_H_BYTES, 256) for l in range(8)]              # H1..H8
MK_HB1 = (8 * MASK_H_BYTES, 96)
MK_HB2 = (MK_HB1[0] + MASK_B_BYTES, 96)
MK_HB3 = (MK_HB2[0] + MASK_B_BYTES, 64)
MK_HB4 = (MK_HB3[0] + MASK_B_BYTES, 64)
MASK_TILE = MK_HB4[0] + MASK_B_BYTES
MASK_IMAGES = [*MK_H, MK_HB1, MK_HB2, MK_HB3, MK_HB4]

# view-dependent head (nrn_common.cuh kVs* / kVg* / kMkHv): view stash [Dir 27 + 5 zero | F | Hv], view gradient stash
# [dYv | dF] and the Hv mask, per tile
VS_DIR, VS_F, VS_HV = (0, 4), (4 * CHUNK, 32), (36 * CHUNK, 16)
V_STASH_TILE = VS_HV[0] + 16 * CHUNK
VG_YV, VG_F = (0, 16), (16 * CHUNK, 32)
V_GRAD_TILE = VG_F[0] + 32 * CHUNK
HV_MASK_TILE = TILE_M * 16                                      # 128 columns, one 16-byte row
TRUNK_FLOATS = 493056                                           # W0 b0 .. W7 b7 of nrn_nerf_views_grad_floats
HEAD_SHAPES = [("views_linears.0.weight", (128, 283)), ("views_linears.0.bias", (128,)), ("feature_linear.weight", (256, 256)),
               ("feature_linear.bias", (256,)), ("alpha_linear.weight", (1, 256)), ("alpha_linear.bias", (1,)),
               ("rgb_linear.weight", (3, 128)), ("rgb_linear.bias", (3,))]

# divergence regulariser: tangent stash [e | t1 s1 | t2 s2 | t3 | t4] and adjoint stash, per tile
T_E, T_1, T_2, T_3, T_4 = (0, 6), (6 * CHUNK, 12), (18 * CHUNK, 12), (30 * CHUNK, 8), (38 * CHUNK, 8)
TAN_TILE = 46 * CHUNK
A_4, A_3, A_2, A_1, A_0 = (0, 2), (2 * CHUNK, 8), (10 * CHUNK, 10), (20 * CHUNK, 12), (32 * CHUNK, 12)
ADJ_TILE = 44 * CHUNK


def tile_slices(buf, tile_bytes, off, nbytes, n_tiles, tiles):
    """[tiles, nbytes] at byte `off` of every tile, or of the listed tiles only (a long tensor on buf's device)."""
    t = buf[:n_tiles * tile_bytes].view(n_tiles, tile_bytes)
    if tiles is not None:
        t = t.index_select(0, tiles)
    return t[:, off:off + nbytes]


def image(buf, tile_bytes, off, chunks, n_tiles, tiles=None):
    """Chunk-major tile images [tile][chunk][128 rows][8] fp16 at byte `off` of every tile -> [n_tiles * 128, 8 * chunks];
    with `tiles` only those tiles, in that order -> [len(tiles) * 128, 8 * chunks]."""
    t = tile_slices(buf, tile_bytes, off, chunks * CHUNK, n_tiles, tiles)
    n = t.shape[0]
    t = t.contiguous().view(torch.float16).view(n, chunks, TILE_M, 8)
    return t.permute(0, 2, 1, 3).reshape(n * TILE_M, chunks * 8)


def boundary_tiles(tile_bytes, n_tiles, limits=(2 ** 31, 2 ** 32)):
    """The tiles of a buffer of n_tiles x tile_bytes whose byte range holds byte `limit` (the first byte a 32-bit signed /
    unsigned offset cannot address), and their neighbours, for every limit the buffer reaches; sorted."""
    out = set()
    for lim in limits:
        t = lim // tile_bytes
        if t < n_tiles:
            out.update(x for x in (t - 1, t, t + 1) if 0 <= x < n_tiles)
    return sorted(out)


def _mask_geometry(ncols):
    kh = 2 if ncols > 128 else 1
    c = torch.arange(ncols)
    j, q, odd = c // 8, (c % 8) // 2, c % 2
    word = q * kh + j // 16            # word of the row: byte q * 4 kH + 4 h
    bit = j % 16 + 16 * odd
    return kh, word, bit


def relu_bits(buf, off, ncols, n_tiles, tile_bytes=MASK_TILE, tiles=None):
    """ReluMask image (field_mma.cuh) at byte `off` of every tile -> bool [n_tiles * 128, ncols].  Row r holds one 32-bit
    word per (q, h) at byte r * 16 kH + q * 4 kH + 4 h; bit k is column 8 (16 h + k) + 2 q, bit 16 + k that column + 1;
    kH = 2 for 256 columns, else 1.  With `tiles` only those tiles, as image() does."""
    kh, word, bit = _mask_geometry(ncols)
    t = tile_slices(buf, tile_bytes, off, TILE_M * 16 * kh, n_tiles, tiles)
    w = t.contiguous().view(torch.int32).reshape(t.shape[0] * TILE_M, 4 * kh).long() & 0xFFFFFFFF
    return ((w[:, word.to(w.device)] >> bit.to(w.device)) & 1).bool()


def encode_relu_bits(bits):
    """Inverse of relu_bits for one image: bool [n_tiles * 128, ncols] -> uint8 [n_tiles, 128 * 16 kH]; unused bits 0."""
    rows, ncols = bits.shape
    kh, word, bit = _mask_geometry(ncols)
    w = torch.zeros(rows, 4 * kh, dtype=torch.int64, device=bits.device)
    v = bits.long() << bit.to(bits.device)
    w.index_add_(1, word.to(bits.device), v)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)
    return w.view(torch.uint8).reshape(rows // TILE_M, TILE_M * 16 * kh)


def loss_scale(amax):
    """The power-of-two loss scale of field_bwd.cu / wgrad.cu / div.cu: 2^clip(10 - e, -60, 60) with amax = m 2^e,
    m in [0.5, 1), so that amax * scale lies in [512, 1024); 1 when amax is 0, not finite or >= 3e38."""
    amax = float(amax)
    if not (amax > 0.0 and amax < 3.0e38):
        return 1.0
    _, e = math.frexp(amax)
    return 2.0 ** min(max(10 - e, -60), 60)


# Flat parameter maps of the weight-gradient buffers (wgrad.cu, wgrad_reduce_kernel): (name, shape) in order
def nerf_param_shapes(out_ch, tc=False):
    """tc: the time-conditioned layout (nrn_nerf_tc_grad_floats), W0 [256][63 + 32] and W5 [256][63 + 32 + 256]."""
    in_ch = 63 + (32 if tc else 0)
    shapes = [("w0", (256, in_ch)), ("b0", (256,))]
    for l in range(1, 8):
        shapes += [(f"w{l}", (256, in_ch + 256 if l == 5 else 256)), (f"b{l}", (256,))]
    return shapes + [("w_out", (out_ch, 256)), ("b_out", (out_ch,))]


def views_param_shapes():
    """nrn_nerf_views_grad_floats: the trunk W0 b0 .. W7 b7 (no output layer), then the head block in module order."""
    return nerf_param_shapes(4)[:-2] + HEAD_SHAPES


def bender_param_shapes():
    shapes = [("net_w0", (64, 35)), ("net_b0", (64,)), ("net_w1", (64, 64)), ("net_b1", (64,)), ("net_w2", (64, 64)),
              ("net_b2", (64,)), ("net_w3", (64, 64)), ("net_b3", (64,)), ("net_w4", (3, 64))]
    return shapes + [("rig_w0", (32, 3)), ("rig_b0", (32,)), ("rig_w1", (32, 32)), ("rig_b1", (32,)), ("rig_w2", (1, 32)),
                     ("rig_b2", (1,))]


# Peer-memory window (c_abi.cu fill_peer, peer.py): [flags: ARRIVE / DONE / GATHER x 8 u32, padded | 2 row slots | arena]
PEER_FLAG_BYTES = 1024
PEER_MAX_RANKS = 8
PEER_ARRIVE, PEER_DONE, PEER_GATHER = 0, 1, 2


def peer_window_layout(arena_floats, slot_floats):
    """(slot_off, slot_bytes, arena_off, window_bytes); slots and arena each rounded up to 256 bytes."""
    slot_bytes = (4 * slot_floats + 255) // 256 * 256
    arena_off = PEER_FLAG_BYTES + 2 * slot_bytes
    return PEER_FLAG_BYTES, slot_bytes, arena_off, arena_off + (4 * arena_floats + 255) // 256 * 256


def split_flat(flat, shapes):
    out, o = {}, 0
    for name, shape in shapes:
        n = math.prod(shape)
        out[name] = flat[o:o + n].view(shape)
        o += n
    assert o == flat.numel(), (o, flat.numel())
    return out
