"""The LPIPS workspace layout (csrc/lpips.cuh, lpips.cu: lpips_dims, lpips_mask_bytes, lpips_frame_bytes, lpips_chunk),
mirrored for tests that read every stage back from a workspace they own.  tests/test_lpips_layout_cpu.py pins it to
the library's sizes and to the header's constants.  Plain Python and torch; no kernel code.

Workspace: the mask [H][W] u8 (rounded up to 256 bytes), then one chunk of fc frames: per stage s = 0..7 the 2 fc
images [2 fc][h_s][w_s][C_s] fp16 (ground truth 0..fc-1, then renders), each stage one 256-byte aligned buffer; then
the distance partials [5][fc][max blocks] fp64 and right after them the saturation words [2 fc] u32.
"""
import torch

TAPS = 5
STAGES = 8
STAGE_CHANNELS = (8, 64, 64, 192, 192, 384, 256, 256)
TAP_STAGES = (1, 3, 5, 6, 7)
DIST_PIXELS = 256
CHUNK_BUDGET = 256 << 20
MAX_CHUNK = 4096
MIN_SIDE, MAX_SIDE = 31, 16384
# (cin_real, cin, cout, ks, stride, pad, split) of kLpipsConv
CONVS = ((3, 8, 64, 11, 4, 2, 1), (64, 64, 192, 5, 1, 2, 1), (192, 192, 384, 3, 1, 1, 2), (384, 384, 256, 3, 1, 1, 1),
         (256, 256, 256, 3, 1, 1, 1))
IN_STAGE = (0, 2, 4, 5, 6)   # the stage each convolution reads
SLAB_CHUNKS = 8


def a256(v):
    return (v + 255) // 256 * 256


def dims(h, w):
    """[(h_s, w_s)] of the 8 stages: input, conv1, pool1, conv2, pool2, conv3, conv4, conv5"""
    conv = lambda n, c: (n + 2 * c[5] - c[3]) // c[4] + 1
    pool = lambda n: (n - 3) // 2 + 1 if n >= 3 else 0
    c1 = (conv(h, CONVS[0]), conv(w, CONVS[0]))
    p1 = (pool(c1[0]), pool(c1[1]))
    c2 = (conv(p1[0], CONVS[1]), conv(p1[1], CONVS[1]))
    p2 = (pool(c2[0]), pool(c2[1]))
    return [(h, w), c1, p1, c2, p2, p2, p2, p2]


def px(h, w, s):
    hh, ww = dims(h, w)[s]
    return hh * ww


def dist_blocks(h, w, tap):
    return -(-px(h, w, TAP_STAGES[tap]) // DIST_PIXELS)


def max_blocks(h, w):
    return max(dist_blocks(h, w, k) for k in range(TAPS))


def image_bytes(h, w, s):
    return px(h, w, s) * STAGE_CHANNELS[s] * 2


def mask_bytes(h, w):
    return a256(h * w)


def frame_bytes(h, w):
    b = sum(a256(2 * image_bytes(h, w, s)) for s in range(STAGES))
    return b + a256(TAPS * max_blocks(h, w) * 8 + 2 * 4)


def default_chunk(f, h, w):
    return min(max(1, min(CHUNK_BUDGET // frame_bytes(h, w), MAX_CHUNK)), f)


def workspace_bytes(f, h, w):
    """nrn_lpips_workspace_bytes(f, h, w): 0 out of range"""
    if f < 0 or not (MIN_SIDE <= h <= MAX_SIDE and MIN_SIDE <= w <= MAX_SIDE):
        return 0
    return mask_bytes(h, w) + default_chunk(f, h, w) * frame_bytes(h, w)


def chunk(fc, h, w):
    """Byte offsets of a chunk of fc frames: {"act": [8 stage offsets], "partials", "sat", "end"}"""
    o = mask_bytes(h, w)
    act = []
    for s in range(STAGES):
        act.append(o)
        o += a256(2 * fc * image_bytes(h, w, s))
    partials = o
    sat = partials + TAPS * fc * max_blocks(h, w) * 8
    return {"act": act, "partials": partials, "sat": sat, "end": sat + 2 * fc * 4}


def stage(ws, fc, h, w, s):
    """Stage s of a chunk of fc frames from the workspace bytes ws (uint8 tensor) -> [2 fc, h_s, w_s, C_s] fp16"""
    hh, ww = dims(h, w)[s]
    off = chunk(fc, h, w)["act"][s]
    n = 2 * fc * image_bytes(h, w, s)
    return ws[off:off + n].view(torch.float16).view(2 * fc, hh, ww, STAGE_CHANNELS[s])


def stage_images(ws, fc, h, w, s, images):
    """Only the listed images of stage s (a list of ints) -> [len(images), h_s, w_s, C_s] fp16, without viewing the rest"""
    hh, ww = dims(h, w)[s]
    off, ib = chunk(fc, h, w)["act"][s], image_bytes(h, w, s)
    return torch.stack([ws[off + i * ib:off + (i + 1) * ib].view(torch.float16).view(hh, ww, STAGE_CHANNELS[s]) for i in images])


def partials(ws, fc, h, w):
    """[5, fc, max blocks] fp64"""
    off, mb = chunk(fc, h, w)["partials"], max_blocks(h, w)
    return ws[off:off + TAPS * fc * mb * 8].view(torch.float64).view(TAPS, fc, mb)


def sat_words(ws, fc, h, w):
    """[2 fc] int32 saturation words: bit l set when conv l + 1 clamped an output of the image"""
    off = chunk(fc, h, w)["sat"]
    return ws[off:off + 2 * fc * 4].view(torch.int32)


def mask(ws, h, w):
    return ws[:h * w].view(h, w)
