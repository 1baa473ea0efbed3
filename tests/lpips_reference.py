"""fp64 restatement of LPIPS v0.1 with the AlexNet backbone (lpips.LPIPS(net='alex') in eval mode, as
free_viewpoint_rendering.py:788-849 calls it), built from torch.nn.functional on the CPU, plus seeded weights and frames
for the tests.

Per frame pair gt, gen [H, W, 3] in [0, 1]: zero the masked pixels of both, t = 2x - 1, s = (t - shift) / scale, the
AlexNet features (conv + bias + ReLU; conv1 11x11 stride 4 pad 2, max-pool 3/2, conv2 5x5 pad 2, max-pool 3/2, conv3-5
3x3 pad 1), whose five ReLU outputs are the taps; per tap the mean over pixels of sum_c w[c] (g_c / (|g| + 1e-10) -
r_c / (|r| + 1e-10))^2; LPIPS is the sum of the five tap scores.
"""
import numpy as np
import torch
import torch.nn.functional as F

CONVS = (("net.slice1.0", 64, 3, 11, 4, 2), ("net.slice2.3", 192, 64, 5, 1, 2), ("net.slice3.6", 384, 192, 3, 1, 1),
         ("net.slice4.8", 256, 384, 3, 1, 1), ("net.slice5.10", 256, 256, 3, 1, 1))
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
EPS = 1e-10


def random_state_dict(seed: int, lin_scale: float = 1.0) -> dict:
    """An lpips.LPIPS(net='alex') state dict with the AlexNet convolutions at PyTorch's default Conv2d initialisation and
    non-negative tap weights uniform in [0, lin_scale), including the scaling layer and the duplicate lins.* keys."""
    g = torch.Generator().manual_seed(seed)
    sd = {"scaling_layer.shift": torch.tensor(SHIFT).reshape(1, 3, 1, 1), "scaling_layer.scale": torch.tensor(SCALE).reshape(1, 3, 1, 1)}
    torch.manual_seed(seed)
    for key, cout, cin, k, _, _ in CONVS:
        conv = torch.nn.Conv2d(cin, cout, k)   # kaiming_uniform(a=sqrt(5)) weight, uniform(+-1/sqrt(fan_in)) bias
        sd[key + ".weight"], sd[key + ".bias"] = conv.weight.detach().clone(), conv.bias.detach().clone()
    for k, (_, cout, _, _, _, _) in enumerate(CONVS):
        w = torch.rand((1, cout, 1, 1), generator=g) * lin_scale
        sd[f"lin{k}.model.1.weight"] = w
        sd[f"lins.{k}.model.1.weight"] = w.clone()
    return sd


def he_state_dict(seed: int, gain: float) -> dict:
    """random_state_dict(seed) with every convolution replaced by He-normal weights (std sqrt(2 / fan_in), which keeps the
    activations' second moment from layer to layer through ReLU) and biases uniform in +-0.1, both times `gain` per
    layer, so that activations grow or shrink by about gain per layer: an activation scale set by the weights, as
    trained weights set it."""
    sd = random_state_dict(seed)
    g = torch.Generator().manual_seed(1000 + seed)
    for key, cout, cin, k, _, _ in CONVS:
        sd[key + ".weight"] = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5 * gain
        sd[key + ".bias"] = (torch.rand((cout,), generator=g) * 0.2 - 0.1) * gain
    return sd


def taps(x: torch.Tensor, sd: dict) -> list:
    """The five ReLU outputs of the AlexNet features of x [N, 3, H, W] (already scaled), in fp64."""
    out = []
    h = x.double()
    for i, (key, _, _, _, stride, pad) in enumerate(CONVS):
        if i in (1, 2):
            h = F.max_pool2d(h, kernel_size=3, stride=2)
        h = F.relu(F.conv2d(h, sd[key + ".weight"].double(), sd[key + ".bias"].double(), stride=stride, padding=pad))
        out.append(h)
    return out


def scaled(img: torch.Tensor, sd: dict) -> torch.Tensor:
    """[N, H, W, 3] in [0, 1] -> (2x - 1 - shift) / scale as [N, 3, H, W] fp64"""
    shift = sd.get("scaling_layer.shift", torch.tensor(SHIFT).reshape(1, 3, 1, 1)).double().reshape(1, 3, 1, 1)
    scale = sd.get("scaling_layer.scale", torch.tensor(SCALE).reshape(1, 3, 1, 1)).double().reshape(1, 3, 1, 1)
    t = 2 * torch.as_tensor(img).double().permute(0, 3, 1, 2) - 1
    return (t - shift) / scale


def mask_from(gt0) -> np.ndarray:
    """the reference's mask: pixels of the first ground-truth frame whose channels sum to 0 (in fp32, as numpy does)"""
    return np.asarray(gt0, dtype=np.float32).sum(axis=-1) == 0


def lpips(gt, gen, sd: dict, mask=None):
    """(lpips [F], per-tap scores [F, 5]) in fp64 for frames gt, gen [F, H, W, 3]; mask [H, W] bool (True = zeroed)
    defaults to mask_from(gt[0])."""
    gt = torch.as_tensor(np.asarray(gt)).double().clone()
    gen = torch.as_tensor(np.asarray(gen)).double().clone()
    m = torch.as_tensor(mask_from(gt[0].numpy()) if mask is None else np.asarray(mask) != 0)
    gt[:, m] = 0
    gen[:, m] = 0
    per = []
    for i in range(gt.shape[0]):   # frame by frame: the batch does not enter the score
        fa, fb = taps(scaled(gt[i:i + 1], sd), sd), taps(scaled(gen[i:i + 1], sd), sd)
        row = []
        for k, (a, b) in enumerate(zip(fa, fb)):
            na = a / (torch.sqrt((a * a).sum(dim=1, keepdim=True)) + EPS)
            nb = b / (torch.sqrt((b * b).sum(dim=1, keepdim=True)) + EPS)
            w = sd[f"lin{k}.model.1.weight"].double().reshape(1, -1, 1, 1)
            row.append(float((w * (na - nb) ** 2).sum(dim=1).mean()))
        per.append(row)
    per = np.array(per, dtype=np.float64).reshape(-1, 5)
    return per.sum(axis=1), per


def smooth_field(rng, h: int, w: int, octaves: int = 4) -> np.ndarray:
    """[h, w, 3] in [0, 1]: a sum of random low-frequency cosines per channel"""
    y, x = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    img = np.zeros((h, w, 3))
    for c in range(3):
        for o in range(octaves):
            fy, fx = rng.uniform(0.5, 3) * 2 ** o, rng.uniform(0.5, 3) * 2 ** o
            img[..., c] += rng.uniform(0.2, 1) / 2 ** o * np.cos(2 * np.pi * (fy * y + fx * x) + rng.uniform(0, 2 * np.pi))
    img -= img.min()
    return img / max(img.max(), 1e-12)


def frames(seed: int, n: int, h: int, w: int, perturb=(0.0, 0.01, 0.03, 0.1, 0.3)):
    """(gt, gen) [n, h, w, 3] fp32: smooth fields plus noise; frame i's render is its ground truth with noise of size
    perturb[i % len(perturb)] added and clipped, or (every sixth frame) an unrelated image"""
    rng = np.random.default_rng(seed)
    gt = np.empty((n, h, w, 3), dtype=np.float32)
    gen = np.empty_like(gt)
    for i in range(n):
        base = 0.8 * smooth_field(rng, h, w) + 0.2 * rng.random((h, w, 3))
        gt[i] = base
        if i % 6 == 5:
            gen[i] = 0.8 * smooth_field(rng, h, w) + 0.2 * rng.random((h, w, 3))
        else:
            s = perturb[i % len(perturb)]
            gen[i] = np.clip(base + s * (0.5 * rng.standard_normal((h, w, 3)) + smooth_field(rng, h, w) - 0.5), 0, 1)
    return gt, gen
