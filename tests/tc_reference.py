"""fp32 CPU restatement of the time-conditioned baseline (run_nerf_helpers.py:206-209, 273-282; train.py:574-578) on top
of oracle/nrnerf_oracle.py: the per-ray latent z joins the positional encoding at layer 0 and at the skip layer, so
nerf_mlp's input is emb = [PE(63) | z(32)] and its skip concatenation [emb | h] is the reference's [PE | z | h].
Drives golden case L (tests/golden/make_golden_tc.py) and the GPU tests of the time-conditioned path."""
import numpy as np
import torch

import oracle.nrnerf_oracle as O

SEED = 1000


def make_params(seed: int):
    """Coarse and fine parameters of case L (W0 [256][95], W5 [256][351])."""
    return O.make_nerf_params(seed, 5, 30.0, input_ch=95), O.make_nerf_params(seed + 1, 5, 30.0, input_ch=95)


def query(npar, pts: torch.Tensor, latents: torch.Tensor) -> torch.Tensor:
    """pts [N,S,3], latents [N,32] -> raw [N,S,C]."""
    n, s, _ = pts.shape
    lat = latents[:, None, :].expand(n, s, latents.shape[-1]).reshape(n * s, -1)
    emb = torch.cat([O.positional_encoding(pts.reshape(-1, 3)), lat], -1)
    return O.nerf_mlp(npar, emb).reshape(n, s, -1)


def render_rays(cp, fp, rays_o, rays_d, near, far, latents, s_c=64, n_imp=64, perturb=False, raw_noise_std=0.0, rnd=None):
    """render_rays (train.py:792-980) with the time-conditioned coarse / fine NeRFs and no bender."""
    n, dev = rays_o.shape[0], rays_o.device
    near_t = torch.full((n, 1), float(near), device=dev)
    far_t = torch.full((n, 1), float(far), device=dev)
    z = O.stratified_z(near_t, far_t, s_c, rnd["t_rand"] if perturb else None)
    raw = query(cp, rays_o[:, None, :] + rays_d[:, None, :] * z[:, :, None], latents)
    noise_c = rnd["noise_c"] * raw_noise_std if raw_noise_std > 0 else None
    rgb0, _, acc0, _, w, _ = O.raw2outputs(raw, z, rays_d, noise_c)
    u = rnd["u"] if perturb else O.det_u(n, n_imp, dev)
    z_samples = O.sample_pdf(0.5 * (z[:, 1:] + z[:, :-1]), w[:, 1:-1], u).detach()
    z_f, _ = torch.sort(torch.cat([z, z_samples], -1), -1)
    raw = query(fp, rays_o[:, None, :] + rays_d[:, None, :] * z_f[:, :, None], latents)
    noise_f = rnd["noise_f"] * raw_noise_std if raw_noise_std > 0 else None
    rgb, _, acc, _, _, _ = O.raw2outputs(raw, z_f, rays_d, noise_f)
    return {"rgb_map": rgb, "acc_map": acc, "rgb0": rgb0, "acc0": acc0, "raw": raw}


def training_loss(g, cp, fp, latent_table: torch.Tensor):
    """Per-ray loss of training_wrapper_class.forward for case L (no regularisers): latent lookup by image id, training-mode
    render (perturb = 1, raw_noise_std = 1), fine + coarse image terms."""
    seed, n = int(g["seed"]), int(g["n"])
    r = O.make_rays(seed, n)
    return training_loss_rays(cp, fp, r, latent_table, g["i2t"], torch.from_numpy(g["pix"]), O.make_randomness(seed, n, 64, 64))


def training_loss_rays(cp, fp, rays, latent_table: torch.Tensor, imageid_to_timestepid, pixel_indices: torch.Tensor, rnd):
    """training_loss on given rays (rays_o, rays_d, near, far, target), injected random draws, (image, y, x) pixel indices
    and latent table, on their device."""
    i2t = torch.as_tensor(imageid_to_timestepid, device=pixel_indices.device)
    lat = latent_table[i2t[pixel_indices[:, 0]], :]
    ret = render_rays(cp, fp, rays["rays_o"], rays["rays_d"], rays["near"], rays["far"], lat, perturb=True, raw_noise_std=1.0,
                      rnd=rnd)
    return O.training_loss(ret, rays["target"])


def rel(a, b) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))
