"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's differentiable (train / guidance) render path.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module; the product (ssdnerf_b200/)
never does.  Parity unpinned by reference tests (the reference ships none); pinned instead by (i) a finite-difference
check of the autograd gradient and (ii) the identity "torch autograd of the K7 forward == K8's analytic backward"
checked against the C restatement of K8 (tests/test_oracle_cpu.py).

Restates, per scene:
  lib/models/decoders/base_volume_renderer.py:59-77   train branch: march_rays_train -> point_decode -> composite
  lib/ops/raymarching/src/raymarching.cu:503-581      K7 forward (T *= 1 - alpha; stop once T < T_thresh, crossing sample included)
  lib/ops/raymarching/src/raymarching.cu:606-687      K8 backward (the crossing sample receives NO gradient: `break` precedes the writes)
  lib/models/autodecoders/base_nerf.py:276-296        BaseNeRF.loss: MSE(image + bg (1 - ws), target) * w * 3 * scale + RegLoss
  lib/models/diffusions/gaussian_diffusion.py:180-293 pred_x_0 with guidance (grad w.r.t. x_0), p_sample_langevin, p_sample_ddim
"""
import math

import numpy as np
import torch

import oracle as orc
from oracle import render_port as rp


def _as_dtype(params, dtype):
    return {k: v.to(dtype) for k, v in params.items()}


def render_train_scene(params, code_single, rays_o, rays_d, bitfield, noises=None, grid_size=64, bound=1.0, min_near=0.2,
                       max_steps=256, dt_gamma=0.0, T_thresh=1e-4, dtype=torch.float64, trunc_exp=True, return_samples=False):
    """One scene. code_single (3,C,h,w) torch (may require grad); rays (N,3) float32 numpy; bitfield uint8 numpy.
    Returns weights_sum (N,), depth (N,), image (N,3) as torch tensors connected to `code_single`.
    trunc_exp: density activation as in `render_port.point_decode` (the reference's TruncExp by default).
    return_samples: also return a dict of the marched samples -- `xyzs`, `dirs` (M,3) float32 numpy, `grad_mask` (M,) bool numpy of
    the samples K8 writes a gradient for (composited and not the one at which T drops below T_thresh) and `counts` (N,) int64
    numpy of the samples each ray composites (K7's count, the crossing sample included)."""
    rays_o = np.ascontiguousarray(rays_o, np.float32)
    rays_d = np.ascontiguousarray(rays_d, np.float32)
    n = rays_o.shape[0]
    aabb = np.array([-bound, -bound, -bound, bound, bound, bound], np.float32)
    nears, fars = orc.near_far_from_aabb(rays_o, rays_d, aabb, min_near)
    xyzs, dirs, deltas, rays = orc.march_rays_train(rays_o, rays_d, bound, bitfield, 1, grid_size, nears, fars, dt_gamma=dt_gamma,
                                                    max_steps=max_steps, noises=noises)
    counts = rays[:, 2].astype(np.int64)
    offsets = rays[:, 1].astype(np.int64)
    assert np.array_equal(rays[:, 0], np.arange(n))
    m = int(counts.sum())
    if m == 0:
        z = code_single.sum() * 0
        res = z + torch.zeros(n, dtype=dtype), z + torch.zeros(n, dtype=dtype), z + torch.zeros(n, 3, dtype=dtype)
        if return_samples:
            res = res + (dict(xyzs=xyzs[:0], dirs=dirs[:0], grad_mask=np.zeros(0, bool), counts=np.zeros(n, np.int64)),)
        return res
    p = _as_dtype(params, dtype)
    sig, rgb = rp.point_decode(p, torch.from_numpy(xyzs[:m]).to(dtype), torch.from_numpy(dirs[:m]), code_single.to(dtype),
                               trunc_exp=trunc_exp)
    smax = int(counts.max())
    s_idx = torch.arange(smax)[None, :]
    valid = s_idx < torch.from_numpy(counts)[:, None]                                   # (N,S)
    idx = (torch.from_numpy(offsets)[:, None] + s_idx).clamp(max=m - 1)
    dt = torch.from_numpy(deltas[:m, 0]).to(dtype)[idx]
    tt = torch.from_numpy(deltas[:m, 1]).to(dtype)[idx]
    sg, cl = sig[idx], rgb[idx]                                                         # (N,S), (N,S,3)
    with torch.no_grad():
        a0 = (1 - torch.exp(-sg * dt)) * valid
        T_after0 = torch.cumprod(1 - a0, dim=1)
        prev = torch.cat([torch.ones(n, 1, dtype=dtype), T_after0[:, :-1]], dim=1)
        included = valid & (prev >= T_thresh)                                           # K7/K8: not yet broken out
        crossing = included & (T_after0 < T_thresh)                                     # sample at which both kernels break
    sg = torch.where(crossing, sg.detach(), sg)
    cl = torch.where(crossing[..., None], cl.detach(), cl)
    alpha = (1 - torch.exp(-sg * dt)) * included
    T_before = torch.cat([torch.ones(n, 1, dtype=dtype), torch.cumprod(1 - alpha, dim=1)[:, :-1]], dim=1)
    w = alpha * T_before
    res = w.sum(1), (w * tt).sum(1), (w[..., None] * cl).sum(1)
    if return_samples:
        grad_mask = np.zeros(m, bool)
        grad_mask[idx[included & ~crossing].numpy()] = True
        res = res + (dict(xyzs=xyzs[:m], dirs=dirs[:m], grad_mask=grad_mask, counts=included.sum(1).numpy().astype(np.int64)),)
    return res


def render_loss(params, code, rays_o, rays_d, targets, bitfields, noises=None, dt_gamma=None, bg_color=1.0, pixel_weight=1.0,
                loss_coef=None, scale_num_ray=1.0, reg_weight=None, dtype=torch.float64, **cfg):
    """BaseNeRF.loss (base_nerf.py:276-296) with MSELoss(mean) and RegLoss(power=2). code (B,3,C,h,w) torch;
    rays (B,N,3) / targets (B,N,3) numpy; returns (loss, out_rgbs (B,N,3))."""
    B = code.shape[0]
    outs = []
    for b in range(B):
        ws, _, img = render_train_scene(params, code[b], rays_o[b], rays_d[b], bitfields[b], None if noises is None else noises[b],
                                        dt_gamma=0.0 if dt_gamma is None else float(dt_gamma[b]), dtype=dtype, **cfg)
        outs.append(img + bg_color * (1 - ws[:, None]))
    out = torch.stack(outs)
    scale = 1 - math.exp(-loss_coef * scale_num_ray) if loss_coef is not None else 1
    loss = torch.mean((out - torch.as_tensor(np.asarray(targets)).to(dtype)) ** 2) * pixel_weight * (scale * 3)
    if reg_weight is not None:
        loss = loss + (code.to(dtype).abs() ** 2).mean() * reg_weight
    return loss, out


def render_loss_grad(params, code, *args, **kwargs):
    """d loss / d code through the whole restated chain (torch autograd, float64 by default)."""
    code = code.detach().clone().requires_grad_(True)
    loss, out = render_loss(params, code, *args, **kwargs)
    grad, = torch.autograd.grad(loss, code)
    return loss.detach(), grad, out.detach()


def guided_ddim_sample(denoise_fn, noise, dv, grad_guide_fn, num_timesteps=50, T=1000, clip_range=(-2, 2), clip_denoised=True,
                       guidance_gain=1.0, snr_weight_power=0.5, langevin_steps=0, langevin_delta=0.1, langevin_t_range=(0, 1000),
                       langevin_noises=None):
    """gaussian_diffusion.py:295-331 with pred_x_0's `grad_through_unet=False` guidance (:213-227) and the langevin
    correction steps (:242-262, :318-324).  denoise_fn(x_t, t[B]) -> v;  grad_guide_fn(x_0) -> d loss / d x_0.
    `langevin_noises`: iterator of noise tensors consumed in call order (the reference draws torch.randn)."""
    from oracle.unet_port import ddim_timesteps
    lang = iter(langevin_noises) if langevin_noises is not None else None

    def pred_x_0(x_t, t):
        sa, s1 = float(dv['sqrt_alphas_bar'][t]), float(dv['sqrt_one_minus_alphas_bar'][t])
        v = denoise_fn(x_t, torch.full((x_t.size(0),), t, dtype=torch.long))
        x0 = sa * x_t - s1 * v
        if grad_guide_fn is not None:
            if clip_denoised:
                x0 = x0.clamp(*clip_range)
            grad = grad_guide_fn(x0)
            x0 = x0 - grad * ((s1 ** (2 - snr_weight_power * 2)) * (sa ** (snr_weight_power * 2 - 1)) * guidance_gain)
        if clip_denoised:
            x0 = x0.clamp(*clip_range)
        return x0

    x_t = noise
    ts = [int(t) for t in ddim_timesteps(T, num_timesteps)]
    for step, t in enumerate(ts):
        t_prev = ts[step + 1] if step + 1 < len(ts) else -1
        ab_prev = dv['alphas_bar'][t_prev] if t_prev >= 0 else dv['alphas_bar_prev'][0]
        x0 = pred_x_0(x_t, t)
        eps = (x_t - float(dv['sqrt_alphas_bar'][t]) * x0) / float(dv['sqrt_one_minus_alphas_bar'][t])
        x_t = float(np.sqrt(ab_prev)) * x0 + float(np.sqrt(1 - ab_prev)) * eps
        if langevin_steps > 0 and langevin_t_range[0] < t_prev < langevin_t_range[1]:
            for _ in range(langevin_steps):
                sigma = float(dv['sqrt_one_minus_alphas_bar'][t_prev])
                x0 = pred_x_0(x_t, t_prev)
                eps = (x_t - float(dv['sqrt_alphas_bar'][t_prev]) * x0) / sigma
                nz = next(lang) if lang is not None else torch.randn_like(x_t)
                x_t = x_t - 0.5 * langevin_delta * sigma * eps + math.sqrt(langevin_delta) * sigma * nz
    return x_t
