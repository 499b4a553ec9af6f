"""CHECKER (tests only): the train-branch renderer composed op by op -- this library's per-op kernels, which are bit-exact with the
reference's own (tests/test_ref_gpu.py): near/far K1, march_rays_train K6, composite_rays_train K7/K8 -- around a plain PyTorch
decode (grid_sample + Linear, autograd) of the shipped-config decoder.  Its density activation is the library's trunc_exp, pinned to the
reference's TruncExp, so the comparison also holds where the density gradient is floored (logits below ln 1e-6).  It is the A/B partner
of the fused differentiable renderer (csrc/render_train.cu); the product has no such composition (a trainable decoder raises)."""
import torch
import torch.nn.functional as F

from ssdnerf_b200.activation import trunc_exp
from ssdnerf_b200.raymarching import batch_composite_rays_train, batch_near_far_from_aabb, march_rays_train
from ssdnerf_b200.shencoder import sh_encode


def torch_point_decode(params, xyz, dirs, code_single, sat=0.001):
    """one scene: xyz, dirs [M,3], code [3,C,h,w] -> sigma [M], rgb [M,3] (feature index = c*3 + plane)"""
    grid = torch.stack([xyz[:, :2], xyz[:, ::2], xyz[:, 1:]], dim=0).unsqueeze(1)                  # [3,1,M,2]
    feat = F.grid_sample(code_single, grid, mode='bilinear', padding_mode='border', align_corners=False).squeeze(-2)
    feat = feat.permute(2, 1, 0).reshape(xyz.shape[0], -1)
    base = F.linear(feat, params['base_net.0.weight'], params['base_net.0.bias'])
    sigma = trunc_exp(F.linear(F.silu(base), params['density_net.0.weight'], params['density_net.0.bias'])).squeeze(-1)
    h = F.silu(base + F.linear(sh_encode(dirs, 4, False), params['dir_net.0.weight'], params['dir_net.0.bias']))
    rgb = torch.sigmoid(F.linear(h, params['color_net.0.weight'], params['color_net.0.bias']))
    return sigma, rgb * (1 + 2 * sat) - sat


def per_op_train_render(params, rays_o, rays_d, code, bitfield, dt_gamma, noises, T_thresh=1e-4, bound=1.0, min_near=0.2, max_steps=256,
                        grid_size=64):
    """rays [B,N,3], code [B,3,6,H,W] (may require grad), bitfield [B,G^3/8], dt_gamma list[B], noises [B,N] -> dict like the decoder"""
    dev = rays_o.device
    params = {k: v.to(dev) for k, v in params.items()}
    aabb = torch.tensor([-bound] * 3 + [bound] * 3, dtype=torch.float32, device=dev)
    nears, fars = batch_near_far_from_aabb(rays_o, rays_d, aabb, min_near)
    sig, rgb, deltas, rays, npts = [], [], [], [], []
    for b in range(rays_o.shape[0]):
        x, d, de, r = march_rays_train(rays_o[b], rays_d[b], bound, bitfield[b], 1, grid_size, nears[b], fars[b], perturb=True, align=128,
                                       force_all_rays=True, dt_gamma=float(dt_gamma[b]), max_steps=max_steps, noises=noises[b])
        s, c = torch_point_decode(params, x, d, code[b])
        sig.append(s); rgb.append(c); deltas.append(de); rays.append(r); npts.append(x.shape[0])
    ws, depth, image = batch_composite_rays_train(torch.cat(sig), torch.cat(rgb), deltas, rays, npts, T_thresh)
    return dict(weights_sum=ws, depth=depth, image=image)
