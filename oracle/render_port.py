"""PyTorch-CPU + C restatement of the reference's triplane renderer -- TEST INFRASTRUCTURE ONLY.

Each function cites the reference file:line it follows (paths relative to Lakonik/SSDNeRF).
Parity is unpinned by reference tests (none exist); see oracle/__init__.py.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

import oracle as orc


# ----------------------------------------------------------------------------- rays
def get_cam_rays(c2w, intrinsics, h, w):
    """lib/core/utils/nerf_utils.py:17-61 (get_ray_directions + get_rays(norm=True)).

    c2w (*, 4, 4) or (*, 3, 4); intrinsics (*, 4) = fx, fy, cx, cy. Returns rays_o, rays_d (*, h, w, 3)."""
    batch = intrinsics.shape[:-1]
    x = torch.linspace(0.5, w - 0.5, w)
    y = torch.linspace(0.5, h - 0.5, h)
    dxy = torch.stack(
        [((x - intrinsics[..., 2:3]) / intrinsics[..., 0:1])[..., None, :].expand(*batch, h, w),
         ((y - intrinsics[..., 3:4]) / intrinsics[..., 1:2])[..., :, None].expand(*batch, h, w)], dim=-1)
    directions = F.pad(dxy, [0, 1], mode='constant', value=1.0)
    rays_d = directions @ c2w[..., None, :3, :3].transpose(-1, -2)
    rays_o = c2w[..., None, None, :3, 3].expand(rays_d.shape)
    rays_d = F.normalize(rays_d, dim=-1)
    return rays_o.contiguous(), rays_d.contiguous()


# ----------------------------------------------------------------------------- decoder
def xavier_uniform_linear(out_f, in_f, gen):
    """mmcv xavier_init(distribution='uniform', gain=1, bias=0) as used at triplane_decoder.py:97-100."""
    bound = math.sqrt(6.0 / (in_f + out_f))
    w = (torch.rand(out_f, in_f, generator=gen) * 2 - 1) * bound
    return w, torch.zeros(out_f)


def make_decoder_params(variant, seed=0, nonzero_dir=True):
    """Random decoder weights, keys = reference state-dict keys (SURVEY.md Appendix D).

    variant 'P' : shipped configs  base 18->64, density 64->1, dir_net 16->64, color 64->3
                  (configs/paper_cfgs/ssdnerf_cars_uncond.py:40-51)
    variant 'S' : TriPlaneDecoder class defaults base 96->128, density 128->1, color 144->128->3
                  (lib/models/decoders/triplane_decoder.py:24-39)
    The reference zero-inits dir_net (constant_init, :101-102); `nonzero_dir` re-draws it so the
    view-dependent path is exercised."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    if variant == 'P':
        p['base_net.0.weight'], p['base_net.0.bias'] = xavier_uniform_linear(64, 18, g)
        p['density_net.0.weight'], p['density_net.0.bias'] = xavier_uniform_linear(1, 64, g)
        p['dir_net.0.weight'], p['dir_net.0.bias'] = xavier_uniform_linear(64, 16, g)
        if not nonzero_dir:
            p['dir_net.0.weight'].zero_()
        p['color_net.0.weight'], p['color_net.0.bias'] = xavier_uniform_linear(3, 64, g)
    elif variant == 'S':
        p['base_net.0.weight'], p['base_net.0.bias'] = xavier_uniform_linear(128, 96, g)
        p['density_net.0.weight'], p['density_net.0.bias'] = xavier_uniform_linear(1, 128, g)
        p['color_net.0.weight'], p['color_net.0.bias'] = xavier_uniform_linear(128, 144, g)
        p['color_net.2.weight'], p['color_net.2.bias'] = xavier_uniform_linear(3, 128, g)
    else:
        raise ValueError(variant)
    # small random biases so bias handling is tested too
    for k in list(p):
        if k.endswith('.bias'):
            p[k] = (torch.rand(p[k].shape, generator=g) - 0.5) * 0.2
    return p


def xyz_transform(xyz):
    """triplane_decoder.py:104-117 (flip_z False): planes 0:(x,y) 1:(x,z) 2:(y,z) -> (3,1,M,2)."""
    xy = xyz[..., :2]
    xz = xyz[..., ::2]
    yz = xyz[..., 1:]
    return torch.stack([xy, xz, yz], dim=0).unsqueeze(1)


def _cast(params, xyzs, code_single, dtype):
    if dtype is None:
        return params, xyzs, code_single
    return {k: v.to(dtype) for k, v in params.items()}, xyzs.to(dtype), code_single.to(dtype)


def point_preacts(params, xyzs, dirs, code_single, dtype=None):
    """Pre-activations of the shipped-config decoder (variant P) at the given points: base_net (M,64), base_net + dir_net (the
    colour branch's SiLU input, (M,64)) and the density logit (M,).  `dtype` as in `point_decode`."""
    params, xyzs, code_single = _cast(params, xyzs, code_single, dtype)
    M = xyzs.shape[0]
    pc = F.grid_sample(code_single, xyz_transform(xyzs), mode='bilinear', padding_mode='border',
                       align_corners=False).squeeze(-2).permute(2, 1, 0).reshape(M, -1)
    base_x = F.linear(pc, params['base_net.0.weight'], params['base_net.0.bias'])
    logit = F.linear(F.silu(base_x), params['density_net.0.weight'], params['density_net.0.bias']).squeeze(-1)
    sh = torch.from_numpy(orc.sh_encode(dirs.numpy(), 4)).to(base_x.dtype)
    return base_x, base_x + F.linear(sh, params['dir_net.0.weight'], params['dir_net.0.bias']), logit


class TruncExp(torch.autograd.Function):
    """lib/ops/activation.py:8-22 (_trunc_exp): y = exp(x); dy/dx := clamp(y, 1e-6, 1e6).  Unlike the reference it keeps the input's
    precision, so the float64 oracle stays float64."""

    @staticmethod
    def forward(ctx, x):
        y = torch.exp(x)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return g * y.clamp(min=1e-6, max=1e6)


def point_decode(params, xyzs, dirs, code_single, density_only=False, sigmoid_saturation=0.001, dtype=None, trunc_exp=True):
    """triplane_decoder.py:119-179 for ONE scene. xyzs (M,3), dirs (M,3), code (3,C,h,w) -> sigmas (M,), rgbs (M,3).

    dtype: run the MLP (grid_sample, linears, SiLU, exp, sigmoid) in this precision, e.g. torch.float64 as the high-precision
    reference of the float32 kernels; None keeps the inputs' precision.  The SH encoding of `dirs` is float32 either way.
    trunc_exp: the density activation is the reference's TruncExp, whose gradient is floored at 1e-6 (a density logit below
    ln 1e-6 = -13.8 still passes gradient); False differentiates plain exp."""
    params, xyzs, code_single = _cast(params, xyzs, code_single, dtype)
    M = xyzs.shape[0]
    pc = F.grid_sample(code_single, xyz_transform(xyzs), mode='bilinear', padding_mode='border',
                       align_corners=False).squeeze(-2)          # (3, C, M)
    pc = pc.permute(2, 1, 0).reshape(M, -1)                        # feature index = c*3 + plane
    base_x = F.linear(pc, params['base_net.0.weight'], params['base_net.0.bias'])
    base_act = F.silu(base_x)
    logit = F.linear(base_act, params['density_net.0.weight'], params['density_net.0.bias'])
    sig = (TruncExp.apply(logit) if trunc_exp else torch.exp(logit)).squeeze(-1)
    if density_only:
        return sig, None
    sh = torch.from_numpy(orc.sh_encode(dirs.numpy(), 4)).to(base_x.dtype)
    if 'dir_net.0.weight' in params:
        color_in = F.silu(base_x + F.linear(sh, params['dir_net.0.weight'], params['dir_net.0.bias']))
        rgb = torch.sigmoid(F.linear(color_in, params['color_net.0.weight'], params['color_net.0.bias']))
    else:
        color_in = torch.cat([base_act, sh], dim=-1)
        hdn = F.silu(F.linear(color_in, params['color_net.0.weight'], params['color_net.0.bias']))
        rgb = torch.sigmoid(F.linear(hdn, params['color_net.2.weight'], params['color_net.2.bias']))
    if sigmoid_saturation > 0:
        rgb = rgb * (1 + sigmoid_saturation * 2) - sigmoid_saturation
    return sig, rgb


# ----------------------------------------------------------------------------- eval renderer
def render_eval_scene(params, rays_o, rays_d, code_single, bitfield, grid_size=64, bound=1.0, min_near=0.2,
                      max_steps=256, dt_gamma=0.0, T_thresh=1e-4, return_trace=False, return_samples=False, dtype=None):
    """lib/models/decoders/base_volume_renderer.py:79-123 for one scene (eval branch, perturb=False).

    rays_o/d: float32 numpy (N,3); bitfield uint8 numpy (H^3/8,). Returns dict of numpy arrays
    (weights_sum, depth, image) and, with return_trace, per-ray list of sampled voxel bit indices;
    with return_samples, `samples` = (xyzs, dirs) float32 (S,3) of every sample the compositor consumed.
    dtype: precision of the MLP (`point_decode`); sigmas and colours are rounded to float32 before compositing, so the march
    and the compositor stay float32 whatever the MLP runs in."""
    return_trace = return_trace or return_samples
    rays_o = np.ascontiguousarray(rays_o, np.float32)
    rays_d = np.ascontiguousarray(rays_d, np.float32)
    N = rays_o.shape[0]
    aabb = np.array([-bound, -bound, -bound, bound, bound, bound], np.float32)
    nears, fars = orc.near_far_from_aabb(rays_o, rays_d, aabb, min_near)
    ws = np.zeros(N, np.float32)
    depth = np.zeros(N, np.float32)
    image = np.zeros((N, 3), np.float32)
    rays_alive = np.arange(N, dtype=np.int32)
    rays_t = nears.copy()
    trace = [[] for _ in range(N)] if return_trace else None
    samples = [] if return_samples else None
    step = 0
    n_quanta = 0
    with torch.no_grad():
        while step < max_steps:
            n_alive = rays_alive.shape[0]
            if n_alive == 0:
                break
            n_step = min(max(N // n_alive, 1), 8)
            out = orc.march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, bitfield, 1, grid_size,
                                 nears, fars, align=128, dt_gamma=dt_gamma, max_steps=max_steps,
                                 return_voxels=return_trace)
            xyzs, dirs, deltas = out[:3]
            sig, rgb = point_decode(params, torch.from_numpy(xyzs), torch.from_numpy(dirs), code_single, dtype=dtype)
            sig = sig.float().numpy()
            rgb = rgb.float().numpy()
            if return_trace:
                vox = out[3]
                # a sample is *consumed* by the compositor unless an earlier one in the quantum broke the loop
                ws_before = ws[rays_alive].copy()
            alive_before = rays_alive.copy()
            if return_trace:
                picked = _consumed_trace(trace, alive_before, n_step, vox, sig, deltas, ws_before, T_thresh)
                if return_samples:
                    samples.append((xyzs[picked], dirs[picked]))
            orc.composite_rays(n_alive, n_step, rays_alive, rays_t, sig, rgb, deltas, ws, depth, image, T_thresh)
            rays_alive = np.ascontiguousarray(rays_alive[rays_alive >= 0])
            step += n_step
            n_quanta += 1
    res = dict(weights_sum=ws, depth=depth, image=image, nears=nears, fars=fars, total_budget=step, n_quanta=n_quanta)
    if return_trace:
        res['trace'] = trace
    if return_samples:
        res['samples'] = tuple(np.concatenate([s[i] for s in samples]).reshape(-1, 3) for i in range(2))
    return res


def _consumed_trace(trace, alive, n_step, vox, sig, deltas, ws_before, T_thresh):
    """Replays K10's control flow (raymarching.cu:865-897) to record which samples were accumulated; returns their indices."""
    picked = []
    for n, ridx in enumerate(alive):
        w_sum = float(ws_before[n])
        for s in range(n_step):
            k = n * n_step + s
            if deltas[k, 0] == 0:
                break
            trace[ridx].append(int(vox[k]))
            picked.append(k)
            alpha = np.float32(1.0) - np.float32(math.exp(-float(sig[k]) * float(deltas[k, 0])))
            T = np.float32(1.0) - np.float32(w_sum)
            w_sum = float(np.float32(w_sum) + np.float32(alpha * T))
            if T < T_thresh:
                break
    return picked


def render_image(params, code, bitfield, poses, intrinsics, h, w, bg_color=1.0, **kw):
    """lib/models/autodecoders/base_nerf.py:494-533 for one scene: returns (V,h,w,3) rgb, (V,h,w) depth."""
    rays_o, rays_d = get_cam_rays(poses, intrinsics, h, w)
    V = rays_o.shape[0]
    ro = rays_o.reshape(-1, 3).numpy()
    rd = rays_d.reshape(-1, 3).numpy()
    out = render_eval_scene(params, ro, rd, code, bitfield, **kw)
    rgb = out['image'] + bg_color * (1 - out['weights_sum'][:, None])
    return rgb.reshape(V, h, w, 3), out['depth'].reshape(V, h, w), out


# ----------------------------------------------------------------------------- density grid
def voxel_centres(grid_size=64, bound=1.0):
    """base_nerf.py:328-343: ij-meshgrid coords, morton indices, un-jittered centres."""
    X = torch.arange(grid_size, dtype=torch.int32)
    xx, yy, zz = torch.meshgrid(X, X, X, indexing='ij')
    coords = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
    indices = torch.from_numpy(orc.morton3D(coords.numpy())).long()
    xyzs = (coords.float() - (grid_size - 1) / 2) * (2 * bound / grid_size)
    return coords, indices, xyzs


def update_extra_state(params, code, density_grid, rand, density_thresh=0.01, decay=0.9, grid_size=64, bound=1.0):
    """base_nerf.py:318-389, full-update branch (iter_density < 16), with the jitter `rand`
    (= the torch.rand_like tensor of :344, shape (G^3, 3)) injected.

    code (B,3,C,h,w) torch; density_grid (B, G^3) torch float32 or float16 (updated in place).
    Returns the packed bitfield (B, G^3/8) uint8 numpy and the threshold used."""
    B = density_grid.shape[0]
    coords, indices, xyzs = voxel_centres(grid_size, bound)
    half = bound / grid_size
    xyzs = xyzs + (rand * (2 * half) - half)
    tmp = torch.full_like(density_grid, -1)
    with torch.no_grad():
        for b in range(B):
            sig, _ = point_decode(params, xyzs, None, code[b], density_only=True)
            tmp[b, indices] = sig.clamp(max=torch.finfo(tmp.dtype).max).to(tmp.dtype)
    valid = (density_grid >= 0) & (tmp >= 0)
    density_grid[:] = torch.where(valid, torch.maximum(density_grid * decay, tmp), density_grid)
    mean_density = torch.mean(density_grid.clamp(min=0))
    thresh = min(float(mean_density), density_thresh)
    bitfield = orc.packbits(density_grid.float().numpy().reshape(-1), thresh).reshape(B, -1)
    return bitfield, thresh


def get_density(params, code, rands, density_thresh=0.01, grid_size=64, bound=1.0, grid_dtype=torch.float16):
    """base_nerf.py:391-401: density_step iterations, decay=1.0, zero-initialised fp16 grid (:194-197)."""
    B = code.shape[0]
    grid = torch.zeros(B, grid_size ** 3, dtype=grid_dtype)
    bitfield = None
    for r in rands:
        bitfield, thresh = update_extra_state(params, code, grid, r, density_thresh, 1.0, grid_size, bound)
    return grid, bitfield


def sphere_bitfield(grid_size=64, radius=0.6, bound=1.0):
    """Analytic occupancy mask of SURVEY.md §8d config 1(iii): voxel centre inside a sphere, morton order, LSB-first."""
    coords, indices, xyzs = voxel_centres(grid_size, bound)
    occ = (xyzs.norm(dim=-1) < radius)
    grid = torch.zeros(grid_size ** 3)
    grid[indices] = occ.float()
    return orc.packbits(grid.numpy(), 0.5)
