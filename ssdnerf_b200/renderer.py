"""Python front-end of the fused triplane renderer (C ABI section 2 of include/ssdnerf_b200.h).

`render_fwd` replaces the eval branch of the reference's ``VolumeRenderer.forward``
(lib/models/decoders/base_volume_renderer.py:79-123) + ``TriPlaneDecoder.point_decode``
(lib/models/decoders/triplane_decoder.py:119-179) with one launch sequence and no host sync.
"""
import torch

from . import _lib as N

DEC_P = 0   # shipped configs: base 18->64, density 64->1, dir_net 16->64, color 64->3
DEC_S = 1   # TriPlaneDecoder class defaults: base 96->128, density 128->1, color 144->128->3


def detect_variant(params):
    """Pick the kernel instantiation from a decoder state dict (keys: SURVEY.md Appendix D)."""
    w = params['base_net.0.weight']
    if tuple(w.shape) == (64, 18) and 'dir_net.0.weight' in params and tuple(params['color_net.0.weight'].shape) == (3, 64):
        return DEC_P
    if tuple(w.shape) == (128, 96) and 'dir_net.0.weight' not in params \
            and tuple(params['color_net.0.weight'].shape) == (128, 144) and 'color_net.2.weight' in params:
        return DEC_S
    raise N.SSDNeRFNativeError(
        'unsupported TriPlaneDecoder shape: kernels exist for the shipped-config decoder (18->64, dir_net 16->64, 64->3) '
        'and the class-default decoder (96->128, 144->128->3)')


def _plane_major(w, C):
    """columns of a Linear weight [out, 3*C] from the reference feature order c*3+plane to plane*C+c"""
    out = w.shape[0]
    return w.reshape(out, C, 3).permute(0, 2, 1).reshape(out, 3 * C)


def pack_decoder_blob(params, variant=None, sigmoid_saturation=0.001, device='cuda'):
    """Flatten decoder weights into the fp32 blob the kernels read (layout documented in csrc/dec_p.cuh
    `DecP` and csrc/render_common.cuh `DecS`)."""
    if variant is None:
        variant = detect_variant(params)
    p = {k: v.detach().float() for k, v in params.items()}       # packed where the weights live: no host round trip per optimiser step
    src = p['base_net.0.weight'].device

    def pad(t, n):
        return torch.cat([t, torch.zeros(n, device=src)])
    tail = torch.tensor([sigmoid_saturation, 0, 0, 0], dtype=torch.float32, device=src)
    if variant == DEC_P:
        w1 = _plane_major(p['base_net.0.weight'], 6).t().contiguous()           # [18][64], row k = plane*6+c
        parts = [w1.reshape(-1), p['base_net.0.bias'],
                 p['density_net.0.weight'].reshape(-1), pad(p['density_net.0.bias'], 3),
                 p['dir_net.0.weight'].t().contiguous().reshape(-1), p['dir_net.0.bias'],      # [16][64]
                 p['color_net.0.weight'].reshape(-1), pad(p['color_net.0.bias'], 1), tail]
    elif variant == DEC_S:
        w1 = _plane_major(p['base_net.0.weight'], 32)                             # [128][96] (N x K, K contiguous)
        wc0 = p['color_net.0.weight']                                             # [128][144]: cols 0..127 base_act, 128..143 SH
        parts = [w1.reshape(-1), p['base_net.0.bias'],
                 p['density_net.0.weight'].reshape(-1), pad(p['density_net.0.bias'], 3),
                 wc0.reshape(-1), p['color_net.0.bias'],
                 p['color_net.2.weight'].reshape(-1), pad(p['color_net.2.bias'], 1), tail]
    else:
        raise N.SSDNeRFNativeError(f'unknown decoder variant {variant}')
    blob = torch.cat([x.float() for x in parts]).contiguous()
    expect = N.lib().ssdnerf_decoder_blob_floats(N.c_int(variant))
    if blob.numel() != expect:
        raise N.SSDNeRFNativeError(f'decoder blob has {blob.numel()} floats, library expects {expect}')
    return blob.to(device)


DEC_P_PARAM_ORDER = ('base_net.0.weight', 'base_net.0.bias', 'density_net.0.weight', 'density_net.0.bias',
                     'dir_net.0.weight', 'dir_net.0.bias', 'color_net.0.weight', 'color_net.0.bias')


def unpack_decoder_blob_grad(grad_blob):
    """adjoint of `pack_decoder_blob` (variant P): blob-layout gradient [2572] -> tuple of parameter gradients in DEC_P_PARAM_ORDER"""
    g = grad_blob
    H, KF = 64, 18
    o = 0
    w1 = g[o:o + KF * H].reshape(3, 6, H); o += KF * H                     # [plane][c][out]
    b1 = g[o:o + H]; o += H
    wd = g[o:o + H].reshape(1, H); o += H
    bd = g[o:o + 1]; o += 4
    wdir = g[o:o + 16 * H].reshape(16, H); o += 16 * H
    bdir = g[o:o + H]; o += H
    wc = g[o:o + 3 * H].reshape(3, H); o += 3 * H
    bc = g[o:o + 3]
    # reference feature order of base_net's input is c*3 + plane (triplane_decoder.py:135-141)
    return (w1.permute(2, 1, 0).reshape(H, KF).contiguous(), b1.clone(), wd.clone(), bd.clone(),
            wdir.t().contiguous(), bdir.clone(), wc.clone(), bc.clone())


def pack_planes(code, variant):
    """code fp32 [B,3,C,H,W] (reference layout) -> channels-last gather layout (fp32 x8 for P, fp16 x32 for S)."""
    N.require_cuda(code)
    code = code.contiguous().float()
    B, three, C, H, W = code.shape
    assert three == 3
    nbytes = N.lib().ssdnerf_planes_bytes(N.c_int(variant), N.c_u32(B), N.c_u32(H), N.c_u32(W))
    planes = torch.empty(nbytes, dtype=torch.uint8, device=code.device)
    N.check(N.lib().ssdnerf_pack_planes(N.c_int(variant), N.ptr(code), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W),
                                        N.ptr(planes), N.stream_ptr()))
    return planes


def render_fwd(variant, planes, plane_hw, bitfield, blob, rays_o=None, rays_d=None, poses=None, intrinsics=None,
               img_hw=None, grid_size=64, bound=1.0, min_near=0.2, max_steps=256, T_thresh=1e-4, bg_color=1.0,
               dt_gamma=None, emulate_schedule=True, trace_cap=0, want_blend=True, want_counts=True):
    """One fused render of B scenes.

    Either explicit rays (rays_o, rays_d: [B,N,3]) or cameras (poses [B,V,4,4], intrinsics [B,V,4], img_hw).
    Returns dict(weights_sum [B,N], depth [B,N], image [B,N,3], rgb [B,N,3] (blended), num_samples [B,N] int32,
    trace [B,N,trace_cap] int32)."""
    N.require_cuda(planes, bitfield, blob)
    dev = planes.device
    if rays_o is not None:
        rays_o = rays_o.contiguous().float()
        rays_d = rays_d.contiguous().float()
        B, n = rays_o.shape[0], rays_o.shape[1]
        V = h = w = 0
    else:
        poses = poses.contiguous().float()
        intrinsics = intrinsics.contiguous().float()
        B, V = poses.shape[0], poses.shape[1]
        h, w = img_hw
        n = V * h * w
        if tuple(poses.shape[-2:]) != (4, 4):
            raise N.SSDNeRFNativeError('poses must be [B,V,4,4]')
    bitfield = bitfield.contiguous()
    if dt_gamma is not None:
        dt_gamma = dt_gamma.contiguous().float().to(dev)
    f32 = dict(dtype=torch.float32, device=dev)
    out = dict(weights_sum=torch.empty(B, n, **f32), depth=torch.empty(B, n, **f32), image=torch.empty(B, n, 3, **f32))
    out['rgb'] = torch.empty(B, n, 3, **f32) if want_blend else None
    out['num_samples'] = torch.empty(B, n, dtype=torch.int32, device=dev) if want_counts else None
    out['trace'] = torch.empty(B, n, trace_cap, dtype=torch.int32, device=dev) if trace_cap > 0 else None
    ws_bytes = N.lib().ssdnerf_render_workspace_bytes(N.c_u32(B), N.c_u32(n), N.c_u32(max_steps))
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    a = N.RenderArgs()
    a.variant = variant
    a.num_scenes, a.rays_per_scene = B, n
    a.rays_o, a.rays_d = N.ptr(rays_o), N.ptr(rays_d)
    a.poses, a.intrinsics = N.ptr(poses), N.ptr(intrinsics)
    a.num_views, a.img_h, a.img_w = V, h, w
    a.planes, a.plane_h, a.plane_w = N.ptr(planes), plane_hw[0], plane_hw[1]
    a.bitfield, a.grid_size = N.ptr(bitfield), grid_size
    a.decoder_blob, a.dt_gamma = N.ptr(blob), N.ptr(dt_gamma)
    a.bound, a.min_near, a.T_thresh, a.bg_color = bound, min_near, T_thresh, bg_color
    a.max_steps, a.emulate_schedule = max_steps, int(emulate_schedule)
    a.weights_sum, a.depth, a.image = N.ptr(out['weights_sum']), N.ptr(out['depth']), N.ptr(out['image'])
    a.rgb_blend, a.num_samples = N.ptr(out['rgb']), N.ptr(out['num_samples'])
    a.voxel_trace, a.trace_cap = N.ptr(out['trace']), trace_cap
    a.workspace, a.workspace_bytes = N.ptr(workspace), ws_bytes
    import ctypes
    N.check(N.lib().ssdnerf_render_fwd(ctypes.byref(a), N.stream_ptr()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# fused differentiable renderer (C ABI section 2b): train / guidance branch, gradient w.r.t. the triplane code
# ---------------------------------------------------------------------------------------------------------------------
def _train_args(planes, plane_hw, bitfield, blob, rays_o, rays_d, noises, dt_gamma, grid_size, bound, min_near, max_steps, T_thresh):
    B, n = rays_o.shape[0], rays_o.shape[1]
    a = N.RenderTrainArgs()
    a.variant = DEC_P
    a.num_scenes, a.rays_per_scene = B, n
    a.rays_o, a.rays_d, a.noises = N.ptr(rays_o), N.ptr(rays_d), N.ptr(noises)
    a.planes, a.plane_h, a.plane_w = N.ptr(planes), plane_hw[0], plane_hw[1]
    a.bitfield, a.grid_size = N.ptr(bitfield), grid_size
    a.decoder_blob, a.dt_gamma = N.ptr(blob), N.ptr(dt_gamma)
    a.bound, a.min_near, a.T_thresh, a.max_steps = bound, min_near, T_thresh, max_steps
    return a


def render_train_fwd(planes, plane_hw, bitfield, blob, rays_o, rays_d, noises=None, dt_gamma=None, grid_size=64, bound=1.0,
                     min_near=0.2, max_steps=256, T_thresh=1e-4, want_counts=False):
    """Train-branch forward (K6 march + decode + K7 compositing fused). rays [B,N,3]; noises [B,N] in [0,1) or None.
    Returns dict(weights_sum [B,N], depth [B,N], image [B,N,3], num_samples [B,N] | None)."""
    import ctypes
    N.require_cuda(planes, bitfield, blob, rays_o, rays_d)
    dev = planes.device
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    bitfield = bitfield.contiguous()
    noises = None if noises is None else noises.contiguous().float()
    dt_gamma = None if dt_gamma is None else dt_gamma.contiguous().float().to(dev)
    B, n = rays_o.shape[0], rays_o.shape[1]
    f32 = dict(dtype=torch.float32, device=dev)
    out = dict(weights_sum=torch.empty(B, n, **f32), depth=torch.empty(B, n, **f32), image=torch.empty(B, n, 3, **f32),
               num_samples=torch.empty(B, n, dtype=torch.int32, device=dev) if want_counts else None)
    counter = torch.empty(1, dtype=torch.int32, device=dev)
    a = _train_args(planes, plane_hw, bitfield, blob, rays_o, rays_d, noises, dt_gamma, grid_size, bound, min_near, max_steps, T_thresh)
    a.weights_sum, a.depth, a.image, a.num_samples = N.ptr(out['weights_sum']), N.ptr(out['depth']), N.ptr(out['image']), N.ptr(out['num_samples'])
    a.counter = N.ptr(counter)
    N.check(N.lib().ssdnerf_render_train_fwd(ctypes.byref(a), N.stream_ptr()))
    return out


def render_train_bwd(planes, plane_hw, bitfield, blob, rays_o, rays_d, weights_sum, image, grad_ws, grad_image, noises=None,
                     dt_gamma=None, grid_size=64, bound=1.0, min_near=0.2, max_steps=256, T_thresh=1e-4, code=None, reg_coef=0.0,
                     want_decoder_grad=False):
    """Train-branch backward: d(loss)/d(code) [B,3,6,H,W] from d(loss)/d(image) [B,N,3] and d(loss)/d(weights_sum) [B,N]
    (+ reg_coef * code when `code` is given: the RegLoss(power=2) gradient of BaseNeRF.loss).
    want_decoder_grad: also return d(loss)/d(decoder weights) in blob layout (-> `unpack_decoder_blob_grad`)."""
    import ctypes
    N.require_cuda(planes, bitfield, blob, rays_o, rays_d, weights_sum, image, grad_image)
    dev = planes.device
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    bitfield = bitfield.contiguous()
    noises = None if noises is None else noises.contiguous().float()
    dt_gamma = None if dt_gamma is None else dt_gamma.contiguous().float().to(dev)
    weights_sum, image = weights_sum.contiguous().float(), image.contiguous().float()
    grad_image = grad_image.contiguous().float()
    grad_ws = None if grad_ws is None else grad_ws.contiguous().float()
    B = rays_o.shape[0]
    H, W = plane_hw
    gplanes = torch.zeros(B, 3, H, W, 8, dtype=torch.float32, device=dev)
    counter = torch.empty(1, dtype=torch.int32, device=dev)
    a = _train_args(planes, plane_hw, bitfield, blob, rays_o, rays_d, noises, dt_gamma, grid_size, bound, min_near, max_steps, T_thresh)
    a.weights_sum, a.image = N.ptr(weights_sum), N.ptr(image)
    a.grad_ws, a.grad_image, a.grad_planes = N.ptr(grad_ws), N.ptr(grad_image), N.ptr(gplanes)
    a.counter = N.ptr(counter)
    grad_blob = torch.zeros(blob.numel(), dtype=torch.float32, device=dev) if want_decoder_grad else None
    a.grad_decoder_blob = N.ptr(grad_blob)
    N.check(N.lib().ssdnerf_render_train_bwd(ctypes.byref(a), N.stream_ptr()))
    grad_code = torch.empty(B, 3, 6, H, W, dtype=torch.float32, device=dev)
    if code is not None:
        code = code.contiguous().float()
    N.check(N.lib().ssdnerf_unpack_plane_grads(N.ptr(gplanes), N.ptr(code), N.c_f32(reg_coef), N.c_u32(B), N.c_u32(H), N.c_u32(W),
                                               N.c_int(0), N.ptr(grad_code), N.stream_ptr()))
    if want_decoder_grad:
        return grad_code, grad_blob
    return grad_code


def mse_render_loss(image, weights_sum, target, bg_color, coef_loss, coef_grad, want_rgb=False):
    """Pixel term of BaseNeRF.loss (base_nerf.py:283-287) fused with its gradient.
    Returns (loss [1] = coef_loss * sum((image + bg (1 - ws) - target)^2), grad_image, grad_ws, out_rgb | None)."""
    N.require_cuda(image, weights_sum, target)
    image, weights_sum, target = image.contiguous().float(), weights_sum.contiguous().float(), target.contiguous().float()
    rays = weights_sum.numel()
    loss = torch.zeros(1, dtype=torch.float32, device=image.device)
    g_image, g_ws = torch.empty_like(image), torch.empty_like(weights_sum)
    out_rgb = torch.empty_like(image) if want_rgb else None
    N.check(N.lib().ssdnerf_mse_render_loss(N.ptr(image), N.ptr(weights_sum), N.ptr(target), N.ctypes.c_uint64(rays), N.c_f32(bg_color),
                                            N.c_f32(coef_loss), N.c_f32(coef_grad), N.ptr(out_rgb), N.ptr(g_image), N.ptr(g_ws),
                                            N.ptr(loss), N.stream_ptr()))
    return loss, g_image, g_ws, out_rgb


def get_cam_rays(c2w, intrinsics, h, w):
    """lib/core/utils/nerf_utils.py:57-61 (+ :17-54): pixel-centre pinhole rays, -> rays_o, rays_d [B,V,h,w,3].
    Same arithmetic as the in-kernel ray generation of the fused eval renderer (csrc/render_common.cuh make_ray)."""
    N.require_cuda(c2w, intrinsics)
    B, V = c2w.shape[0], c2w.shape[1]
    poses = c2w.float()
    if poses.shape[-2] == 3:
        poses = torch.cat([poses, poses.new_tensor([0, 0, 0, 1]).expand(B, V, 1, 4)], dim=-2)
    poses, intrinsics = poses.contiguous(), intrinsics.contiguous().float()
    rays_o = torch.empty(B, V, h, w, 3, dtype=torch.float32, device=c2w.device)
    rays_d = torch.empty_like(rays_o)
    N.check(N.lib().ssdnerf_cam_rays(N.ptr(poses), N.ptr(intrinsics), N.c_u32(B), N.c_u32(V), N.c_u32(h), N.c_u32(w),
                                     N.ptr(rays_o), N.ptr(rays_d), N.stream_ptr()))
    return rays_o, rays_d
