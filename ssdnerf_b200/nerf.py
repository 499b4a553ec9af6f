"""`BaseNeRF` / `MultiSceneNeRF` / `DiffusionNeRF` -- the registered models of the reference's configs.

Plugin surface of lib/models/autodecoders/{base_nerf,multiscene_nerf,diffusion_nerf}.py: constructor kwargs, the registered names,
`val_step(data, viz_dir=, viz_dir_guide=, **kw) -> {log_vars, num_samples, pred_imgs}` with all four branches of
diffusion_nerf.py:406-469 (stored scenes / `guide` / `optim` / `guide_optim` / unconditional), `val_uncond`, `val_guide`, `val_optim`,
`inverse_code`, `loss`, `loss_decoder`, `ray_sample`, `get_raybatch_inds`, `update_extra_state`, `get_density`, `render`,
`load_scene` / `save_scene`, `code_diff_pr(_inv)`, the `train()` override that applies `test_cfg.override_cfg`.

HOW it runs differs: DDIM = one replayed CUDA graph (diffusion.py), occupancy grid = 2 launches per iteration (density.py), render and
the render loss = fused kernels (renderer.py), guidance through the denoiser and the diffusion-prior gradient of `val_optim` = the
hand-written UNet input-gradient pass (unet.py `_UNetInputGrad`).  Stage-1 training (`MultiSceneNeRF.train_step`: latents + decoder,
scene cache) runs on the fused differentiable renderer with decoder-weight gradients; `DiffusionNeRF.train_step` (single-stage / stage-2
training) adds the denoiser's weight-gradient pass (unet_train.py, csrc/wgrad.cu).
"""
import functools
import math
import os
import warnings
from contextlib import contextmanager
from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib as N
from . import density as D
from . import mesh as MC
from . import metrics as M
from . import renderer as R
from . import viz as V
from .registry import MODELS, MODULES, build_module
from .scene_cache import SceneCache, restore_optimizer_state


# --------------------------------------------------------------------------------------------------------------------- small modules
@MODULES.register_module()
class TanhCode(nn.Module):
    """latent activation tanh(x) * scale and its inverse (base_nerf.py:25-37)"""

    def __init__(self, scale=1.0, eps=1e-5):
        super().__init__()
        self.scale, self.eps = scale, eps

    def forward(self, code_, update_stats=False):
        return code_.tanh() if self.scale == 1 else code_.tanh() * self.scale

    def inverse(self, code):
        return code.div(self.scale).clamp(min=-1 + self.eps, max=1 - self.eps).atanh()


@MODULES.register_module()
class IdentityCode(nn.Module):
    """base_nerf.py:40-48"""

    @staticmethod
    def forward(code_, update_stats=False):
        return code_

    @staticmethod
    def inverse(code):
        return code


@MODULES.register_module()
class NormalizedTanhCode(nn.Module):
    """tanh on codes standardised by running statistics (base_nerf.py:51-76); buffers `running_mean`, `running_var` are part of the
    released checkpoints' state dict.  Statistics only move in training (`update_stats and self.training`)."""

    def __init__(self, mean=0.0, std=1.0, clip_range=1, eps=1e-5, momentum=0.001):
        super().__init__()
        self.mean, self.std, self.clip_range, self.eps, self.momentum = mean, std, clip_range, eps, momentum
        self.register_buffer('running_mean', torch.tensor([0.0]))
        self.register_buffer('running_var', torch.tensor([std ** 2]))

    def _gain(self):
        return self.std / (self.running_var.sqrt() + self.eps)

    def forward(self, code_, update_stats=False):
        if update_stats and self.training:
            with torch.no_grad():
                var, mean = torch.var_mean(code_)
                if torch.distributed.is_available() and torch.distributed.is_initialized():
                    world = torch.distributed.get_world_size()
                    torch.distributed.all_reduce(mean); torch.distributed.all_reduce(var)
                    mean, var = mean / world, var / world
                self.running_mean.lerp_(mean.to(self.running_mean), self.momentum)
                self.running_var.lerp_(var.to(self.running_var), self.momentum)
        gain = self._gain().to(code_.device)
        offset = self.mean - self.running_mean.to(code_.device) * gain
        return torch.tanh((code_ * gain + offset) / self.clip_range) * self.clip_range

    def inverse(self, code):
        inv_gain = (1.0 / self._gain()).to(code.device)
        z = torch.atanh((code / self.clip_range).clamp(min=-1 + self.eps, max=1 - self.eps)) * self.clip_range
        return z * inv_gain + (self.running_mean.to(code.device) - self.mean * inv_gain)


@MODULES.register_module()
class MSELoss(nn.Module):
    """mmgen.models.losses.pixelwise_loss.MSELoss [mmgen-memory]: mean squared error * loss_weight."""

    def __init__(self, loss_weight=1.0, reduction='mean', **kwargs):
        super().__init__()
        assert reduction == 'mean'
        self.loss_weight = loss_weight

    def forward(self, pred, target, **kwargs):
        return torch.nn.functional.mse_loss(pred, target) * self.loss_weight


@MODULES.register_module()
class RegLoss(nn.Module):
    """lib/models/losses/reg_loss.py:7-30"""

    def __init__(self, power=1, loss_weight=1.0):
        super().__init__()
        self.power, self.loss_weight = power, loss_weight

    def forward(self, tensor, **kwargs):
        return (tensor.abs().mean() if self.power == 1 else (tensor.abs() ** self.power).mean()) * self.loss_weight


@MODULES.register_module()
class TVLoss(nn.Module):
    """lib/models/losses/tv_loss.py:9-37: mean over all elements of (L2 norm over `dims` of the forward differences, zero at the far
    edge) ** power, times loss_weight (regulariser of the stage-1 auto-decoder configs)"""

    def __init__(self, dims=[-2, -1], power=1, loss_weight=1.0):
        super().__init__()
        self.dims, self.power, self.loss_weight = list(dims), power, loss_weight

    def forward(self, tensor, weight=None, avg_factor=None):
        diffs = []
        for dim in self.dims:
            d = torch.diff(tensor, dim=dim)
            diffs.append(torch.nn.functional.pad(d, [0, 0] * ((-dim - 1) % tensor.dim()) + [0, 1]))
        # vector_norm, not sqrt(sum of squares): its backward is 0 (not 0 * inf) where all differences vanish, e.g. the all-zero
        # latents every scene starts from under init_from_mean
        loss = torch.linalg.vector_norm(torch.stack(diffs), dim=0).pow(self.power)
        if weight is not None:
            loss = loss * weight
        loss = loss.mean() if avg_factor is None else loss.sum() / avg_factor
        return loss * self.loss_weight


def rgetattr(obj, attr, *default):
    """dotted getattr (lib/core/utils/misc.py:129-134)"""
    return functools.reduce(lambda o, a: getattr(o, a, *default), [obj] + attr.split('.'))


def rsetattr(obj, attr, val):
    """dotted setattr (lib/core/utils/misc.py:137-142); a name whose owner is a dict is set as an item, so plain-dict configs
    (`train_cfg.optimizer.lr`) take settings as mmcv's ConfigDict does"""
    head, _, tail = attr.rpartition('.')
    owner = obj
    for name in head.split('.') if head else []:
        owner = owner[name] if isinstance(owner, dict) else getattr(owner, name)
    if isinstance(owner, dict):
        owner[tail] = val
    else:
        setattr(owner, tail, val)


@contextmanager
def module_requires_grad(module, requires_grad=True):
    """temporarily set requires_grad of every parameter (lib/core/utils/misc.py)"""
    prev = [p.requires_grad for p in module.parameters()]
    for p in module.parameters():
        p.requires_grad_(requires_grad)
    try:
        yield
    finally:
        for p, r in zip(module.parameters(), prev):
            p.requires_grad_(r)


def extract_fields(decoder, code_single, resolution=256, margin=0.1):
    """density sigma on a resolution^3 lattice over [aabb_min - margin, aabb_max + margin] (lib/core/utils/nerf_utils.py:64-81 + the
    query of :98-106): ONE native point-decode launch instead of the reference's 8 chunked host round trips; points outside the AABB
    read 0.  Returns a float32 CUDA tensor [R, R, R] indexed [x, y, z]."""
    dev = code_single.device
    lo, hi = decoder.aabb[:3].to(dev) - margin, decoder.aabb[3:].to(dev) + margin
    axes = [torch.linspace(float(lo[i]), float(hi[i]), resolution, device=dev) for i in range(3)]
    pts = torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=-1).reshape(1, -1, 3)
    sigma, _ = decoder.point_density_decode(pts, code_single[None])
    outside = ((pts[0] < decoder.aabb[:3].to(dev)) | (pts[0] > decoder.aabb[3:].to(dev))).any(dim=-1)
    return sigma.masked_fill(outside, 0).reshape(resolution, resolution, resolution)


def extract_geometry(decoder, code_single, resolution=256, threshold=10):
    """nerf_utils.py:84-112: marching cubes on the device (`mesh.marching_cubes`, PyMCubes' contract) over `extract_fields`, mapped to
    world coordinates by the reference's formula.  Returns numpy float64 vertices [V, 3] and int64 triangles [T, 3]."""
    with torch.no_grad():
        u = extract_fields(decoder, code_single, resolution)
    vertices, triangles = MC.marching_cubes(u, threshold)
    vertices, triangles = vertices.cpu().numpy(), triangles.cpu().numpy()
    lo = (decoder.aabb[:3] - 0.1).cpu().numpy()
    hi = (decoder.aabb[3:] + 0.1).cpu().numpy()
    return vertices / (resolution - 1.0) * (hi - lo)[None, :] + lo[None, :], triangles


class _RenderMSELoss(torch.autograd.Function):
    """pixel + reg terms of BaseNeRF.loss as ONE differentiable op on the fused renderer: forward = render_train_fwd +
    mse_render_loss (which also leaves d/d image, d/d weights_sum), backward = render_train_bwd (+ RegLoss gradient)."""

    @staticmethod
    def forward(ctx, code, rays_o, rays_d, target, bitfield, blob, noises, dt_gamma, cfg, bg_color, pix_coef, reg_weight, *params):
        planes = R.pack_planes(code, R.DEC_P)
        hw = tuple(code.shape[-2:])
        out = R.render_train_fwd(planes, hw, bitfield, blob, rays_o, rays_d, noises=noises, dt_gamma=dt_gamma, **cfg)
        n_el = target.numel()
        loss, g_image, g_ws, rgb = R.mse_render_loss(out['image'], out['weights_sum'], target, bg_color, pix_coef / n_el,
                                                     2.0 * pix_coef / n_el, want_rgb=True)
        reg = None
        if reg_weight is not None:
            reg = code.square().mean() * reg_weight
        ctx.save_for_backward(planes, rays_o, rays_d, bitfield, blob, noises, dt_gamma, out['weights_sum'], out['image'], g_image, g_ws,
                              code if reg_weight is not None else None)
        ctx.hw, ctx.cfg, ctx.reg_weight = hw, cfg, reg_weight
        ctx.mark_non_differentiable(rgb)
        return loss.reshape(()), (reg if reg is not None else loss.new_zeros(())), rgb

    @staticmethod
    def backward(ctx, g_pix, g_reg, g_rgb):
        planes, rays_o, rays_d, bitfield, blob, noises, dt_gamma, ws, image, g_image, g_ws, code = ctx.saved_tensors
        want = any(ctx.needs_input_grad[12:])
        grad = R.render_train_bwd(planes, ctx.hw, bitfield, blob, rays_o, rays_d, ws, image, g_ws, g_image, noises=noises,
                                  dt_gamma=dt_gamma, want_decoder_grad=want, **ctx.cfg)
        gparams = (None,) * len(ctx.needs_input_grad[12:])
        if want:      # trainable decoder (multiscene_nerf.py:203-207): weight gradients from the same backward launch
            grad, gblob = grad
            gparams = tuple(g * g_pix for g in R.unpack_decoder_blob_grad(gblob))
        if code is not None:      # RegLoss(power=2): d/d code = 2 w code / numel, with its own upstream gradient
            return (torch.addcmul(grad * g_pix, code, g_reg, value=2.0 * ctx.reg_weight / code.numel()),) + (None,) * 11 + gparams
        return (grad * g_pix,) + (None,) * 11 + gparams


# --------------------------------------------------------------------------------------------------------------------- BaseNeRF
class BaseNeRF(nn.Module):
    """base_nerf.py:79-673, inference side"""

    def __init__(self, code_size=(3, 8, 64, 64), code_activation=dict(type='TanhCode', scale=1), grid_size=64,
                 decoder=dict(type='TriPlaneDecoder'), decoder_use_ema=False, bg_color=1, pixel_loss=dict(type='MSELoss'), reg_loss=None,
                 update_extra_interval=16, use_lpips_metric=True, init_from_mean=False, init_scale=1e-4, mean_ema_momentum=0.001,
                 mean_scale=1.0, train_cfg=dict(), test_cfg=dict(), pretrained=None):
        super().__init__()
        self.code_size = tuple(code_size)
        self.code_activation = build_module(code_activation)
        self.grid_size = grid_size
        self.decoder = build_module(decoder)
        self.decoder_use_ema = decoder_use_ema
        if self.decoder_use_ema:
            self.decoder_ema = deepcopy(self.decoder)
        self.bg_color = bg_color
        self.pixel_loss = build_module(pixel_loss if pixel_loss is not None else dict(type='MSELoss'))
        self.reg_loss = build_module(reg_loss) if reg_loss is not None else None
        self.train_cfg = train_cfg if train_cfg is not None else dict()     # live dicts, like the reference (base_nerf.py:115-116)
        self.test_cfg = test_cfg if test_cfg is not None else dict()
        self.update_extra_interval = update_extra_interval
        self.use_lpips_metric = use_lpips_metric
        # base_nerf.py:116: a list, so the LPIPS network stays out of the state dict; filled on first use from the default weight files
        # (ssdnerf_b200/lpips.py), or by the caller with its own `LPIPS(vgg_path, lin_path)`
        self.lpips = [] if use_lpips_metric else None
        self._lpips_missing_warned = False
        if init_from_mean:
            self.register_buffer('init_code', torch.zeros(self.code_size))
        else:
            self.init_code = None
        self.init_scale, self.mean_ema_momentum, self.mean_scale = init_scale, mean_ema_momentum, mean_scale
        if pretrained is not None and os.path.isfile(pretrained):
            state = torch.load(pretrained, map_location='cpu')
            self.load_state_dict(state.get('state_dict', state), strict=False)
        self.train_cfg_backup = dict()
        for key in self.test_cfg.get('override_cfg', dict()):
            self.train_cfg_backup[key] = rgetattr(self, key, None)

    def train(self, mode=True):
        """base_nerf.py:128-139: attributes listed in test_cfg.override_cfg take their test values in eval mode"""
        if mode:
            for key, value in self.train_cfg_backup.items():
                rsetattr(self, key, value)
        else:
            for key, value in self.test_cfg.get('override_cfg', dict()).items():
                if self.training:
                    self.train_cfg_backup[key] = rgetattr(self, key)
                rsetattr(self, key, value)
        return super().train(mode)

    # ------------------------------------------------------------------ scene I/O (base_nerf.py:141-170)
    def load_scene(self, data, load_density=False):
        """scene states as written by `save_scene` / the training cache: dict(param=dict(code | code_, density_grid, density_bitfield))"""
        device = next(self.parameters()).device
        codes, grids, bits = [], [], []
        for state in data['code']:
            param = state['param']
            codes.append(param['code'] if 'code' in param else self.code_activation(param['code_']))
            if load_density:
                grids.append(param['density_grid'])
                bits.append(param['density_bitfield'])
        code = torch.stack(codes, dim=0).to(device=device, dtype=torch.float32)
        if not load_density:
            return code, None, None
        return code, torch.stack(grids, dim=0).to(device), torch.stack(bits, dim=0).to(device)

    @staticmethod
    def save_scene(save_dir, code, density_grid, density_bitfield, scene_name):
        """one `<scene_name>.pth` per scene: code fp32 [3,C,H,W], density_grid (fp16, morton order) [G^3], density_bitfield u8 [G^3/8]"""
        os.makedirs(save_dir, exist_ok=True)
        for i, name in enumerate(scene_name):
            torch.save(dict(scene_name=name, param=dict(code=code.data[i].cpu(), density_grid=density_grid.data[i].cpu(),
                                                        density_bitfield=density_bitfield.data[i].cpu())),
                       os.path.join(save_dir, name) + '.pth')

    @staticmethod
    def save_mesh(save_dir, decoder, code, scene_name, mesh_resolution, mesh_threshold):
        """base_nerf.py:172-182: one binary `<scene_name>.stl` per scene -- density lattice and marching cubes on the device
        (`extract_geometry`), file by `mesh.write_stl`"""
        os.makedirs(save_dir, exist_ok=True)
        for code_single, name in zip(code, scene_name):
            vertices, triangles = extract_geometry(decoder, code_single, mesh_resolution, mesh_threshold)
            MC.write_stl(os.path.join(save_dir, name) + '.stl', vertices, triangles)

    def get_init_code_(self, num_scenes, device=None):
        code_ = torch.empty(self.code_size if num_scenes is None else (num_scenes, *self.code_size), device=device, requires_grad=True,
                            dtype=torch.float32)
        if self.init_code is None:
            code_.data.uniform_(-self.init_scale, self.init_scale)
        else:
            code_.data[:] = self.code_activation.inverse(self.init_code * self.mean_scale)
        return code_

    def get_init_density_grid(self, num_scenes, device=None):
        return torch.zeros(self.grid_size ** 3 if num_scenes is None else (num_scenes, self.grid_size ** 3), device=device, dtype=torch.float16)

    def get_init_density_bitfield(self, num_scenes, device=None):
        return torch.zeros(self.grid_size ** 3 // 8 if num_scenes is None else (num_scenes, self.grid_size ** 3 // 8), device=device,
                           dtype=torch.uint8)

    @staticmethod
    def build_optimizer(code_, cfg):
        """base_nerf.py:204-214: torch.optim class named by cfg['optimizer'] on the latent(s)"""
        ocfg = dict(cfg['optimizer'])
        cls = getattr(torch.optim, ocfg.pop('type'))
        if isinstance(code_, list):
            return [cls([c], **ocfg) for c in code_]
        return cls([code_], **ocfg)

    @staticmethod
    def build_scheduler(code_optimizer, cfg):
        if 'lr_scheduler' not in cfg:
            return None
        scfg = dict(cfg['lr_scheduler'])
        cls = getattr(torch.optim.lr_scheduler, scfg.pop('type'))
        if isinstance(code_optimizer, list):
            return [cls(o, **scfg) for o in code_optimizer]
        return cls(code_optimizer, **scfg)

    # ------------------------------------------------------------------ ray batches (contract of base_nerf.py:231-274)
    @staticmethod
    def _scene_permutations(num_scenes, length, device):
        """one independent random permutation of range(length) per scene, [num_scenes, length] (one randperm draw per scene, scene order)"""
        return torch.stack([torch.randperm(length, device=device) for _ in range(num_scenes)])

    @staticmethod
    def ray_sample(cond_rays_o, cond_rays_d, cond_imgs, n_samples, sample_inds=None):
        """[B,V,h,w,3] rays / colours -> per-scene batches [B,n,3]; all pixels when a scene has no more than n_samples of them"""
        flat = [t.reshape(t.size(0), -1, 3) for t in (cond_rays_o, cond_rays_d, cond_imgs)]
        pixels = flat[0].size(1)
        if pixels <= n_samples:
            return tuple(flat)
        if sample_inds is None:
            sample_inds = BaseNeRF._scene_permutations(flat[0].size(0), pixels, cond_rays_o.device)[:, :n_samples]
        pick = sample_inds.unsqueeze(-1).expand(-1, -1, 3)
        return tuple(t.gather(1, pick) for t in flat)

    @staticmethod
    def get_raybatch_inds(cond_imgs, n_inverse_rays):
        """-> (tuple of index batches [B, <= n_inverse_rays] covering every pixel once, their number), or (None, None) when one batch holds all"""
        pixels = cond_imgs[0].numel() // 3
        if pixels <= n_inverse_rays:
            return None, None
        batches = BaseNeRF._scene_permutations(cond_imgs.size(0), pixels, cond_imgs.device).split(n_inverse_rays, dim=1)
        return batches, len(batches)

    # ------------------------------------------------------------------ losses (base_nerf.py:276-316)
    def loss(self, decoder, code, density_bitfield, target_rgbs, rays_o, rays_d, dt_gamma=0.0, return_decoder_loss=False,
             scale_num_ray=1.0, cfg=dict(), perturb=True, **kwargs):
        """base_nerf.py:276-296.  With a frozen shipped-config decoder and the stock MSELoss / RegLoss(power=2) the whole
        chain (render, blend, MSE, reg) is one fused differentiable op; anything else composes the decoder's differentiable
        forward with the loss modules like the reference.  `perturb` may be a [B,N] tensor of start offsets (tests)."""
        scale = 1 - math.exp(-cfg['loss_coef'] * scale_num_ray) if 'loss_coef' in cfg else 1
        fusable = (isinstance(self.pixel_loss, MSELoss) and (self.reg_loss is None or (isinstance(self.reg_loss, RegLoss) and self.reg_loss.power == 2))
                   and not (return_decoder_loss and decoder.decoder_reg_loss is not None) and isinstance(rays_o, torch.Tensor)
                   and decoder.training and hasattr(decoder, '_fused_train_ok') and decoder._fused_train_ok(rays_o, code, self.grid_size))
        if fusable:
            num_scenes = rays_o.size(0)
            rays_o = rays_o.reshape(num_scenes, -1, 3).contiguous().float()
            rays_d = rays_d.reshape(num_scenes, -1, 3).contiguous().float()
            if isinstance(dt_gamma, (int, float)):
                dtg = None if dt_gamma == 0 else torch.full((num_scenes,), float(dt_gamma), device=rays_o.device)
            else:
                dtg = torch.as_tensor(dt_gamma, dtype=torch.float32, device=rays_o.device).reshape(num_scenes).contiguous()
            if isinstance(perturb, torch.Tensor):
                noises = perturb.reshape(num_scenes, -1).contiguous().float()
            else:
                noises = torch.rand(num_scenes, rays_o.size(1), device=rays_o.device) if perturb else None
            rcfg = dict(grid_size=int(self.grid_size), bound=float(decoder.bound), min_near=float(decoder.min_near),
                        max_steps=int(decoder.max_steps), T_thresh=1e-4)
            pixel_loss, reg_loss, out_rgbs = _RenderMSELoss.apply(
                code, rays_o, rays_d, target_rgbs.reshape(num_scenes, -1, 3), density_bitfield.reshape(num_scenes, -1).contiguous(),
                decoder.packed_blob(), noises, dtg, rcfg, float(self.bg_color), float(self.pixel_loss.loss_weight * scale * 3),
                None if self.reg_loss is None else float(self.reg_loss.loss_weight), *decoder.trainable_params())
            loss, loss_dict = pixel_loss, dict(pixel_loss=pixel_loss)
            if self.reg_loss is not None:
                loss = loss + reg_loss
                loss_dict.update(reg_loss=reg_loss)
            return out_rgbs, loss, loss_dict
        outputs = decoder(rays_o, rays_d, code, density_bitfield, self.grid_size, dt_gamma=dt_gamma, perturb=perturb,
                          return_loss=return_decoder_loss)
        out_weights = outputs['weights_sum']
        out_rgbs = outputs['image'] + self.bg_color * (1 - out_weights.unsqueeze(-1))
        pixel_loss = self.pixel_loss(out_rgbs, target_rgbs, **kwargs) * (scale * 3)
        loss, loss_dict = pixel_loss, dict(pixel_loss=pixel_loss)
        if self.reg_loss is not None:
            reg_loss = self.reg_loss(code, **kwargs)
            loss = loss + reg_loss
            loss_dict.update(reg_loss=reg_loss)
        if return_decoder_loss and outputs['decoder_reg_loss'] is not None:
            loss = loss + outputs['decoder_reg_loss']
            loss_dict.update(decoder_reg_loss=outputs['decoder_reg_loss'])
        return out_rgbs, loss, loss_dict

    def loss_decoder(self, decoder, code, density_bitfield, cond_rays_o, cond_rays_d, cond_imgs, dt_gamma=0.0, cfg=dict(), **kwargs):
        """base_nerf.py:298-316"""
        prev = decoder.training
        decoder.train(True)
        rays_o, rays_d, target_rgbs = self.ray_sample(cond_rays_o, cond_rays_d, cond_imgs, n_samples=cfg.get('n_decoder_rays', 4096))
        out_rgbs, loss, loss_dict = self.loss(decoder, code, density_bitfield, target_rgbs, rays_o, rays_d, dt_gamma, return_decoder_loss=True,
                                              scale_num_ray=cond_rays_o.shape[1:4].numel(), cfg=cfg, **kwargs)
        decoder.train(prev)
        return loss, {k: float(v.detach()) for k, v in loss_dict.items()}, out_rgbs, target_rgbs

    # ------------------------------------------------------------------ occupancy grid (base_nerf.py:318-401)
    def update_extra_state(self, decoder, code, density_grid, density_bitfield, iter_density, density_thresh=0.01, decay=0.9,
                           S=128, jitter=None):
        """full-update branch (iter_density < 16; the partial update only occurs in training)."""
        if iter_density >= 16:
            raise NotImplementedError('partial occupancy-grid update (iter_density >= 16) is a training-only branch (SURVEY.md §8 f2)')
        with torch.no_grad():
            variant = decoder.fused_variant()
            planes = R.pack_planes(code.detach(), variant)
            D.update_extra_state(variant, planes, tuple(code.shape[-2:]), decoder.packed_blob(), density_grid, density_bitfield,
                                 jitter=jitter, density_thresh=density_thresh, decay=decay, grid_size=self.grid_size,
                                 bound=float(decoder.bound))

    def get_density(self, decoder, code, cfg=dict(), jitters=None):
        variant = decoder.fused_variant()
        planes = R.pack_planes(code, variant)
        return D.get_density(variant, planes, tuple(code.shape[-2:]), decoder.packed_blob(), code.size(0),
                             density_thresh=cfg.get('density_thresh', 0.01), density_step=cfg.get('density_step', 8),
                             grid_size=self.grid_size, bound=float(decoder.bound), jitters=jitters)

    # ------------------------------------------------------------------ code optimisation by inverse rendering (base_nerf.py:403-492)
    def inverse_code(self, decoder, cond_imgs, cond_rays_o, cond_rays_d, dt_gamma=0, cfg=dict(), code_=None, density_grid=None,
                     density_bitfield=None, iter_density=None, code_optimizer=None, code_scheduler=None, prior_grad=None, show_pbar=False):
        """Adam on the pre-activation latent against the render loss (fused differentiable renderer).  With `prior_grad` the first thing
        each step does is overwrite the latent's .grad with it, so the render gradient ADDS to the diffusion-prior gradient."""
        device = next(self.parameters()).device
        prev = decoder.training
        decoder.train(True)
        with module_requires_grad(decoder, False), torch.enable_grad():
            n_inverse_steps, n_inverse_rays = cfg.get('n_inverse_steps', 1000), cfg.get('n_inverse_rays', 4096)
            assert n_inverse_steps > 0
            num_scenes = cond_imgs.size(0)
            num_scene_pixels = cond_imgs[0].numel() // 3
            raybatch_inds, num_raybatch = self.get_raybatch_inds(cond_imgs, n_inverse_rays)
            # defaults: fresh latent / empty occupancy state / optimiser + schedule from cfg
            code_ = self.get_init_code_(num_scenes, device=device) if code_ is None else code_
            density_grid = self.get_init_density_grid(num_scenes, device) if density_grid is None else density_grid
            density_bitfield = self.get_init_density_bitfield(num_scenes, device) if density_bitfield is None else density_bitfield
            iter_density = 0 if iter_density is None else iter_density
            if code_optimizer is None:
                assert code_scheduler is None
                code_optimizer = self.build_optimizer(code_, cfg)
            code_scheduler = self.build_scheduler(code_optimizer, cfg) if code_scheduler is None else code_scheduler
            optimizers = code_optimizer if isinstance(code_optimizer, list) else [code_optimizer]
            schedulers = [] if code_scheduler is None else (code_scheduler if isinstance(code_scheduler, list) else [code_scheduler])
            for step in range(n_inverse_steps):
                code = self.code_activation(torch.stack(code_, dim=0) if isinstance(code_, list) else code_)
                if step % self.update_extra_interval == 0:
                    self.update_extra_state(decoder, code, density_grid, density_bitfield, iter_density,
                                            density_thresh=cfg.get('density_thresh', 0.01))
                inds = raybatch_inds[step % num_raybatch] if raybatch_inds is not None else None
                rays_o, rays_d, target_rgbs = self.ray_sample(cond_rays_o, cond_rays_d, cond_imgs, n_inverse_rays, sample_inds=inds)
                out_rgbs, loss, loss_dict = self.loss(decoder, code, density_bitfield, target_rgbs, rays_o, rays_d, dt_gamma,
                                                      scale_num_ray=num_scene_pixels, cfg=cfg)
                if prior_grad is not None:
                    if isinstance(code_, list):
                        for c, g in zip(code_, prior_grad):
                            c.grad.copy_(g)
                    else:
                        code_.grad.copy_(prior_grad)
                else:
                    for o in optimizers:
                        o.zero_grad()
                loss.backward()
                for o in optimizers:
                    o.step()
                for sch in schedulers:
                    sch.step()
        decoder.train(prev)
        return code.detach(), density_grid, density_bitfield, loss, loss_dict, out_rgbs, target_rgbs

    # ------------------------------------------------------------------ render (base_nerf.py:494-533)
    def render(self, decoder, code, density_bitfield, h, w, intrinsics, poses, cfg=dict()):
        """-> image [B,V,h,w,3] (background-blended), depth [B,V,h,w]; rays are generated inside the kernel (eval-mode fused renderer,
        whatever `decoder.training` is: the reference switches the decoder to eval for this call, base_nerf.py:495-496)."""
        N.require_cuda(code, density_bitfield, intrinsics, poses)
        num_scenes, num_imgs = poses.shape[0], poses.shape[1]
        dt_gamma_scale = cfg.get('dt_gamma_scale', 0.0)
        dt_gamma = None
        if dt_gamma_scale != 0:
            dt_gamma = dt_gamma_scale * 2 / (intrinsics[..., 0] + intrinsics[..., 1]).mean(dim=-1)
        variant = decoder.fused_variant()
        planes = R.pack_planes(code.detach(), variant)
        poses44 = poses
        if poses.shape[-2] == 3:
            poses44 = torch.cat([poses, poses.new_tensor([0, 0, 0, 1]).expand(*poses.shape[:-2], 1, 4)], dim=-2)
        out = R.render_fwd(variant, planes, tuple(code.shape[-2:]), density_bitfield.reshape(num_scenes, -1), decoder.packed_blob(),
                           poses=poses44, intrinsics=intrinsics, img_hw=(h, w), grid_size=self.grid_size, bound=float(decoder.bound),
                           min_near=float(decoder.min_near), max_steps=int(decoder.max_steps), bg_color=float(self.bg_color),
                           dt_gamma=dt_gamma, want_counts=False)
        return out['rgb'].reshape(num_scenes, num_imgs, h, w, 3), out['depth'].reshape(num_scenes, num_imgs, h, w)

    def _lpips_metric(self):
        """the LPIPS network of `self.lpips` (an instance, or a list holding one), built from the default weight files on first use;
        None when the metric is off or the files are missing (warned once)"""
        from . import lpips as LP
        if self.lpips is None or isinstance(self.lpips, LP.LPIPS):
            return self.lpips
        if len(self.lpips) == 0:
            if not LP.default_files_exist():
                if not self._lpips_missing_warned:
                    vgg, lin = LP.default_paths()
                    warnings.warn(f'test_lpips is not reported: LPIPS weights not found ({vgg}, {lin or "lpips package not installed"}); '
                                  'put an ssdnerf_b200.lpips.LPIPS(vgg_path, lin_path) in model.lpips to enable it')
                    self._lpips_missing_warned = True
                return None
            self.lpips.append(LP.LPIPS())
        return self.lpips[0]

    def eval_and_viz(self, data, decoder, code, density_bitfield, viz_dir=None, cfg=dict()):
        """base_nerf.py:535-673: render, clamp, 8-bit rounding -> `pred_imgs`.  With `test_imgs` in `data` the log holds `test_psnr`
        (metrics.py:52-55), `test_ssim` (skimage's SSIM, `metrics.ssim`) and, when `use_lpips_metric` is on and LPIPS weights are available
        (`self.lpips`, see ssdnerf_b200/lpips.py), `test_lpips`: means over all scenes and views.  Without weights `test_lpips` is left out
        with one warning.  With `viz_dir` (or cfg['viz_dir']) the reference's PNG files are written there (ssdnerf_b200/viz.py): one per
        view, real | prediction when `test_imgs` are given (named from the per-image metrics, after deleting that view's older files),
        then `decoder.visualize` of the codes and of `init_code` as `000_mean`."""
        h, w = cfg['img_size']
        image, depth = self.render(decoder, code, density_bitfield, h, w, data['test_intrinsics'], data['test_poses'], cfg=cfg)
        num_scenes, num_imgs = image.shape[:2]
        pred_imgs = image.permute(0, 1, 4, 2, 3).reshape(num_scenes * num_imgs, 3, h, w).clamp(min=0, max=1)
        pred_imgs = torch.round(pred_imgs * 255) / 255
        log_vars = dict()
        psnr = ssim = lpips = None
        if data.get('test_imgs') is not None:
            target = data['test_imgs'].permute(0, 1, 4, 2, 3).reshape(num_scenes * num_imgs, 3, h, w)
            mse = (pred_imgs - target).square().flatten(1).mean(dim=1)
            psnr = -10 * torch.log10(mse + 1e-6)          # eval_psnr (lib/core/evaluation/metrics.py:52-55): eps 1e-6
            log_vars.update(test_psnr=float(psnr.mean()))
            # channels-last views of the same values for the kernels: pred_imgs keeps `image`'s memory order, so this permute copies nothing
            pred_cl = pred_imgs.permute(0, 2, 3, 1).contiguous()
            target_cl = data['test_imgs'].reshape(num_scenes * num_imgs, h, w, 3).contiguous()
            ssim = M.ssim(pred_cl, target_cl)
            log_vars.update(test_ssim=float(ssim.mean()))
            lp = self._lpips_metric()
            if lp is not None:
                lpips = lp(pred_cl, target_cl)
                log_vars.update(test_lpips=float(lpips.mean()))
        if viz_dir is None:
            viz_dir = cfg.get('viz_dir', None)
        if viz_dir is not None:
            self._write_viz(viz_dir, data, decoder, code, image, psnr, ssim, lpips, cfg)
        return log_vars, pred_imgs.reshape(num_scenes, num_imgs, 3, h, w)

    def _write_viz(self, viz_dir, data, decoder, code, image, psnr, ssim, lpips, cfg):
        """base_nerf.py:574-608 on the device encoder: view files, then the triplane maps"""
        num_scenes, num_imgs, h, w, _ = image.shape
        os.makedirs(viz_dir, exist_ok=True)
        test_imgs = data.get('test_imgs') if not cfg.get('skip_eval', False) else None      # base_nerf.py:542: skip_eval -> no real half
        names, bases = V.view_file_names(data['scene_name'], num_imgs, data.get('test_img_paths') if test_imgs is not None else None,
                                         None if psnr is None else psnr.tolist(), None if ssim is None else ssim.tolist(),
                                         None if lpips is None else lpips.tolist())
        real = None if test_imgs is None else test_imgs.reshape(num_scenes * num_imgs, h, w, 3)
        V.write_view_files(viz_dir, names, bases, V.encode_png(pred=image.reshape(num_scenes * num_imgs, h, w, 3), real=real))
        code_range = cfg.get('clip_range', [-1, 1])
        decoder.visualize(code, data['scene_name'], viz_dir, code_range=code_range)
        if self.init_code is not None:
            decoder.visualize(self.init_code[None], ['000_mean'], viz_dir, code_range=code_range)

    def mean_ema_update(self, code):
        if self.init_code is None:
            return
        mean_code = code.detach().mean(dim=0)
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.all_reduce(mean_code)
            mean_code /= torch.distributed.get_world_size()
        self.init_code.lerp_(mean_code, self.mean_ema_momentum)

    def train_step(self, data, optimizer, running_status=None):
        raise NotImplementedError('BaseNeRF has no train_step (the reference defines it on MultiSceneNeRF / DiffusionNeRF)')


# --------------------------------------------------------------------------------------------------------------------- MultiSceneNeRF
def _dist_info():
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_rank(), torch.distributed.get_world_size()
    return 0, 1


def _average_grads_across_ranks(module):
    """what the reference gets from wrapping the decoder in DistributedDataParallel (apis/train.py): the shared decoder's gradient
    is the mean over ranks, one flat all-reduce; per-scene latents are rank-private and are not reduced."""
    rank, ws = _dist_info()
    if ws == 1:
        return
    grads = [p.grad for p in module.parameters() if p.grad is not None]
    if not grads:
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    torch.distributed.all_reduce(flat)
    flat /= ws
    o = 0
    for g in grads:
        g.copy_(flat[o:o + g.numel()].view_as(g))
        o += g.numel()


@MODELS.register_module()
class MultiSceneNeRF(BaseNeRF):
    """multiscene_nerf.py:32-252 -- stage-1 auto-decoder: per-scene latents + shared decoder, trained jointly by `train_step` on the
    fused differentiable renderer (code AND decoder-weight gradients from one backward launch); `val_step` renders stored scenes or
    fits codes to `cond_imgs`.  Scene state between visits lives in `scene_cache.SceneCache`."""

    def __init__(self, *args, cache_size=0, cache_16bit=False, num_file_writers=0, **kwargs):
        super().__init__(*args, **kwargs)
        self.cache_size, self.cache_16bit, self.num_file_writers = cache_size, cache_16bit, num_file_writers
        rank, ws = _dist_info()
        self.scene_cache = SceneCache(cache_size, rank, ws, half=cache_16bit, num_file_writers=num_file_writers)

    # the reference exposes the raw dict / flag; keep them readable under the same names
    @property
    def cache(self):
        return self.scene_cache.entries

    @property
    def cache_loaded(self):
        return self.scene_cache.loaded

    def load_cache(self, data):
        """multiscene_nerf.py:74-134 -> (code_list_, code_optimizers, density_grid [B,G^3], density_bitfield [B,G^3/8])"""
        device = next(self.parameters()).device
        sc = self.scene_cache
        if sc.entries is not None:
            if not sc.loaded:
                src = self.train_cfg.get('cache_load_from', None)
                if src is not None:
                    sc.load_dir(src)
                sc.loaded = True
            states = [sc.get(i) for i in data['scene_id']]
        elif 'code' in data:
            states = data['code']
        else:
            states = [None] * len(data['scene_id'])
        code_list_, grids, bitfields = [], [], []
        for st in states:
            if st is None:
                code_list_.append(self.get_init_code_(None, device))
                grids.append(self.get_init_density_grid(None, device))
                bitfields.append(self.get_init_density_bitfield(None, device))
                continue
            par = st['param']
            if 'code_' in par:
                code_ = par['code_'].to(device=device, dtype=torch.float32, non_blocking=True, copy=True)      # never alias the cache entry
            else:      # only the activated code was stored: invert the activation (lossy at the clip range, as the reference warns)
                code_ = self.code_activation.inverse(par['code'].to(device=device, dtype=torch.float32))
            code_list_.append(code_.requires_grad_(True))
            grids.append(par['density_grid'].to(device, non_blocking=True))
            bitfields.append(par['density_bitfield'].to(device, non_blocking=True))
        code_optimizers = self.build_optimizer(code_list_, self.train_cfg)
        for opt, st in zip(code_optimizers, states):
            if st is not None and st.get('optimizer') is not None:
                restore_optimizer_state(opt, st['optimizer'])
        return code_list_, code_optimizers, torch.stack(grids), torch.stack(bitfields)

    def save_cache(self, code_list_, code_optimizers, density_grid, density_bitfield, scene_id, scene_name):
        """multiscene_nerf.py:136-183"""
        save_dir = self.train_cfg.get('save_dir', None)
        if save_dir is not None:
            os.makedirs(save_dir, exist_ok=True)
        for ind, code_ in enumerate(code_list_):
            self.scene_cache.put(scene_id[ind], scene_name[ind], code_.data, density_grid[ind], density_bitfield[ind],
                                 code_optimizers[ind].state_dict(), save_dir=save_dir)

    def train_step(self, data, optimizer, running_status=None):
        """multiscene_nerf.py:185-252: optional extra code-only steps, then ONE joint step of the scene latents (their own
        optimizers) and the decoder (`optimizer['decoder']`) on `n_decoder_rays` random rays per scene."""
        code_list_, code_optimizers, density_grid, density_bitfield = self.load_cache(data)
        cond_imgs, cond_intrinsics, cond_poses = data['cond_imgs'], data['cond_intrinsics'], data['cond_poses']
        num_scenes, num_imgs, h, w, _ = cond_imgs.size()
        cond_rays_o, cond_rays_d = R.get_cam_rays(cond_poses, cond_intrinsics, h, w)
        dt_gamma = self.train_cfg.get('dt_gamma_scale', 0.0) / cond_intrinsics[..., :2].mean(dim=(-2, -1))

        extra = self.train_cfg.get('extra_scene_step', 0)
        if extra > 0:
            cfg = dict(self.train_cfg, n_inverse_steps=extra)
            self.inverse_code(self.decoder, cond_imgs, cond_rays_o, cond_rays_d, dt_gamma=dt_gamma, cfg=cfg, code_=code_list_,
                              density_grid=density_grid, density_bitfield=density_bitfield, code_optimizer=code_optimizers)

        for o in code_optimizers:
            o.zero_grad()
        optimizer['decoder'].zero_grad()
        code = self.code_activation(torch.stack(code_list_, dim=0), update_stats=True)
        self.update_extra_state(self.decoder, code, density_grid, density_bitfield, 0,
                                density_thresh=self.train_cfg.get('density_thresh', 0.01))
        loss, log_vars, out_rgbs, target_rgbs = self.loss_decoder(self.decoder, code, density_bitfield, cond_rays_o, cond_rays_d,
                                                                  cond_imgs, dt_gamma, cfg=self.train_cfg)
        loss.backward()
        log_vars.update(loss=float(loss.detach()))
        _average_grads_across_ranks(self.decoder)
        optimizer['decoder'].step()
        for o in code_optimizers:
            o.step()

        self.save_cache(code_list_, code_optimizers, density_grid, density_bitfield, data['scene_id'], data['scene_name'])

        with torch.no_grad():
            self.mean_ema_update(code)
            mse = (out_rgbs.reshape(num_scenes, -1) - target_rgbs.reshape(num_scenes, -1)).square().mean(dim=1)
            log_vars.update(train_psnr=float((-10 * torch.log10(mse + 1e-6)).mean()),
                            code_rms=float(code.square().flatten(1).mean().sqrt()))
            if data.get('test_imgs', None) is not None:
                log_vars.update(self.eval_and_viz(data, self.decoder, code, density_bitfield, cfg=self.train_cfg)[0])
        return dict(log_vars=log_vars, num_samples=num_scenes)

    def val_step(self, data, viz_dir=None, show_pbar=False, **kwargs):
        """multiscene_nerf.py:185-252: stored scenes are rendered; otherwise the codes are fitted to `cond_imgs` by inverse rendering"""
        decoder = self.decoder_ema if self.decoder_use_ema else self.decoder
        if 'code' in data:
            code, density_grid, density_bitfield = self.load_scene(data, load_density=True)
        elif 'cond_imgs' in data:
            cond_imgs, cond_intrinsics, cond_poses = data['cond_imgs'], data['cond_intrinsics'], data['cond_poses']
            num_scenes, num_imgs, h, w, _ = cond_imgs.size()
            cond_rays_o, cond_rays_d = R.get_cam_rays(cond_poses, cond_intrinsics, h, w)
            dt_gamma = self.test_cfg.get('dt_gamma_scale', 0.0) / cond_intrinsics[..., :2].mean(dim=(-2, -1))
            code, density_grid, density_bitfield, _, _, _, _ = self.inverse_code(
                decoder, cond_imgs, cond_rays_o, cond_rays_d, dt_gamma=dt_gamma, cfg=self.test_cfg, show_pbar=show_pbar)
        else:
            raise ValueError('MultiSceneNeRF.val_step needs stored scenes (`code`) or conditioning views (`cond_imgs`)')
        with torch.no_grad():
            if 'test_poses' in data:
                log_vars, pred_imgs = self.eval_and_viz(data, decoder, code, density_bitfield, viz_dir=viz_dir, cfg=self.test_cfg)
            else:
                log_vars, pred_imgs = dict(), None
        save_dir = self.test_cfg.get('save_dir', None)
        if save_dir is not None:
            self.save_scene(save_dir, code, density_grid, density_bitfield, data['scene_name'])
        return dict(log_vars=log_vars, num_samples=len(data['scene_name']), pred_imgs=pred_imgs)


# --------------------------------------------------------------------------------------------------------------------- DiffusionNeRF
@MODELS.register_module()
class DiffusionNeRF(MultiSceneNeRF):
    """diffusion_nerf.py:13-469"""

    def __init__(self, *args, diffusion=dict(type='GaussianDiffusion'), diffusion_use_ema=True, freeze_decoder=True, image_cond=False,
                 code_permute=None, code_reshape=None, autocast_dtype=None, **kwargs):
        super().__init__(*args, **kwargs)
        diffusion = dict(diffusion)
        diffusion.update(train_cfg=self.train_cfg, test_cfg=self.test_cfg)
        self.diffusion = build_module(diffusion)
        self.diffusion_use_ema = diffusion_use_ema
        if self.diffusion_use_ema:
            self.diffusion_ema = deepcopy(self.diffusion)
        self.freeze_decoder = freeze_decoder
        if self.freeze_decoder:
            self.decoder.requires_grad_(False)
            if self.decoder_use_ema:
                self.decoder_ema.requires_grad_(False)
        self.image_cond = image_cond
        self.code_permute = code_permute
        self.code_reshape = code_reshape
        self.code_reshape_inv = [self.code_size[axis] for axis in self.code_permute] if code_permute is not None else self.code_size
        self.code_permute_inv = [self.code_permute.index(axis) for axis in range(len(self.code_permute))] \
            if code_permute is not None else None
        # the reference wraps the sampler in torch.autocast(autocast_dtype); the native UNet always computes with fp16 operands /
        # fp32 accumulation, so the setting is accepted and has nothing left to switch
        self.autocast_dtype = autocast_dtype
        for key in self.test_cfg.get('override_cfg', dict()):
            self.train_cfg_backup[key] = rgetattr(self, key)

    # ------------------------------------------------------------------ code <-> diffusion layout (diffusion_nerf.py:50-64)
    def train_step(self, data, optimizer, running_status=None):
        """diffusion_nerf.py:66-189.  One iteration of single-stage training (latents + decoder + denoiser), of stage 2 (denoiser on
        stored scenes: no `optimizer` entry in train_cfg, `code` in data) or of any mix the config's optimizers select:
        diffusion loss -> denoiser step (UNet weight gradients: unet_train.py) with the prior gradient landing on the latents ->
        `extra_scene_step` render-loss Adam steps that START from that prior gradient -> joint render step of latents / decoder ->
        cache write-back.  `optimizer`: dict with keys 'diffusion*' and optionally 'decoder' (the reference's runner builds it)."""
        diffusion = self.diffusion
        decoder = self.decoder_ema if self.freeze_decoder and self.decoder_use_ema else self.decoder
        num_scenes = len(data['scene_id'])
        extra_scene_step = self.train_cfg.get('extra_scene_step', 0)
        if 'optimizer' in self.train_cfg:
            code_list_, code_optimizers, density_grid, density_bitfield = self.load_cache(data)
            code = self.code_activation(torch.stack(code_list_, dim=0), update_stats=True)
        else:
            assert 'code' in data
            code, density_grid, density_bitfield = self.load_scene(data, load_density='decoder' in optimizer)
            code_list_, code_optimizers = [], []
        diffusion_opts = [v for k, v in optimizer.items() if k.startswith('diffusion')]
        for o in diffusion_opts + code_optimizers:
            o.zero_grad()
        if 'decoder' in optimizer:
            optimizer['decoder'].zero_grad()

        has_views = 'cond_imgs' in data
        if has_views:
            cond_imgs, cond_intrinsics, cond_poses = data['cond_imgs'], data['cond_intrinsics'], data['cond_poses']
            num_scenes, num_imgs, h, w, _ = cond_imgs.size()
            cond_rays_o, cond_rays_d = R.get_cam_rays(cond_poses, cond_intrinsics, h, w)
            dt_gamma = self.train_cfg.get('dt_gamma_scale', 0.0) / cond_intrinsics[..., :2].mean(dim=(-2, -1))
            if self.image_cond:
                raise NotImplementedError('image_cond training (concat_cond) is unused by every shipped config and not built')

        loss_diffusion, log_vars = diffusion(self.code_diff_pr(code), concat_cond=None, return_loss=True,
                                             x_t_detach=self.train_cfg.get('x_t_detach', False), cfg=self.train_cfg)
        loss_diffusion.backward()
        _average_grads_across_ranks(diffusion)
        for o in diffusion_opts:
            o.step()

        prior_grad = None
        if extra_scene_step > 0:
            assert len(code_optimizers) > 0
            prior_grad = [c.grad.detach().clone() for c in code_list_]
            cfg = dict(self.train_cfg, n_inverse_steps=extra_scene_step)
            code, _, _, _, loss_dict_decoder, _, _ = self.inverse_code(
                decoder, cond_imgs, cond_rays_o, cond_rays_d, dt_gamma=dt_gamma, cfg=cfg, code_=code_list_, density_grid=density_grid,
                density_bitfield=density_bitfield, code_optimizer=code_optimizers, prior_grad=prior_grad)
            log_vars.update({k: float(v) for k, v in loss_dict_decoder.items()})

        if 'decoder' in optimizer or len(code_optimizers) > 0:
            if len(code_optimizers) > 0:
                code = self.code_activation(torch.stack(code_list_, dim=0))
            self.update_extra_state(decoder, code, density_grid, density_bitfield, 0, density_thresh=self.train_cfg.get('density_thresh', 0.01))
            loss_decoder, log_vars_decoder, out_rgbs, target_rgbs = self.loss_decoder(
                decoder, code, density_bitfield, cond_rays_o, cond_rays_d, cond_imgs, dt_gamma, cfg=self.train_cfg)
            log_vars.update(log_vars_decoder)
            if prior_grad is not None:
                for c, g in zip(code_list_, prior_grad):
                    c.grad.copy_(g)
            loss_decoder.backward()
            if 'decoder' in optimizer:
                _average_grads_across_ranks(decoder)
                optimizer['decoder'].step()
            for o in code_optimizers:
                o.step()
            if len(code_optimizers) > 0:
                self.save_cache(code_list_, code_optimizers, density_grid, density_bitfield, data['scene_id'], data['scene_name'])
            with torch.no_grad():
                if len(code_optimizers) > 0:
                    self.mean_ema_update(code)
                mse = (out_rgbs.reshape(num_scenes, -1) - target_rgbs.reshape(num_scenes, -1)).square().mean(dim=1)
                log_vars.update(train_psnr=float((-10 * torch.log10(mse + 1e-6)).mean()),
                                code_rms=float(code.square().flatten(1).mean().sqrt()))
                if data.get('test_imgs', None) is not None:
                    log_vars.update(self.eval_and_viz(data, self.decoder, code, density_bitfield, cfg=self.train_cfg)[0])
            log_vars.update(loss_decoder=float(loss_decoder.detach()))
        return dict(log_vars=log_vars, num_samples=num_scenes)

    def code_diff_pr(self, code):
        """scene code [B, *code_size] -> the denoiser's layout: optional axis permutation (batch axis kept), then reshape"""
        out = code if self.code_permute is None else code.permute(0, *(a + 1 for a in self.code_permute))
        return out if self.code_reshape is None else out.reshape(code.size(0), *self.code_reshape)

    def code_diff_pr_inv(self, code_diff):
        out = code_diff if self.code_reshape is None else code_diff.reshape(code_diff.size(0), *self.code_reshape_inv)
        return out if self.code_permute_inv is None else out.permute(0, *(a + 1 for a in self.code_permute_inv))

    def _modules_for_eval(self):
        return (self.diffusion_ema if self.diffusion_use_ema else self.diffusion,
                self.decoder_ema if self.decoder_use_ema else self.decoder)

    # ------------------------------------------------------------------ unconditional generation (diffusion_nerf.py:191-239)
    def val_uncond(self, data, show_pbar=False, **kwargs):
        diffusion, decoder = self._modules_for_eval()
        num_batches = len(data['scene_id'])
        noise = data.get('noise', None)
        if noise is None:
            noise = torch.randn((num_batches, *self.code_size), device=next(self.parameters()).device)
        with torch.no_grad():
            code_out = diffusion(self.code_diff_pr(noise), return_loss=False, show_pbar=show_pbar, **kwargs)
        code_list = code_out if isinstance(code_out, list) else [code_out]          # save_intermediates -> [x0, x_t, x0, x_t, ...]
        n_inverse_steps = self.test_cfg.get('n_inverse_steps', 0)
        codes, grids, bits = [], [], []
        for step_id, code in enumerate(code_list):
            code = self.code_diff_pr_inv(code).contiguous()
            if n_inverse_steps > 0 and step_id == len(code_list) - 1:
                # refine the sample against the diffusion prior alone (diffusion_nerf.py:213-229)
                with module_requires_grad(diffusion, False), torch.enable_grad():
                    code_ = self.code_activation.inverse(code).requires_grad_(True)
                    optimizer = self.build_optimizer(code_, self.test_cfg)
                    scheduler = self.build_scheduler(optimizer, self.test_cfg)
                    for _ in range(n_inverse_steps):
                        optimizer.zero_grad()
                        loss, _ = diffusion(self.code_diff_pr(self.code_activation(code_)), return_loss=True, cfg=self.test_cfg)
                        loss.backward()
                        optimizer.step()
                        if scheduler is not None:
                            scheduler.step()
                code = self.code_activation(code_).detach()
            with torch.no_grad():
                density_grid, density_bitfield = self.get_density(decoder, code, cfg=self.test_cfg)
            codes.append(code); grids.append(density_grid); bits.append(density_bitfield)
        if isinstance(code_out, list):
            return codes, grids, bits
        return codes[-1], grids[-1], bits[-1]

    def _cond_rays(self, data):
        cond_imgs, cond_intrinsics, cond_poses = data['cond_imgs'], data['cond_intrinsics'], data['cond_poses']
        num_scenes, num_imgs, h, w, _ = cond_imgs.size()
        cond_rays_o, cond_rays_d = R.get_cam_rays(cond_poses, cond_intrinsics, h, w)          # native: refuses CPU tensors
        dt_gamma = self.test_cfg.get('dt_gamma_scale', 0.0) / cond_intrinsics[..., :2].mean(dim=(-2, -1))
        if self.image_cond:
            raise NotImplementedError('image-conditioned (concat_cond) denoisers are not used by the shipped configs')
        return cond_imgs, cond_rays_o, cond_rays_d, dt_gamma

    # ------------------------------------------------------------------ guided generation (diffusion_nerf.py:241-311)
    def val_guide(self, data, **kwargs):
        """Render-loss guided DDIM (+ langevin).  `test_cfg.grad_through_unet` (default True, as in the reference) takes the guidance
        gradient w.r.t. x_t through the denoiser; False takes it w.r.t. x_0."""
        diffusion, decoder = self._modules_for_eval()
        device = next(self.parameters()).device
        cond_imgs, cond_rays_o, cond_rays_d, dt_gamma = self._cond_rays(data)
        num_scenes = cond_imgs.size(0)
        prev = decoder.training
        decoder.train(True)
        try:
            with module_requires_grad(diffusion, False), module_requires_grad(decoder, False):
                n_inverse_rays = self.test_cfg.get('n_inverse_rays', 4096)
                raybatch_inds, num_raybatch = self.get_raybatch_inds(cond_imgs, n_inverse_rays)
                density_grid = torch.zeros((num_scenes, self.grid_size ** 3), device=device)
                density_bitfield = torch.zeros((num_scenes, self.grid_size ** 3 // 8), dtype=torch.uint8, device=device)
                state = dict(step=0)

                def grad_guide_fn(x_0_pred):
                    code_pred = self.code_diff_pr_inv(x_0_pred)
                    self.update_extra_state(decoder, code_pred, density_grid, density_bitfield, 0,
                                            density_thresh=self.test_cfg.get('density_thresh', 0.01))
                    inds = raybatch_inds[state['step'] % num_raybatch] if raybatch_inds is not None else None
                    rays_o, rays_d, target_rgbs = self.ray_sample(cond_rays_o, cond_rays_d, cond_imgs, n_inverse_rays, sample_inds=inds)
                    _, loss, _ = self.loss(decoder, code_pred, density_bitfield, target_rgbs, rays_o, rays_d, dt_gamma,
                                           scale_num_ray=target_rgbs.size(1), cfg=self.test_cfg)
                    state['step'] += 1
                    return loss * num_scenes

                noise = data.get('noise', None)
                if noise is None:
                    noise = torch.randn((num_scenes, *self.code_size), device=device)
                code = diffusion(self.code_diff_pr(noise), return_loss=False, grad_guide_fn=grad_guide_fn, **kwargs)
        finally:
            decoder.train(prev)
        return self.code_diff_pr_inv(code), density_grid, density_bitfield

    # ------------------------------------------------------------------ code optimisation with the diffusion prior (diffusion_nerf.py:313-404)
    def val_optim(self, data, code_=None, density_grid=None, density_bitfield=None, show_pbar=False, **kwargs):
        """K_out outer steps: gradient of the diffusion loss w.r.t. the latent (UNet input-gradient pass), then either
        `extra_scene_step`+1 inner render-loss steps that start from that prior gradient (`inverse_code(prior_grad=...)`) or one joint
        step.  Optimiser = torch.optim as configured in test_cfg (the reference does the same; it is host-side plumbing)."""
        diffusion, decoder = self._modules_for_eval()
        cond_imgs, cond_rays_o, cond_rays_d, dt_gamma = self._cond_rays(data)
        num_scenes = cond_imgs.size(0)
        prev = decoder.training
        decoder.train(True)
        extra_scene_step = self.test_cfg.get('extra_scene_step', 0)
        n_inverse_steps = self.test_cfg.get('n_inverse_steps', 100)
        assert n_inverse_steps > 0
        try:
            with module_requires_grad(diffusion, False), module_requires_grad(decoder, False), torch.enable_grad():
                if code_ is None:
                    code_ = self.get_init_code_(num_scenes, cond_imgs.device)
                if density_grid is None:
                    density_grid = self.get_init_density_grid(num_scenes, cond_imgs.device)
                if density_bitfield is None:
                    density_bitfield = self.get_init_density_bitfield(num_scenes, cond_imgs.device)
                optimizer = self.build_optimizer(code_, self.test_cfg)
                scheduler = self.build_scheduler(optimizer, self.test_cfg)
                for step in range(n_inverse_steps):
                    optimizer.zero_grad()
                    code = self.code_activation(code_)
                    loss, _ = diffusion(self.code_diff_pr(code), return_loss=True, x_t_detach=self.test_cfg.get('x_t_detach', False),
                                        cfg=self.test_cfg, **kwargs)
                    loss.backward()
                    if extra_scene_step > 0:
                        cfg = dict(self.test_cfg)
                        cfg['n_inverse_steps'] = extra_scene_step + 1
                        self.inverse_code(decoder, cond_imgs, cond_rays_o, cond_rays_d, dt_gamma=dt_gamma, cfg=cfg, code_=code_,
                                          density_grid=density_grid, density_bitfield=density_bitfield, code_optimizer=optimizer,
                                          code_scheduler=scheduler, prior_grad=code_.grad.data.clone())
                    else:
                        code = self.code_activation(code_)
                        loss_decoder, _, _, _ = self.loss_decoder(decoder, code, density_bitfield, cond_rays_o, cond_rays_d, cond_imgs,
                                                                  dt_gamma, cfg=self.test_cfg)
                        loss_decoder.backward()
                        optimizer.step()
                        if scheduler is not None:
                            scheduler.step()
        finally:
            decoder.train(prev)
        return self.code_activation(code_).detach(), density_grid, density_bitfield

    # ------------------------------------------------------------------ entry point (diffusion_nerf.py:406-469)
    def val_step(self, data, viz_dir=None, viz_dir_guide=None, **kwargs):
        _, decoder = self._modules_for_eval()
        with torch.no_grad():
            if 'code' in data:
                code, density_grid, density_bitfield = self.load_scene(data, load_density=True)
            elif 'cond_imgs' in data:
                cond_mode = self.test_cfg.get('cond_mode', 'guide')
                if cond_mode == 'guide':
                    code, density_grid, density_bitfield = self.val_guide(data, **kwargs)
                elif cond_mode == 'optim':
                    code, density_grid, density_bitfield = self.val_optim(data, **kwargs)
                elif cond_mode == 'guide_optim':
                    code, density_grid, density_bitfield = self.val_guide(data, **kwargs)
                    if viz_dir_guide is not None and 'test_poses' in data:
                        self.eval_and_viz(data, decoder, code, density_bitfield, viz_dir=viz_dir_guide, cfg=self.test_cfg)
                    code, density_grid, density_bitfield = self.val_optim(
                        data, code_=self.code_activation.inverse(code).requires_grad_(True), density_grid=density_grid,
                        density_bitfield=density_bitfield, **kwargs)
                else:
                    raise AttributeError(f'unknown cond_mode {cond_mode}')
            else:
                code, density_grid, density_bitfield = self.val_uncond(data, **kwargs)
            if isinstance(code, list):          # save_intermediates: evaluate the final sample
                code, density_grid, density_bitfield = code[-1], density_grid[-1], density_bitfield[-1]
            if 'test_poses' in data:
                log_vars, pred_imgs = self.eval_and_viz(data, decoder, code, density_bitfield, viz_dir=viz_dir, cfg=self.test_cfg)
            else:
                log_vars, pred_imgs = dict(), None
                if viz_dir is None:
                    viz_dir = self.test_cfg.get('viz_dir', None)
                if viz_dir is not None:          # diffusion_nerf.py:442-451: the sampled codes' triplane maps alone
                    os.makedirs(viz_dir, exist_ok=True)
                    decoder.visualize(code, data['scene_name'], viz_dir, code_range=self.test_cfg.get('clip_range', [-1, 1]))
        save_dir = self.test_cfg.get('save_dir', None)
        if save_dir is not None:
            self.save_scene(save_dir, code, density_grid, density_bitfield, data['scene_name'])
            if self.test_cfg.get('save_mesh', False):
                self.save_mesh(save_dir, decoder, code, data['scene_name'], self.test_cfg.get('mesh_resolution', 256),
                               self.test_cfg.get('mesh_threshold', 10))
        names = data['scene_name'] if 'scene_name' in data else data['scene_id']
        return dict(log_vars=log_vars, num_samples=len(names), pred_imgs=pred_imgs)
