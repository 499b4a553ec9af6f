"""`VolumeRenderer` / `TriPlaneDecoder` -- the reference's decoder plugin, backed by the fused sm_90a renderer.

Plugin surface of lib/models/decoders/base_volume_renderer.py:11-133 and triplane_decoder.py:15-184: registered name
`TriPlaneDecoder`, constructor kwargs, state-dict keys (`aabb`, `base_net.0.*`, `density_net.0.*`, `dir_net.0.*`,
`color_net.{0,2}.*`), `forward(rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh,
return_loss)` returning `dict(weights_sum, depth, image)` as per-scene lists in eval mode, `point_decode`,
`point_density_decode`, attributes `bound / min_near / max_steps / aabb`.

eval mode (`self.training == False`): ONE fused launch sequence (csrc/render.cu, csrc/render_p3.cu, csrc/render_s2.cu).
train mode: decoder of the shipped-config shape -> fused differentiable renderer (csrc/render_train.cu): gradient w.r.t. the
code (guidance / code optimisation with a frozen decoder, diffusion_nerf.py:273) and, when the decoder is trainable (stage-1
auto-decoder training, multiscene_nerf.py:159-252), w.r.t. its weights.  `point_decode` / `point_density_decode` are one native launch (csrc/point_decode.cu).
"""
import os

import torch
import torch.nn as nn

from . import _lib as N
from . import renderer as R
from . import viz as V
from .activation import TruncExp
from .registry import MODULES, build_module
from .shencoder import SHEncoder


class _FusedTrainRender(torch.autograd.Function):
    """march + decode + composite as ONE differentiable op: gradient w.r.t. `code` [B,3,6,H,W] and, when any of them requires
    one, w.r.t. the decoder parameters (`params`, in renderer.DEC_P_PARAM_ORDER; `blob` is their packed copy)."""

    @staticmethod
    def forward(ctx, code, rays_o, rays_d, bitfield, blob, noises, dt_gamma, cfg, *params):
        planes = R.pack_planes(code, R.DEC_P)
        hw = tuple(code.shape[-2:])
        out = R.render_train_fwd(planes, hw, bitfield, blob, rays_o, rays_d, noises=noises, dt_gamma=dt_gamma, **cfg)
        ctx.save_for_backward(planes, rays_o, rays_d, bitfield, blob, noises, dt_gamma, out['weights_sum'], out['image'])
        ctx.hw, ctx.cfg = hw, cfg
        ctx.mark_non_differentiable(out['depth'])      # the reference's K8 has no depth gradient either (raymarching.py:333-343)
        return out['weights_sum'], out['depth'], out['image']

    @staticmethod
    def backward(ctx, grad_ws, grad_depth, grad_image):
        planes, rays_o, rays_d, bitfield, blob, noises, dt_gamma, ws, image = ctx.saved_tensors
        if grad_image is None:
            grad_image = torch.zeros_like(image)
        want = any(ctx.needs_input_grad[8:])
        out = R.render_train_bwd(planes, ctx.hw, bitfield, blob, rays_o, rays_d, ws, image, grad_ws, grad_image,
                                 noises=noises, dt_gamma=dt_gamma, want_decoder_grad=want, **ctx.cfg)
        if not want:
            return (out,) + (None,) * (7 + len(ctx.needs_input_grad[8:]))
        return (out[0],) + (None,) * 7 + R.unpack_decoder_blob_grad(out[1])


class VolumeRenderer(nn.Module):
    def __init__(self, bound=1, min_near=0.2, bg_radius=-1, max_steps=256, decoder_reg_loss=None):
        super().__init__()
        self.bound = bound
        self.min_near = min_near
        self.bg_radius = bg_radius
        self.max_steps = max_steps
        self.decoder_reg_loss = build_module(decoder_reg_loss) if decoder_reg_loss is not None else None
        self.register_buffer('aabb', torch.FloatTensor([-bound, -bound, -bound, bound, bound, bound]))

    def point_decode(self, xyzs, dirs, code):
        raise NotImplementedError

    def point_density_decode(self, xyzs, code):
        raise NotImplementedError

    def loss(self):
        assert self.decoder_reg_loss is None
        return None


def _xavier_uniform_(m):
    nn.init.xavier_uniform_(m.weight, gain=1)
    nn.init.constant_(m.bias, 0)


@MODULES.register_module()
class TriPlaneDecoder(VolumeRenderer):
    activation_dict = {'relu': nn.ReLU, 'silu': nn.SiLU, 'softplus': nn.Softplus, 'trunc_exp': TruncExp}

    def __init__(self, *args, interp_mode='bilinear', base_layers=[3 * 32, 128], density_layers=[128, 1],
                 color_layers=[128, 128, 3], use_dir_enc=True, dir_layers=None, scene_base_size=None, scene_rand_dims=(0, 1),
                 activation='silu', sigma_activation='trunc_exp', sigmoid_saturation=0.001, code_dropout=0.0, flip_z=False, **kwargs):
        super().__init__(*args, **kwargs)
        color_layers = list(color_layers)
        self.interp_mode = interp_mode
        self.in_chn = base_layers[0]
        self.use_dir_enc = use_dir_enc
        self.scene_base = None
        if scene_base_size is not None:
            raise NotImplementedError('scene_base is unused by every reference config and not built')
        self.dir_encoder = SHEncoder() if use_dir_enc else None
        self.sigmoid_saturation = sigmoid_saturation
        act = self.activation_dict[activation.lower()]

        def mlp(layers, last=None):
            mods = []
            for i in range(len(layers) - 1):
                mods.append(nn.Linear(layers[i], layers[i + 1]))
                if i != len(layers) - 2:
                    mods.append(act())
            if last is not None:
                mods.append(last)
            return nn.Sequential(*mods)

        self.base_net = mlp(base_layers)
        self.base_activation = act()
        self.density_net = mlp(density_layers, self.activation_dict[sigma_activation.lower()]())
        self.dir_net = None
        if use_dir_enc:
            if dir_layers is not None:
                self.dir_net = mlp(dir_layers)
            else:
                color_layers[0] = color_layers[0] + 16
        self.color_net = mlp(color_layers, nn.Sigmoid())
        self.code_dropout = nn.Dropout2d(code_dropout) if code_dropout > 0 else None
        self.flip_z = flip_z
        self._fused_cfg = dict(interp_mode=interp_mode, activation=activation.lower(), sigma_activation=sigma_activation.lower(),
                               use_dir_enc=use_dir_enc, flip_z=flip_z, code_dropout=code_dropout)
        self._blob = None
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Linear):
                _xavier_uniform_(m)
        if self.dir_net is not None:
            nn.init.constant_(self.dir_net[-1].weight, 0)
            nn.init.constant_(self.dir_net[-1].bias, 0)

    # ------------------------------------------------------------------ fused path helpers
    def decoder_params(self):
        keys = ['base_net.0', 'density_net.0', 'color_net.0'] + (['dir_net.0'] if self.dir_net is not None else []) \
            + (['color_net.2'] if len([m for m in self.color_net if isinstance(m, nn.Linear)]) > 1 else [])
        sd = self.state_dict()
        return {k + s: sd[k + s] for k in keys for s in ('.weight', '.bias')}

    def fused_variant(self):
        c = self._fused_cfg
        if not (c['interp_mode'] == 'bilinear' and c['activation'] == 'silu' and c['sigma_activation'] == 'trunc_exp'
                and c['use_dir_enc'] and not c['flip_z']):
            raise N.SSDNeRFNativeError('fused renderer covers bilinear / SiLU / trunc_exp / SH-encoded decoders (every reference config)')
        return R.detect_variant(self.decoder_params())

    def refresh_weights(self):
        """drop the packed weight blob; needed only after parameter writes that bypass `Parameter._version` (`p.data...`)"""
        self._blob = None

    def packed_blob(self):
        key = tuple(p._version for p in self.parameters()) + (str(self.aabb.device),)
        if self._blob is None or self._blob[0] != key:
            self._blob = (key, R.pack_decoder_blob(self.decoder_params(), self.fused_variant(), self.sigmoid_saturation, self.aabb.device))
        return self._blob[1]

    # ------------------------------------------------------------------ reference API: stand-alone point decode
    def point_decode(self, xyzs, dirs, code, density_only=False):
        """sigma (and rgb) at arbitrary points: the call contract of triplane_decoder.py:119-179 --
        xyzs: tensor [B,P,3] or a list of B tensors [P_i,3]; dirs: list of B tensors [P_i,3] (or one tensor [B,P,3]), unused when
        `density_only`; code [B,3,C,H,W]  ->  (sigmas [sum P_i], rgbs [sum P_i,3] | None, [P_0, ..., P_{B-1}]).
        One native launch (csrc/point_decode.cu); inference only -- the differentiable decode lives inside the fused
        train-branch renderer (csrc/render_train.cu)."""
        if torch.is_grad_enabled() and (code.requires_grad or (self.training and any(p.requires_grad for p in self.parameters()))):
            raise NotImplementedError('TriPlaneDecoder.point_decode is forward-only; gradients w.r.t. the code flow through the fused '
                                      'differentiable renderer (decoder.forward in train mode), which also produces the decoder-weight gradients')
        if self.code_dropout is not None and self.training:
            raise NotImplementedError('code_dropout > 0 is unused by every reference config and not built')
        N.require_cuda(code)
        variant = self.fused_variant()
        pts = [xyzs[i] for i in range(len(xyzs))] if not isinstance(xyzs, torch.Tensor) else list(xyzs.unbind(0))
        if len(pts) != code.size(0):
            raise ValueError(f'{len(pts)} point sets for {code.size(0)} scenes')
        counts = [int(p.shape[-2]) for p in pts]
        flat_xyz = torch.cat([p.reshape(-1, 3) for p in pts], dim=0).contiguous().float()
        total = flat_xyz.shape[0]
        offsets = torch.tensor([0] + [sum(counts[:i + 1]) for i in range(len(counts))], dtype=torch.int64).to(code.device, non_blocking=True)
        flat_dir = None
        if not density_only:
            if not self.use_dir_enc:
                raise NotImplementedError('decoders without direction encoding are unused by the reference configs and not built')
            ds = list(dirs.unbind(0)) if isinstance(dirs, torch.Tensor) else list(dirs)
            flat_dir = torch.cat([d.reshape(-1, 3) for d in ds], dim=0).contiguous().float()
            if flat_dir.shape[0] != total:
                raise ValueError('xyzs and dirs disagree on the number of points')
        sigmas = torch.empty(total, dtype=torch.float32, device=code.device)
        rgbs = None if density_only else torch.empty(total, 3, dtype=torch.float32, device=code.device)
        planes = R.pack_planes(code.detach(), variant)
        N.check(N.lib().ssdnerf_point_decode(N.c_int(variant), N.ptr(planes), N.c_u32(code.shape[-2]), N.c_u32(code.shape[-1]),
                                             N.ptr(self.packed_blob()), N.ptr(flat_xyz), N.ptr(flat_dir), N.ptr(offsets), N.c_u32(len(counts)),
                                             N.ctypes.c_ulonglong(total), N.ptr(sigmas), N.ptr(rgbs), N.stream_ptr()))
        return sigmas, rgbs, counts

    def point_density_decode(self, xyzs, code, **kwargs):
        """triplane_decoder.py:181-184"""
        sigmas, _, counts = self.point_decode(xyzs, None, code, density_only=True, **kwargs)
        return sigmas, counts

    def visualize(self, code, scene_name, viz_dir, code_range=[-1, 1]):
        """triplane_decoder.py:186-194: scene_<name>.png per scene, the code [n, 3, C, h, w] as a [3 h, C w] viridis map over
        code_range (ssdnerf_b200/viz.py)"""
        maps = V.code_maps(code.detach().float(), self.flip_z)
        V.write_pngs([os.path.join(viz_dir, 'scene_' + s + '.png') for s in scene_name], maps=maps, vmin=code_range[0], vmax=code_range[1])

    # ------------------------------------------------------------------ forward
    def forward(self, rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma=0, perturb=False, T_thresh=1e-4, return_loss=False):
        """base_volume_renderer.py:41-133."""
        num_scenes = len(rays_o)
        assert num_scenes > 0
        if self.training:
            results = self._forward_train(rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh)
        else:
            results = self._forward_eval_fused(rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh)
        if return_loss:
            results.update(decoder_reg_loss=self.loss())
        return results

    def _forward_eval_fused(self, rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh):
        if perturb:
            raise NotImplementedError('perturb=True in eval mode is not used by the reference (base_nerf.py:518) and not built')
        if not isinstance(rays_o, torch.Tensor):
            sizes = {r.size(0) for r in rays_o}
            if len(sizes) != 1:
                raise NotImplementedError('fused renderer needs the same number of rays per scene')
            rays_o, rays_d = torch.stack(list(rays_o)), torch.stack(list(rays_d))
        num_scenes = rays_o.size(0)
        if not isinstance(grid_size, int):
            assert len(set(grid_size)) == 1
            grid_size = grid_size[0]
        if isinstance(dt_gamma, (int, float)):
            dtg = None if dt_gamma == 0 else torch.full((num_scenes,), float(dt_gamma), device=rays_o.device)
        else:
            dtg = torch.as_tensor(dt_gamma, dtype=torch.float32, device=rays_o.device).reshape(num_scenes)
        variant = self.fused_variant()
        planes = R.pack_planes(code, variant)
        out = R.render_fwd(variant, planes, tuple(code.shape[-2:]), density_bitfield.reshape(num_scenes, -1), self.packed_blob(),
                           rays_o=rays_o.reshape(num_scenes, -1, 3), rays_d=rays_d.reshape(num_scenes, -1, 3), grid_size=grid_size,
                           bound=float(self.bound), min_near=float(self.min_near), max_steps=int(self.max_steps), T_thresh=T_thresh,
                           dt_gamma=dtg, want_blend=False, want_counts=False)
        # eval mode returns per-scene lists (base_volume_renderer.py:90-123)
        return dict(weights_sum=list(out['weights_sum']), depth=list(out['depth']), image=list(out['image']))

    def trainable_params(self):
        """the decoder parameters in renderer.DEC_P_PARAM_ORDER when at least one of them wants a gradient, else ()"""
        if not any(p.requires_grad for p in self.parameters()):
            return ()
        named = dict(self.named_parameters())
        return tuple(named[k] for k in R.DEC_P_PARAM_ORDER)

    def _fused_train_ok(self, rays_o, code, grid_size):
        if self.code_dropout is not None:
            return False
        if not isinstance(rays_o, torch.Tensor) and len({r.size(0) for r in rays_o}) != 1:
            return False
        if not isinstance(grid_size, int) and len(set(grid_size)) != 1:
            return False
        try:
            return self.fused_variant() == R.DEC_P and code.size(2) == 6
        except N.SSDNeRFNativeError:
            return False

    def _forward_train_fused(self, rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh):
        if not isinstance(rays_o, torch.Tensor):
            rays_o, rays_d = torch.stack(list(rays_o)), torch.stack(list(rays_d))
        num_scenes = rays_o.size(0)
        rays_o, rays_d = rays_o.reshape(num_scenes, -1, 3).contiguous().float(), rays_d.reshape(num_scenes, -1, 3).contiguous().float()
        if not isinstance(grid_size, int):
            grid_size = grid_size[0]
        if isinstance(dt_gamma, (int, float)):
            dtg = None if dt_gamma == 0 else torch.full((num_scenes,), float(dt_gamma), device=rays_o.device)
        else:
            dtg = torch.as_tensor(dt_gamma, dtype=torch.float32, device=rays_o.device).reshape(num_scenes).contiguous()
        if isinstance(perturb, torch.Tensor):          # extension: inject the K6 start offsets (parity tests)
            noises = perturb.reshape(num_scenes, -1).contiguous().float()
        else:
            noises = torch.rand(num_scenes, rays_o.size(1), device=rays_o.device) if perturb else None
        if isinstance(density_bitfield, (list, tuple)):
            density_bitfield = torch.stack(list(density_bitfield))
        cfg = dict(grid_size=int(grid_size), bound=float(self.bound), min_near=float(self.min_near), max_steps=int(self.max_steps),
                   T_thresh=float(T_thresh))
        ws, depth, image = _FusedTrainRender.apply(code, rays_o, rays_d, density_bitfield.reshape(num_scenes, -1).contiguous(),
                                                   self.packed_blob(), noises, dtg, cfg, *self.trainable_params())
        return dict(weights_sum=ws, depth=depth, image=image)

    def _forward_train(self, rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh):
        """base_volume_renderer.py:59-77.  The train branch exists as ONE fused differentiable op for the shipped-config decoder:
        gradient w.r.t. the code (guidance, code optimisation: diffusion_nerf.py:273,358) and, for a trainable decoder, w.r.t. its
        weights (multiscene_nerf.py:203-207).  Other decoder shapes fail loudly rather than fall back to a PyTorch composition.  The
        reference's per-op kernels stay available one by one in `ssdnerf_b200.raymarching` (march_rays_train, composite_rays_train)."""
        if self._fused_train_ok(rays_o, code, grid_size):
            return self._forward_train_fused(rays_o, rays_d, code, density_bitfield, grid_size, dt_gamma, perturb, T_thresh)
        raise NotImplementedError(
            'TriPlaneDecoder train branch: only the shipped-config decoder (3x6-channel triplanes, hidden 64, dir_net, no code_dropout) '
            'with equal ray counts per scene is built (fused differentiable renderer)')
