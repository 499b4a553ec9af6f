"""`GaussianDiffusion` -- DDIM and DDPM sampling over triplane latents, driven from one CUDA stream.

Plugin surface of lib/models/diffusions/gaussian_diffusion.py:14-464 (constructor kwargs, `forward`, `ddim_sample`, `ddpm_sample`,
`sample_from_noise`, `pred_x_0`, schedule attributes, `test_cfg` read at call time).  The sampler differs in HOW it
runs: the reference re-uploads a 1000-entry table and syncs device->host several times per step
(gaussian_diffusion.py:190-191,275-279,302-304); here the timestep list and all coefficients are computed once on the
host (float64, like the reference's NumPy tables), the per-step time-embedding projections are precomputed for every
step, and ONE captured CUDA graph (UNet forward + fused update, device-side step counter) is replayed `num_timesteps`
times.  The fused update is V->x0->eps->x_prev for DDIM and V->x0->posterior mean + sigma * noise for DDPM, whose noise
the kernel generates from a per-call seed in device memory.
"""
import math
import os
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from . import _lib as N
from .registry import MODULES, build_module


@MODULES.register_module()
class UniformTimeStepSampler:
    """mmgen.models.diffusions.sampler.UniformTimeStepSampler [mmgen-memory]: t ~ Categorical(prob) drawn with NumPy on the host"""

    def __init__(self, num_timesteps, **kwargs):
        self.num_timesteps = num_timesteps
        self.prob = [1 / num_timesteps for _ in range(num_timesteps)]

    def sample(self, batch_size):
        return torch.from_numpy(np.random.choice(self.num_timesteps, size=(batch_size,), p=self.prob)).long()

    def __call__(self, batch_size):
        return self.sample(batch_size)


@MODULES.register_module()
class UniformTimeStepSamplerMod(UniformTimeStepSampler):
    """lib/models/diffusions/sampler.py:7-11"""


@MODULES.register_module()
class SNRWeightedTimeStepSampler(UniformTimeStepSampler):
    """lib/models/diffusions/sampler.py:14-46: per-timestep loss weight from the signal-to-noise ratio (+ optional importance sampling)"""

    def __init__(self, num_timesteps, mean, std, mode, power=1, min=-1, max=-1, bias=0, prob_power=0.0):
        self.num_timesteps = num_timesteps
        weight_x = (mean / std) ** (2 * power) + bias
        if min > 0:
            weight_x = weight_x.clip(min=min)
        if max > 0:
            weight_x = weight_x.clip(max=max)
        mode = mode.upper()
        if mode == 'EPS':
            weight_raw = weight_x * (std / mean) ** 2
        elif mode == 'START_X':
            weight_raw = weight_x
        elif mode == 'V':
            weight_raw = weight_x * (std ** 2)
        else:
            raise AttributeError(f'unknown denoising mean mode {mode}')
        prob = weight_raw ** prob_power
        prob = prob / prob.sum()
        self.weight = torch.from_numpy(weight_raw / (prob * self.num_timesteps)).to(torch.float)
        self.prob = prob.tolist()


@MODULES.register_module()
class DDPMMSELossMod(nn.Module):
    """lib/models/losses/ddpm_loss.py:12-131 on mmgen's DDPMLoss base [mmgen-memory]: per-sample 0.5 * MSE between the tensors named by
    `data_info`, rescaled per timestep (`rescale_mode='timestep_weight'`: sampler.weight[t] * weight_scale), mean over the batch, divided
    by the running `norm_factor` buffer when `scale_norm` (the buffer is part of released checkpoints)."""
    _default_data_info = dict(pred='eps_t_pred', target='noise')

    def __init__(self, rescale_mode=None, rescale_cfg=None, sampler=None, weight=None, weight_scale=1.0, log_cfgs=None, reduction='mean',
                 data_info=None, loss_name='loss_ddpm_mse', scale_norm=False, momentum=0.001):
        super().__init__()
        assert reduction in ('mean', 'sum', 'none', 'flatmean')
        self.rescale_mode, self.weight_scale, self.reduction, self.loss_name = rescale_mode, weight_scale, reduction, loss_name
        self.data_info = dict(self._default_data_info if data_info is None else data_info)
        if rescale_mode == 'timestep_weight':
            w = weight if weight is not None else getattr(sampler, 'weight', None)
            if w is None:
                raise ValueError("rescale_mode='timestep_weight' needs `weight` or a sampler with a `weight` table")
            self._t_weight = torch.as_tensor(w, dtype=torch.float).clone()
        elif rescale_mode == 'constant':
            self._t_weight = None
            self._const = (rescale_cfg or {}).get('scale', 1.0)
        elif rescale_mode is None:
            self._t_weight = None
        else:
            raise NotImplementedError(f'rescale_mode {rescale_mode} is not used by the reference configs')
        self.scale_norm, self.freeze_norm, self.momentum = scale_norm, False, momentum
        if scale_norm:
            self.register_buffer('norm_factor', torch.ones(1, dtype=torch.float))
        self.log_vars = dict()

    def forward(self, output_dict):
        t = output_dict['timesteps']
        pred, target = output_dict[self.data_info['pred']], output_dict[self.data_info['target']]
        loss = (pred - target).square().flatten(1).mean(dim=1) * 0.5
        if self.rescale_mode == 'timestep_weight':
            loss = loss * self._t_weight.to(t.device)[t] * self.weight_scale
        elif self.rescale_mode == 'constant':
            loss = loss * self._const
        self.log_vars = {self.loss_name: float(loss.detach().mean())}
        loss = dict(mean=loss.mean, sum=loss.sum, flatmean=loss.mean, none=lambda: loss)[self.reduction]()
        if self.scale_norm:
            if self.training and not self.freeze_norm:
                with torch.no_grad():
                    nf = output_dict['x_0'].detach().square().mean()
                    if torch.distributed.is_available() and torch.distributed.is_initialized():
                        torch.distributed.all_reduce(nf)
                        nf = nf / torch.distributed.get_world_size()
                    self.norm_factor.lerp_(nf.to(self.norm_factor).reshape(1), self.momentum)
            loss = loss / self.norm_factor
        return loss


MODULES.register_module(name='DDPMMSELoss', module=DDPMMSELossMod)      # the class default of gaussian_diffusion.py:18-21 (mmgen's own)


@MODULES.register_module()
class GaussianDiffusion(nn.Module):

    def __init__(self, denoising, ddpm_loss=None, betas_cfg=dict(type='cosine'), num_timesteps=1000, num_classes=0,
                 sample_method='ddim', timestep_sampler=None, denoising_var_mode='FIXED_LARGE', denoising_mean_mode='V',
                 train_cfg=None, test_cfg=None):
        super().__init__()
        self.num_classes = num_classes
        self.num_timesteps = num_timesteps
        self.sample_method = sample_method
        self._denoising_cfg = deepcopy(denoising)
        self.denoising = denoising if isinstance(denoising, nn.Module) else build_module(
            denoising, default_args=dict(num_classes=num_classes, num_timesteps=num_timesteps))
        self.denoising_var_mode = denoising_var_mode
        self.denoising_mean_mode = denoising_mean_mode
        self.betas_cfg = deepcopy(betas_cfg)
        self.train_cfg = deepcopy(train_cfg) if train_cfg is not None else dict()
        self.test_cfg = deepcopy(test_cfg) if test_cfg is not None else dict()
        self.prepare_diffusion_vars()
        # gaussian_diffusion.py:54-62: the timestep sampler (carries the SNR loss weights) and the diffusion loss -- used at test time by
        # val_optim / n_inverse_steps (the diffusion prior on the latent)
        self.sampler = build_module(timestep_sampler if timestep_sampler is not None else dict(type='UniformTimeStepSampler'),
                                    default_args=dict(num_timesteps=num_timesteps, mean=self.sqrt_alphas_bar, std=self.sqrt_one_minus_alphas_bar,
                                                      mode=self.denoising_mean_mode))
        loss_cfg = dict(ddpm_loss) if ddpm_loss is not None else dict(type='DDPMMSELoss')
        self.ddpm_loss = build_module(loss_cfg, default_args=dict(sampler=self.sampler))
        self._graphs = {}
        self._graph_kernel_nodes = 0

    # ------------------------------------------------------------------ schedules (gaussian_diffusion.py:64-154)
    @staticmethod
    def linear_beta_schedule(diffusion_timesteps, beta_0=1e-4, beta_T=2e-2):
        scale = 1000 / diffusion_timesteps
        return np.linspace(scale * beta_0, scale * beta_T, diffusion_timesteps, dtype=np.float64)

    @staticmethod
    def cosine_beta_schedule(diffusion_timesteps, max_beta=0.999, s=0.008):
        def f(t, T, s):
            return np.cos((t / T + s) / (1 + s) * np.pi / 2) ** 2
        betas = []
        for t in range(diffusion_timesteps):
            betas.append(min(1 - f(t + 1, diffusion_timesteps, s) / f(t, diffusion_timesteps, s), max_beta))
        return np.array(betas)

    def get_betas(self):
        cfg = dict(self.betas_cfg)
        self.betas_schedule = cfg.pop('type')
        if self.betas_schedule == 'linear':
            return self.linear_beta_schedule(self.num_timesteps, **cfg)
        if self.betas_schedule == 'cosine':
            return self.cosine_beta_schedule(self.num_timesteps, **cfg)
        if self.betas_schedule == 'scaled_linear':
            return np.linspace(cfg.get('beta_start', 0.0001) ** 0.5, cfg.get('beta_end', 0.02) ** 0.5, self.num_timesteps,
                               dtype=np.float64) ** 2
        raise AttributeError(f'Unknown method name {self.betas_schedule} for beta schedule.')

    def prepare_diffusion_vars(self):
        self.betas = self.get_betas()
        self.alphas = 1.0 - self.betas
        self.alphas_bar = np.cumprod(self.alphas, axis=0)
        self.alphas_bar_prev = np.append(1.0, self.alphas_bar[:-1])
        self.alphas_bar_next = np.append(self.alphas_bar[1:], 0.0)
        self.sqrt_alphas_bar = np.sqrt(self.alphas_bar)
        self.sqrt_one_minus_alphas_bar = np.sqrt(1.0 - self.alphas_bar)
        self.log_one_minus_alphas_bar = np.log(1.0 - self.alphas_bar)
        self.sqrt_recip_alplas_bar = np.sqrt(1.0 / self.alphas_bar)
        self.sqrt_recipm1_alphas_bar = np.sqrt(1.0 / self.alphas_bar - 1)
        self.tilde_betas_t = self.betas * (1 - self.alphas_bar_prev) / (1 - self.alphas_bar)
        self.log_tilde_betas_t_clipped = np.log(np.append(self.tilde_betas_t[1], self.tilde_betas_t[1:]))
        self.tilde_mu_t_coef1 = np.sqrt(self.alphas_bar_prev) / (1 - self.alphas_bar) * self.betas
        self.tilde_mu_t_coef2 = np.sqrt(self.alphas) * (1 - self.alphas_bar_prev) / (1 - self.alphas_bar)

    # ------------------------------------------------------------------ single-step API
    def _coef(self, x_t, table, t):
        """the reference indexes a table rebuilt in x_t's dtype with the device timestep (gaussian_diffusion.py:190-191)"""
        return x_t.new_tensor(table)[t].reshape(-1, 1, 1, 1)

    def q_sample(self, x_0, t, noise=None):
        """gaussian_diffusion.py:166-178"""
        if noise is None:
            noise = torch.randn_like(x_0)
        idx = t.cpu()
        mean = torch.from_numpy(self.sqrt_alphas_bar)[idx].float().to(x_0.device).reshape(-1, 1, 1, 1)
        std = torch.from_numpy(self.sqrt_one_minus_alphas_bar)[idx].float().to(x_0.device).reshape(-1, 1, 1, 1)
        return x_0 * mean + noise * std, mean, std

    def _x0_from_output(self, x_t, out, sa, s1):
        mode = self.denoising_mean_mode.upper()
        if mode == 'EPS':
            return (x_t - s1 * out) / sa
        if mode == 'START_X':
            return out
        if mode == 'V':
            return sa * x_t - s1 * out
        raise AttributeError(f'Unknown denoising mean output type [{self.denoising_mean_mode}].')

    def pred_x_0(self, x_t, t, grad_guide_fn=None, concat_cond=None, cfg=dict(), update_denoising_output=False):
        """gaussian_diffusion.py:180-240.  With `grad_guide_fn` the guidance gradient is taken w.r.t. x_t THROUGH the denoiser
        (`grad_through_unet=True`, the reference default: the UNet's hand-written input-gradient pass, unet.py `_UNetInputGrad`)
        or w.r.t. the clamped x_0 (`grad_through_unet=False`)."""
        clip_denoised = cfg.get('clip_denoised', True)
        clip_range = cfg.get('clip_range', [-1, 1])
        guidance_gain = cfg.get('guidance_gain', 1.0)
        grad_through_unet = cfg.get('grad_through_unet', True)
        snr_weight_power = cfg.get('snr_weight_power', 0.5)
        num_batches = x_t.size(0)
        if not torch.is_tensor(t):
            t = torch.as_tensor(t, device=x_t.device)
        if t.dim() == 0 or len(t) != num_batches:
            t = t.expand(num_batches)
        sa = self._coef(x_t, self.sqrt_alphas_bar, t)
        s1 = self._coef(x_t, self.sqrt_one_minus_alphas_bar, t)
        through = grad_guide_fn is not None and grad_through_unet
        if through:
            x_t = x_t.detach().requires_grad_(True)
        # no guidance: the ambient autograd mode applies (forward_train differentiates the denoiser w.r.t. x_t for val_optim)
        with torch.set_grad_enabled(through or (grad_guide_fn is None and torch.is_grad_enabled())):
            out = self.denoising(x_t, t, concat_cond=concat_cond)
            x_0 = self._x0_from_output(x_t, out, sa, s1)
            if grad_guide_fn is not None and clip_denoised:
                x_0 = x_0.clamp(*clip_range)
            if through:
                grad = torch.autograd.grad(grad_guide_fn(x_0), x_t)[0]
        if grad_guide_fn is not None:
            if not through:
                with torch.enable_grad():
                    x_0 = x_0.detach().requires_grad_(True)
                    grad = torch.autograd.grad(grad_guide_fn(x_0), x_0)[0]
            x_t, out = x_t.detach(), out.detach()
            x_0 = x_0.detach() - grad * ((s1 ** (2 - snr_weight_power * 2)) * (sa ** (snr_weight_power * 2 - 1)) * guidance_gain)
        if clip_denoised:
            x_0 = x_0.clamp(*clip_range)
        if update_denoising_output and grad_guide_fn is not None:
            mode = self.denoising_mean_mode.upper()
            if mode == 'EPS':
                out = (x_t - x_0 * sa) / s1
            elif mode == 'START_X':
                out = x_0
            else:
                out = (sa * x_t - x_0) / s1
        return x_0, out

    @torch.no_grad()
    def p_sample_langevin(self, x_t, t, noise=None, cfg=dict(), grad_guide_fn=None, **kwargs):
        """gaussian_diffusion.py:242-262"""
        t = int(t)
        langevin_delta = cfg.get('langevin_delta', 0.1)
        sigma = float(self.sqrt_one_minus_alphas_bar[t])
        x_0_pred, _ = self.pred_x_0(x_t, torch.as_tensor(t, device=x_t.device), grad_guide_fn=grad_guide_fn, cfg=cfg, **kwargs)
        eps_t_pred = (x_t - float(self.sqrt_alphas_bar[t]) * x_0_pred) / sigma
        if noise is None:
            noise = torch.randn_like(x_t)
        return x_t - 0.5 * langevin_delta * sigma * eps_t_pred + math.sqrt(langevin_delta) * sigma * noise

    @torch.no_grad()
    def p_sample_ddim(self, x_t, t, t_prev, noise=None, cfg=dict(), grad_guide_fn=None, **kwargs):
        """gaussian_diffusion.py:264-293"""
        t, t_prev = int(t), int(t_prev)
        eta = cfg.get('eta', 0)
        alpha_bar_t_prev = self.alphas_bar[t_prev] if t_prev >= 0 else self.alphas_bar_prev[0]
        tilde_beta_t = self.tilde_betas_t[t]
        x_0_pred, _ = self.pred_x_0(x_t, torch.as_tensor(t, device=x_t.device), grad_guide_fn=grad_guide_fn, cfg=cfg, **kwargs)
        eps_t_pred = (x_t - float(self.sqrt_alphas_bar[t]) * x_0_pred) / float(self.sqrt_one_minus_alphas_bar[t])
        x_prev = float(np.sqrt(alpha_bar_t_prev)) * x_0_pred + float(np.sqrt(1 - alpha_bar_t_prev - tilde_beta_t * (eta ** 2))) * eps_t_pred
        if eta > 0:
            if noise is None:
                noise = torch.randn_like(x_t)
            x_prev = x_prev + eta * float(np.sqrt(tilde_beta_t)) * noise
        return x_prev, x_0_pred

    def _table_f32(self, x, table, t):
        """mmgen's var_to_tensor: the float64 table entry at t rounded to float32, shaped to broadcast over x"""
        return torch.from_numpy(np.asarray(table))[torch.as_tensor(t).cpu()].float().to(x.device).reshape(-1, 1, 1, 1)

    def q_posterior_mean(self, x_0, x_t, t):
        """gaussian_diffusion.py:156-164"""
        return self._table_f32(x_0, self.tilde_mu_t_coef1, t) * x_0 + self._table_f32(x_0, self.tilde_mu_t_coef2, t) * x_t

    def _ddpm_var_table(self):
        """gaussian_diffusion.py:343-349: FIXED_LARGE indexes [tilde_beta_1, betas...] at t, i.e. betas[t - 1] for t >= 1"""
        mode = self.denoising_var_mode.upper()
        if mode == 'FIXED_LARGE':
            return np.append(self.tilde_betas_t[1], self.betas)
        if mode == 'FIXED_SMALL':
            return self.tilde_betas_t
        raise AttributeError(f'Unknown denoising var output type [{self.denoising_var_mode}].')

    @torch.no_grad()
    def p_sample_ddpm(self, x_t, t, noise=None, cfg=dict(), grad_guide_fn=None, **kwargs):
        """gaussian_diffusion.py:333-365: posterior mean of the predicted x_0, plus sqrt(var_t) * noise unless t == 0"""
        var = self._table_f32(x_t, self._ddpm_var_table(), t)
        x_0_pred, _ = self.pred_x_0(x_t, torch.as_tensor(t, device=x_t.device), grad_guide_fn=grad_guide_fn, cfg=cfg, **kwargs)
        mean = self.q_posterior_mean(x_0_pred, x_t, t)
        if noise is None:
            noise = torch.randn_like(x_t)
        nonzero_mask = (torch.as_tensor(t) != 0).float().reshape(-1, 1, 1, 1).to(x_t.device)
        return mean + nonzero_mask * torch.sqrt(var) * noise, x_0_pred

    @torch.no_grad()
    def _ddim_sample_stepwise(self, noise, concat_cond=None, save_intermediates=False, grad_guide_fn=None, langevin_noises=None,
                              show_pbar=False, **kwargs):
        """gaussian_diffusion.py:295-331 step by step (host timesteps: no device->host sync): guidance, langevin
        correction steps, eta > 0 and `save_intermediates`.  The unguided eta=0 loop uses the captured graph instead.
        `langevin_noises`: optional iterator of the tensors the langevin steps add (parity tests; default torch.randn)."""
        if concat_cond is not None:
            raise NotImplementedError('concat_cond (image-conditioned denoiser) is not used by the shipped configs')
        cfg = self.test_cfg
        x_t = noise.detach().float()
        num_timesteps = cfg.get('num_timesteps', self.num_timesteps)
        langevin_steps = cfg.get('langevin_steps', 0)
        langevin_t_range = cfg.get('langevin_t_range', [0, 1000])
        timesteps = [int(t) for t in self.ddim_timesteps(num_timesteps)]
        out = [] if save_intermediates else None
        for step, t in enumerate(timesteps):
            t_prev = timesteps[step + 1] if step + 1 < len(timesteps) else -1
            x_t, x_0_pred = self.p_sample_ddim(x_t, t, t_prev, cfg=cfg, grad_guide_fn=grad_guide_fn, **kwargs)
            if langevin_steps > 0 and langevin_t_range[0] < t_prev < langevin_t_range[1]:
                for _ in range(langevin_steps):
                    x_t = self.p_sample_langevin(x_t, t_prev, cfg=cfg, grad_guide_fn=grad_guide_fn,
                                                 noise=next(langevin_noises) if langevin_noises is not None else None, **kwargs)
            if out is not None:
                out.extend([x_0_pred, x_t])
        return out if save_intermediates else x_t

    def ddim_timesteps(self, num_timesteps):
        """gaussian_diffusion.py:302-304, kept on the HOST (the reference moves them to the GPU and syncs per step)"""
        return torch.arange(start=self.num_timesteps - 1, end=-1, step=-(self.num_timesteps / num_timesteps)).long()

    def ddim_coefficients(self, timesteps, eta=0.0):
        """float64 host tables -> fp32 rows {sqrt(ab_t), sqrt(1-ab_t), sqrt(ab_prev), sqrt(1-ab_prev-eta^2 beta~_t)} (:275-281)"""
        rows = []
        ts = [int(t) for t in timesteps]
        for i, t in enumerate(ts):
            t_prev = ts[i + 1] if i + 1 < len(ts) else -1
            ab_prev = self.alphas_bar[t_prev] if t_prev >= 0 else self.alphas_bar_prev[0]
            rows.append([self.sqrt_alphas_bar[t], self.sqrt_one_minus_alphas_bar[t], np.sqrt(ab_prev),
                         np.sqrt(1 - ab_prev - self.tilde_betas_t[t] * eta ** 2)])
        return torch.tensor(np.asarray(rows, np.float64), dtype=torch.float32)

    # ------------------------------------------------------------------ the loops
    @torch.no_grad()
    def ddim_sample(self, noise, show_pbar=False, concat_cond=None, save_intermediates=False, use_graph=True, **kwargs):
        """gaussian_diffusion.py:295-331.  Unguided eta=0 V-parameterisation (every unconditional config) = captured graph;
        guidance / langevin / eta > 0 / save_intermediates = the step-wise loop on the same engine."""
        cfg = self.test_cfg
        eta = cfg.get('eta', 0)
        if (kwargs.get('grad_guide_fn') is not None or cfg.get('langevin_steps', 0) > 0 or save_intermediates or eta != 0
                or self.denoising_mean_mode.upper() != 'V'):
            return self._ddim_sample_stepwise(noise, concat_cond=concat_cond, save_intermediates=save_intermediates, **kwargs)
        if concat_cond is not None:
            raise NotImplementedError('concat_cond (image-conditioned denoiser) is not used by the shipped configs')
        N.require_cuda(noise)
        B, C, H, W = noise.shape
        # Lanes (optional): the batch can be split into independent sub-batches, each with its own engine, captured step and CUDA stream.
        # The persistent GEMM kernels own all SMs, so lanes serialise and only add launches; the default stays 1.
        n_lanes = int(os.environ.get('SSDNERF_DDIM_STREAMS', cfg.get('ddim_streams', 1)))
        if n_lanes < 1 or B % n_lanes or not use_graph:
            n_lanes = 1
        st = self._sampler_state('ddim', noise, use_graph, n_lanes, lambda ts: self.ddim_coefficients(ts, eta))
        L = N.lib()

        def update(ln, v, s):
            eng = ln['eng']
            N.check(L.ssdnerf_ddim_update(N.ptr(ln['x_t']), N.ptr(v), N.c_u32(ln['hi'] - ln['lo']), N.c_u32(C), N.c_u32(H), N.c_u32(W),
                                          N.c_u32(v.shape[-1]), N.ptr(st['coef']), N.ptr(ln['step_ptr']), N.c_int(int(st['clip'])),
                                          N.c_f32(st['clip_range'][0]), N.c_f32(st['clip_range'][1]), None, N.ptr(eng.x_in), N.c_u32(eng.CPAD_IN), s))
        return self._run_sampler(st, noise, update, use_graph)

    @torch.no_grad()
    def _ddpm_sample_stepwise(self, noise, grad_guide_fn=None, ddpm_noises=None, **kwargs):
        """gaussian_diffusion.py:367-386 step by step (host timesteps): guidance, EPS / START_X denoisers and injected noise.
        `ddpm_noises`: optional iterator of the tensors the steps add (parity tests; default torch.randn, as the reference)."""
        cfg = self.test_cfg
        x_t = noise.detach().float()
        for t in self.ddim_timesteps(cfg.get('num_timesteps', self.num_timesteps)).tolist():
            x_t, _ = self.p_sample_ddpm(x_t, t, noise=next(ddpm_noises) if ddpm_noises is not None else None, cfg=cfg,
                                        grad_guide_fn=grad_guide_fn, **kwargs)
        return x_t

    def ddpm_coefficients(self, timesteps):
        """float64 host tables -> fp32 rows {sqrt(ab_t), sqrt(1-ab_t), coef1_t, coef2_t, (t != 0) sqrt(var_t)} (:156-164,333-365):
        each table entry rounded to float32 (var_to_tensor), the square root of the variance taken in float32 (torch.sqrt)"""
        var = self._ddpm_var_table()
        rows = []
        for t in (int(t) for t in timesteps):
            rows.append([np.float32(self.sqrt_alphas_bar[t]), np.float32(self.sqrt_one_minus_alphas_bar[t]), np.float32(self.tilde_mu_t_coef1[t]),
                         np.float32(self.tilde_mu_t_coef2[t]), np.sqrt(np.float32(var[t])) if t != 0 else np.float32(0)])
        return torch.from_numpy(np.asarray(rows, np.float32))

    @torch.no_grad()
    def ddpm_sample(self, noise, show_pbar=False, concat_cond=None, use_graph=True, ddpm_noises=None, **kwargs):
        """gaussian_diffusion.py:367-386: the posterior step at each of the strided timesteps of `ddim_timesteps`.  Unguided V-parameterisation
        = captured graph (UNet forward + ssdnerf_ddpm_update, whose noise is generated in the kernel from a seed drawn per call with
        `torch.empty(1, dtype=torch.int64).random_()`, so `torch.manual_seed` makes a call repeatable); guidance, EPS / START_X and
        injected `ddpm_noises` = the step-wise loop."""
        if 'save_intermediates' in kwargs:
            raise TypeError('ddpm_sample keeps no intermediates: save_intermediates is a ddim_sample option')
        if concat_cond is not None:
            raise NotImplementedError('concat_cond (image-conditioned denoiser) is not used by the shipped configs')
        self._ddpm_var_table()                # an unknown denoising_var_mode raises before any work, as in p_sample_ddpm
        if kwargs.get('grad_guide_fn') is not None or ddpm_noises is not None or self.denoising_mean_mode.upper() != 'V':
            return self._ddpm_sample_stepwise(noise, ddpm_noises=ddpm_noises, **kwargs)
        N.require_cuda(noise)
        B, C, H, W = noise.shape
        st = self._sampler_state(('ddpm', self.denoising_var_mode.upper()), noise, use_graph, 1, self.ddpm_coefficients)
        if 'seed' not in st:
            st['seed'] = torch.empty(1, dtype=torch.int64, device=noise.device)
        st['seed'].copy_(torch.empty(1, dtype=torch.int64).random_())
        L = N.lib()

        def update(ln, v, s):
            eng = ln['eng']
            N.check(L.ssdnerf_ddpm_update(N.ptr(ln['x_t']), N.ptr(v), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W), N.c_u32(v.shape[-1]),
                                          N.ptr(st['coef']), N.ptr(ln['step_ptr']), N.ptr(st['seed']), N.c_int(int(st['clip'])),
                                          N.c_f32(st['clip_range'][0]), N.c_f32(st['clip_range'][1]), N.ptr(eng.x_in), N.c_u32(eng.CPAD_IN), s))
        return self._run_sampler(st, noise, update, use_graph)

    def _sampler_state(self, kind, noise, use_graph, n_lanes, coef_fn):
        """The state of a device-side sampling loop: per lane an engine, an x_t buffer and a device step counter; the fp32 coefficient
        rows `coef_fn(timesteps)` and every step's time-embedding projections (host precompute, no x dependence).  One entry per
        (sampler kind, denoiser weights, device, batch shape, sampler settings); a ragged last batch alternates between two entries instead of
        re-capturing.  Stale entries (changed weights) and anything beyond 4 entries are dropped, oldest first."""
        cfg = self.test_cfg
        num_steps = cfg.get('num_timesteps', self.num_timesteps)
        clip = bool(cfg.get('clip_denoised', True))
        clip_range = tuple(float(c) for c in cfg.get('clip_range', [-1, 1]))
        dev = noise.device
        B, C, H, W = noise.shape
        unet = self.denoising
        Bl = B // n_lanes
        key = (id(unet), tuple(p._version for p in unet.parameters()), str(dev), B, C, H, W, num_steps, clip, clip_range, bool(use_graph), n_lanes,
               kind)
        for k in [k for k in self._graphs if k[0] == id(unet) and k[1] != key[1]]:
            del self._graphs[k]
        st = self._graphs.get(key)
        if st is None:
            from .unet import UNetEngine
            ts = self.ddim_timesteps(num_steps)
            lanes = []
            for i in range(n_lanes):
                eng = unet.engine(Bl, dev, (H, W)) if i == 0 else UNetEngine(unet, Bl, dev, (H, W))
                lanes.append(dict(eng=eng, graph=None, lo=i * Bl, hi=(i + 1) * Bl,
                                  stream=torch.cuda.Stream(device=dev) if n_lanes > 1 else None,
                                  x_t=torch.empty(Bl, C, H, W, dtype=torch.float32, device=dev),
                                  step_ptr=torch.zeros(1, dtype=torch.int32, device=dev)))
            st = dict(key=key, S=len(ts), lanes=lanes, clip=clip, clip_range=clip_range, coef=coef_fn(ts).to(dev),
                      ss_table=lanes[0]['eng'].scale_shift_rows(unet.embedding(ts.to(dev))).contiguous())          # [S, ss_total]
            while len(self._graphs) >= 4:
                del self._graphs[next(iter(self._graphs))]
            self._graphs[key] = st
        return st

    def _run_sampler(self, st, noise, update, use_graph):
        """S steps of [select the step's embedding rows, UNet forward, `update(lane, v, stream)`, advance the step counter]: S replays of
        each lane's captured step on its stream, or (`use_graph=False`) the same launches uncaptured"""
        ss_table, S, lanes = st['ss_table'], st['S'], st['lanes']
        dev = noise.device
        n_lanes = len(lanes)
        L = N.lib()

        def one_step(ln):
            eng, step_ptr = ln['eng'], ln['step_ptr']
            s = N.stream_ptr()
            N.check(L.ssdnerf_select_row(N.ptr(ss_table), N.c_u32(eng.ss_total), N.ptr(step_ptr), N.ptr(eng.ss_cur), N.c_u32(ln['hi'] - ln['lo']), s))
            update(ln, eng.forward_nhwc(), s)
            N.check(L.ssdnerf_step_counter(N.ptr(step_ptr), N.c_int(1), N.c_int(0), s))

        def reset(ln):
            ln['x_t'].copy_(noise[ln['lo']:ln['hi']].detach().float())
            ln['step_ptr'].zero_()
            ln['eng'].load_input_nchw(ln['x_t'])

        cur = torch.cuda.current_stream(dev)
        if not use_graph:
            reset(lanes[0])
            for _ in range(S):
                one_step(lanes[0])
            return lanes[0]['x_t'].clone()
        if lanes[0]['graph'] is None:
            # warm up once on a side stream (lazy allocations / function attributes), then capture ONE step per lane
            L.ssdnerf_launch_count.restype = __import__('ctypes').c_ulonglong
            nodes = 0
            for ln in lanes:
                side = ln['stream'] or torch.cuda.Stream(device=dev)
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    reset(ln)
                    one_step(ln)
                cur.wait_stream(side)
                torch.cuda.synchronize(dev)
                graph = torch.cuda.CUDAGraph()
                c0 = L.ssdnerf_launch_count()
                with torch.cuda.graph(graph, stream=side):
                    one_step(ln)
                nodes += int(L.ssdnerf_launch_count() - c0)
                ln['graph'] = graph
            self._graph_kernel_nodes = nodes
        # the S-step loop = S replays of each lane's captured step on its stream (device-side step counters)
        if n_lanes == 1:
            reset(lanes[0])
            for _ in range(S):
                lanes[0]['graph'].replay()
            return lanes[0]['x_t'].clone()
        for ln in lanes:
            ln['stream'].wait_stream(cur)
            with torch.cuda.stream(ln['stream']):
                reset(ln)
        for _ in range(S):
            for ln in lanes:
                with torch.cuda.stream(ln['stream']):
                    ln['graph'].replay()
        for ln in lanes:
            cur.wait_stream(ln['stream'])
        return torch.cat([ln['x_t'] for ln in lanes], dim=0)

    def refresh_weights(self):
        """drop every captured graph and the denoiser's packed weights (after parameter writes that bypass `Parameter._version`)"""
        self._graphs.clear()
        if hasattr(self.denoising, 'refresh_weights'):
            self.denoising.refresh_weights()

    def sample_from_noise(self, noise, **kwargs):
        fn = getattr(self, f'{self.sample_method.lower()}_sample', None)
        if fn is None:
            raise AttributeError(f'Cannot find sample method [{self.sample_method.lower()}_sample] correspond to [{self.sample_method}].')
        return fn(noise=noise, **kwargs)

    def forward_test(self, data, **kwargs):
        assert data.dim() == 4
        return self.sample_from_noise(data, **kwargs)

    def loss(self, denoising_output, x_0, noise, t, mean, std):
        """gaussian_diffusion.py:404-421"""
        mode = self.denoising_mean_mode.upper()
        key = dict(EPS='eps_t_pred', START_X='x_0_pred', V='v_t_pred').get(mode)
        if key is None:
            raise AttributeError(f'Unknown denoising mean output type [{self.denoising_mean_mode}].')
        loss_kwargs = {key: denoising_output, 'x_0': x_0, 'noise': noise, 'timesteps': t}
        if mode == 'V':
            loss_kwargs.update(v_t=mean * noise - std * x_0)
        return self.ddpm_loss(loss_kwargs)

    def forward_train(self, x_0, concat_cond=None, grad_guide_fn=None, cfg=dict(), x_t_detach=False, t=None, noise=None, **kwargs):
        """gaussian_diffusion.py:423-450: diffusion loss of x_0 at sampled timesteps.  Differentiable w.r.t. x_0 (test-time code
        optimisation with a frozen denoiser: input-gradient pass) and, when the denoiser's parameters require gradients (training),
        w.r.t. them as well (unet_train.py weight-gradient pass).  `t` / `noise` may be injected."""
        assert x_0.dim() == 4
        num_batches = x_0.size(0)
        if t is None:
            t = self.sampler(num_batches)
        t = t.to(x_0.device)
        if noise is None:
            noise = torch.randn_like(x_0)
        x_t, mean, std = self.q_sample(x_0, t, noise)
        if x_t_detach:
            x_t = x_t.detach()
        _, denoising_output = self.pred_x_0(x_t, t, grad_guide_fn=grad_guide_fn, concat_cond=concat_cond, cfg=cfg, update_denoising_output=True)
        loss = self.loss(denoising_output, x_0, noise, t, mean, std)
        log_vars = dict(self.ddpm_loss.log_vars)
        log_vars.update(loss_ddpm_mse=float(loss.detach()))
        return loss, log_vars

    def forward(self, data, return_loss=False, **kwargs):
        if return_loss:
            return self.forward_train(data, **kwargs)
        return self.forward_test(data, **kwargs)
