"""DDPM sampling (sample_method='ddpm') on the GPU: the fused posterior step k_ddpm_update against the torch composition of
p_sample_ddpm bit for bit, its in-kernel Gaussian generator, whole chains against the fp32 oracle (oracle/ddpm_port.py) fed the kernel's
own noise, the captured graph against the step-wise loop, and the shipped configs through val_step.

Chain bars: tests/perf/ddpm_precision_probe.py injects the native path's fp16 roundings into the fp32 oracle chain and measures how far
the final sample moves (same noise on both sides); each bar is twice that probe value (DESIGN.md §4 lists both, and the measured errors)."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import ddpm_port as dp
from oracle import unet_port as up
from tests.common import GOLDEN, spiral_poses

pytestmark = pytest.mark.gpu

SMALL = dict(image_size=32, in_channels=18, base_channels=64, channels_cfg=[1, 2, 2], resblocks_per_downsample=1,
             num_heads=2, attention_res=[16, 8], use_scale_shift_norm=True)
FULL = dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
            num_heads=4, attention_res=[32, 16, 8], use_scale_shift_norm=True)
# twice the fp16-rounding probe of tests/perf/ddpm_precision_probe.py (small: 1000 steps B=2; cars: 50 steps B=2; guided: 10 steps)
BAR_SMALL, BAR_CARS, BAR_GUIDED = 2 * 5.2e-4, 2 * 4.4e-5, 2 * 1.3e-5


def _rel_l2(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _spec(cfg):
    return up.unet_spec(**{k: v for k, v in cfg.items() if k != 'use_scale_shift_norm'})


def _unet(cfg, sd, cuda):
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(**cfg)
    m.load_state_dict(sd, strict=True)
    return m.to(cuda).eval()


def _update(x, v, coef, step, seed, clip=(-2.0, 2.0), next_in=None):
    """one ssdnerf_ddpm_update launch on x [B,C,H,W] in place with v [B,H,W,Cv]"""
    from ssdnerf_b200 import _lib as N
    B, C, H, W = x.shape
    dev = x.device
    sp = torch.tensor([step], dtype=torch.int32, device=dev)
    sd = torch.tensor([seed], dtype=torch.int64, device=dev)
    cpad = next_in.shape[-1] if next_in is not None else (C + 7) // 8 * 8
    N.check(N.lib().ssdnerf_ddpm_update(N.ptr(x), N.ptr(v), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W), N.c_u32(v.shape[-1]), N.ptr(coef),
                                        N.ptr(sp), N.ptr(sd), N.c_int(clip is not None), N.c_f32(clip[0] if clip else 0), N.c_f32(clip[1] if clip else 0),
                                        N.ptr(next_in), N.c_u32(cpad), N.stream_ptr()))
    return x


def kernel_noise(seed, step, shape, dev):
    """the noise k_ddpm_update adds at (seed, step), read back through the coefficient row {0, 0, 0, 0, 1}"""
    B, C, H, W = shape
    coef = torch.tensor([[0, 0, 0, 0, 1]], dtype=torch.float32).repeat(step + 1, 1).to(dev)
    return _update(torch.zeros(shape, device=dev), torch.zeros(B, H, W, C, device=dev), coef, step, seed, clip=None)


def _seed_of_call(k):
    """the seed ddpm_sample draws first after torch.manual_seed(k)"""
    torch.manual_seed(k)
    return int(torch.empty(1, dtype=torch.int64).random_())


def _last_seed(d):
    """the seed of the last captured DDPM call of diffusion d"""
    return next(int(st['seed']) for k, st in d._graphs.items() if k[-1][0] == 'ddpm' and k[-3])


class _Fixed(torch.nn.Module):
    def __init__(self, out):
        super().__init__()
        self.out = out

    def forward(self, x_t, t, concat_cond=None):
        return self.out


@pytest.mark.parametrize('var_mode', ['FIXED_LARGE', 'FIXED_SMALL'])
def test_kernel_equals_torch_composition_bit_for_bit(cuda, var_mode):
    """mid t, the strided last step (t = 19, noise added) and t = 0 (none added); next input = x_prev in fp16 with zero padding"""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    g = torch.Generator().manual_seed(1)
    B, C, H, W, Cv = 2, 18, 16, 16, 24
    x = (torch.randn(B, C, H, W, generator=g) * 1.3).to(cuda)
    v = (torch.randn(B, H, W, Cv, generator=g) * 1.1).to(cuda)
    d = GaussianDiffusion(_Fixed(v[..., :C].permute(0, 3, 1, 2).contiguous()), betas_cfg=dict(type='linear'), sample_method='ddpm',
                          denoising_var_mode=var_mode)
    cfg = dict(clip_range=[-2, 2])
    for n, step in ((50, 20), (50, 49), (1000, 999)):
        ts = d.ddim_timesteps(n)
        t = int(ts[step])
        coef = d.ddpm_coefficients(ts).to(cuda)
        z = kernel_noise(12345, step, x.shape, cuda)
        nxt = torch.full((B, H, W, 24), 7.0, dtype=torch.float16, device=cuda)
        got = _update(x.clone(), v, coef, step, 12345, next_in=nxt)
        want, _ = d.p_sample_ddpm(x.clone(), t, noise=z, cfg=cfg)
        assert torch.equal(got, want), (var_mode, t, float((got - want).abs().max()))
        assert torch.equal(nxt[..., :C], got.permute(0, 2, 3, 1).half()) and not nxt[..., C:].any()
        if t == 0:
            assert torch.equal(got, d.q_posterior_mean(d.pred_x_0(x, torch.tensor(0, device=cuda), cfg=cfg)[0], x, 0))
        else:
            assert not torch.equal(got, d.q_posterior_mean(d.pred_x_0(x, torch.tensor(t, device=cuda), cfg=cfg)[0], x, t))


def test_generator_repeatable_grid_independent_and_normal(cuda):
    n = 16 * 18 * 128 * 128                    # the bench's batch: 4.7 M values per step
    z = kernel_noise(2024, 3, (1, 1, 1, n), cuda)
    assert torch.equal(z, kernel_noise(2024, 3, (1, 1, 1, n), cuda))
    assert torch.equal(kernel_noise(2024, 3, (1, 1, 1, 1000), cuda), z[..., :1000])          # a prefix of a longer launch
    assert torch.equal(kernel_noise(2024, 3, (16, 18, 128, 128), cuda).flatten(), z.flatten())   # same NCHW index, other grid
    assert torch.isfinite(z).all()
    zd = z.double().flatten()
    mean, var = float(zd.mean()), float(zd.var())
    assert abs(mean) < 5 / math.sqrt(n) and abs(var - 1) < 5 * math.sqrt(2 / n), (mean, var)
    s = zd.sort().values
    cdf = torch.special.ndtr(s)
    i = torch.arange(1, n + 1, device=cuda, dtype=torch.float64)
    ks = float(torch.maximum(i / n - cdf, cdf - (i - 1) / n).max())
    print(f'generator: n {n} mean {mean:.2e} var-1 {var - 1:.2e} KS {ks:.2e} (1% critical {1.63 / math.sqrt(n):.2e})')
    assert ks < 1.63 / math.sqrt(n)
    for other in (kernel_noise(2024, 4, (1, 1, 1, n), cuda), kernel_noise(2025, 3, (1, 1, 1, n), cuda)):
        r = float(torch.corrcoef(torch.stack([zd, other.double().flatten()]))[0, 1])
        assert abs(r) < 5 / math.sqrt(n), r


def _oracle_chain(sd, spec, noise, seed, steps, cuda, clip=(-2, 2), **kw):
    up.fp32_reference_mode()
    sdg = up.state_dict_to(sd, cuda)
    dv = up.diffusion_vars(up.linear_betas())
    zs = (kernel_noise(seed, s, noise.shape, cuda) for s in range(steps))
    return dp.ddpm_sample(lambda x, t: up.unet_forward(sdg, spec, x, t.to(x.device)), noise.to(cuda), dv, zs, num_timesteps=steps,
                          clip_range=clip, **kw)


def _diffusion(m, steps, **kw):
    from ssdnerf_b200.diffusion import GaussianDiffusion
    return GaussianDiffusion(m, betas_cfg=dict(type='linear'), num_timesteps=1000, sample_method='ddpm',
                             test_cfg=dict(num_timesteps=steps, clip_range=[-2, 2], **kw))


def test_small_unet_1000_steps_vs_oracle(cuda):
    sd = up.random_state_dict(_spec(SMALL), seed=21, std=0.04)
    d = _diffusion(_unet(SMALL, sd, cuda), 1000)
    noise = torch.randn(2, 18, 32, 32, generator=torch.Generator().manual_seed(22)).to(cuda)
    torch.manual_seed(5)
    out = d(noise, return_loss=False)
    with torch.no_grad():
        ref = _oracle_chain(sd, _spec(SMALL), noise, _seed_of_call(5), 1000, cuda)
    err = _rel_l2(out, ref)
    print(f'ddpm small UNet 1000 steps rel l2 {err:.3e} (bar {BAR_SMALL:.1e})')
    assert err < BAR_SMALL


def test_cars_unet_50_steps_graph_vs_oracle(cuda):
    """the 122 M-parameter ssdnerf_cars_uncond UNet, 50 strided steps (the last at t = 19 adds noise), B = 2, captured graph"""
    sd = up.random_state_dict(_spec(FULL), seed=7, std=0.02)
    d = _diffusion(_unet(FULL, sd, cuda), 50)
    noise = torch.randn(2, 18, 128, 128, generator=torch.Generator().manual_seed(9)).to(cuda)
    torch.manual_seed(6)
    out = d(noise, return_loss=False)
    assert d._graph_kernel_nodes > 0
    with torch.no_grad():
        ref = _oracle_chain(sd, _spec(FULL), noise, _seed_of_call(6), 50, cuda)
    err = _rel_l2(out, ref)
    print(f'ddpm cars UNet 50 steps B=2 rel l2 {err:.3e} (bar {BAR_CARS:.1e})')
    assert err < BAR_CARS


def test_guided_stepwise_vs_oracle(cuda):
    sd = up.random_state_dict(_spec(SMALL), seed=23, std=0.04)
    d = _diffusion(_unet(SMALL, sd, cuda), 10, guidance_gain=37.5, snr_weight_power=0.25)
    g = torch.Generator().manual_seed(24)
    noise = torch.randn(2, 18, 32, 32, generator=g).to(cuda)
    target = torch.randn(2, 18, 32, 32, generator=g).to(cuda)
    guide = lambda x0: 0.5 * ((x0 - target) ** 2).mean() * x0.size(0)
    zs = [torch.randn(2, 18, 32, 32, generator=g).to(cuda) for _ in range(10)]
    d.denoising.requires_grad_(False)
    out = d(noise, return_loss=False, grad_guide_fn=guide, ddpm_noises=iter(zs))
    up.fp32_reference_mode()
    sdg = up.state_dict_to(sd, cuda)
    ref = dp.ddpm_sample(lambda x, t: up.unet_forward(sdg, _spec(SMALL), x, t.to(x.device)), noise, up.diffusion_vars(up.linear_betas()),
                         iter(zs), num_timesteps=10, clip_range=(-2, 2), grad_guide_fn=guide, guidance_gain=37.5, snr_weight_power=0.25)
    err = _rel_l2(out, ref)
    print(f'ddpm guided 10 steps rel l2 {err:.3e} (bar {BAR_GUIDED:.1e})')
    assert err < BAR_GUIDED


def test_graph_matches_stepwise_seeds_and_recapture(cuda):
    sd = up.random_state_dict(_spec(SMALL), seed=25, std=0.04)
    m = _unet(SMALL, sd, cuda)
    d = _diffusion(m, 8)
    noise = torch.randn(2, 18, 32, 32, generator=torch.Generator().manual_seed(26)).to(cuda)
    torch.manual_seed(3)
    a = d(noise, return_loss=False)
    assert _last_seed(d) == _seed_of_call(3)                               # torch.manual_seed makes a call repeatable
    zs = [kernel_noise(_seed_of_call(3), s, noise.shape, cuda) for s in range(8)]
    b = d(noise, return_loss=False, ddpm_noises=iter(zs))                  # step-wise loop, the graph's own noise
    torch.manual_seed(3)
    c = d(noise, return_loss=False, use_graph=False)                       # the native step uncaptured
    torch.manual_seed(3)
    a2 = d(noise, return_loss=False)
    floor = 1e-3                                                           # fp32 GroupNorm atomics (DESIGN §2), as the DDIM graph test
    print('graph vs step-wise %.2e, vs uncaptured %.2e, repeat %.2e' % (_rel_l2(a, b), _rel_l2(a, c), _rel_l2(a, a2)))
    assert _rel_l2(a, b) < floor and _rel_l2(a, c) < floor and _rel_l2(a, a2) < floor
    torch.manual_seed(4)
    assert _rel_l2(d(noise, return_loss=False), a) > 0.1                    # another seed, another sample
    # a DDIM and a DDPM state of the same shape live side by side; a weight change re-captures; refresh_weights drops both
    d.sample_method = 'ddim'
    d(noise, return_loss=False)
    kinds = sorted(str(k[-1]) for k in d._graphs)
    assert len(d._graphs) == 3 and kinds.count('ddim') == 1, kinds          # ddpm graph + ddpm uncaptured + ddim graph
    d.sample_method = 'ddpm'
    with torch.no_grad():
        [p for p in m.parameters() if p.dim() == 4][-1].mul_(3.0)           # the output convolution
    torch.manual_seed(3)
    a3 = d(noise, return_loss=False)
    torch.manual_seed(3)
    c3 = d(noise, return_loss=False, use_graph=False)
    assert _rel_l2(a3, c3) < floor and _rel_l2(a3, a) > 100 * _rel_l2(a3, c3)
    d.refresh_weights()
    assert not d._graphs


def _config_model(cuda, name, test_over, load_sd=True):
    import ssdnerf_b200 as S
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))[name]
    model_cfg = dict(c['model'], diffusion=dict(c['model']['diffusion'], sample_method='ddpm'))
    torch.manual_seed(0)
    model = S.build_model(model_cfg, train_cfg=c['train_cfg'], test_cfg=dict(c['test_cfg'], **test_over))
    assert model.diffusion_ema.sample_method == 'ddpm'
    sd = up.random_state_dict(up.unet_spec(), seed=7, std=0.02)
    if load_sd:
        for diff in (model.diffusion, model.diffusion_ema):
            diff.denoising.load_state_dict(sd, strict=True)
    else:                                   # a denoiser with dropout has its own key layout: random weights as test_config4_gpu.py draws them
        g = torch.Generator().manual_seed(0)
        for p in model.diffusion_ema.denoising.parameters():
            if p.dim() > 1:
                p.data.copy_(torch.randn(p.shape, generator=g) * 0.02)
    return model.to(cuda).eval(), sd, c


def test_cars_uncond_val_step_ddpm_vs_oracle_chain(cuda, tmp_path):
    model, sd, c = _config_model(cuda, 'configs/paper_cfgs/ssdnerf_cars_uncond.py', dict(num_timesteps=5, n_inverse_steps=0, save_dir=str(tmp_path)))
    B, res = 1, 128
    noise = torch.randn(B, 3, 6, 128, 128, generator=torch.Generator().manual_seed(3)).to(cuda)
    poses = torch.from_numpy(spiral_poses(2))[None].to(cuda)
    intr = torch.tensor([131.25, 131.25, 64.0, 64.0]).expand(B, 2, 4).contiguous().to(cuda)
    torch.manual_seed(11)
    out = model.val_step(dict(scene_id=[0], scene_name=['a'], noise=noise, test_poses=poses, test_intrinsics=intr))
    assert out['pred_imgs'].shape == (B, 2, 3, res, res) and torch.isfinite(out['pred_imgs']).all()
    code = torch.load(os.path.join(tmp_path, 'a.pth'))['param']['code'].to(cuda)[None]
    with torch.no_grad():
        ref = _oracle_chain(sd, up.unet_spec(), model.code_diff_pr(noise).contiguous(), _last_seed(model.diffusion_ema), 5, cuda,
                            clip=tuple(c['test_cfg']['clip_range']))
    err = _rel_l2(model.code_diff_pr(code), ref)
    print(f'cars_uncond val_step ddpm 5 steps rel l2 {err:.3e}')
    assert err < BAR_CARS


def test_chairs_recons1v_guide_optim_ddpm(cuda):
    model, sd, c = _config_model(cuda, 'configs/paper_cfgs/ssdnerf_chairs_recons1v.py',
                                 dict(num_timesteps=3, n_inverse_steps=2, extra_scene_step=1, n_inverse_rays=2 ** 12), load_sd=False)
    assert model.test_cfg['cond_mode'] == 'guide_optim'
    B, res = 1, 128
    g = torch.Generator().manual_seed(4)
    poses = torch.from_numpy(spiral_poses(3))[None].to(cuda)
    intr = torch.tensor([131.25, 131.25, 64.0, 64.0]).expand(B, 3, 4).contiguous().to(cuda)
    code0 = (torch.randn(B, 3, 6, 128, 128, generator=g) * 0.5).to(cuda)
    with torch.no_grad():
        _, bits0 = model.get_density(model.decoder_ema, code0, cfg=dict(density_thresh=0.1))
        img0, _ = model.render(model.decoder_ema, code0, bits0, res, res, intr[:, :1].contiguous(), poses[:, :1].contiguous(), cfg=model.test_cfg)
    noise = torch.randn(B, 3, 6, 128, 128, generator=g).to(cuda)
    seen = []
    orig = model.val_guide
    model.val_guide = lambda *a, **k: seen.append(orig(*a, **k)) or seen[-1]
    data = dict(scene_id=[0], scene_name=['a'], cond_imgs=img0, cond_intrinsics=intr[:, :1].contiguous(), cond_poses=poses[:, :1].contiguous(),
                test_poses=poses[:, 1:].contiguous(), test_intrinsics=intr[:, 1:].contiguous(), noise=noise)
    torch.manual_seed(12)
    out = model.val_step(data)
    assert out['pred_imgs'].shape == (B, 2, 3, res, res) and torch.isfinite(out['pred_imgs']).all()
    guided = seen[-1][0]
    assert torch.isfinite(guided).all()
    with torch.no_grad():
        torch.manual_seed(12)
        uncond = model.code_diff_pr_inv(model.diffusion_ema(model.code_diff_pr(noise), return_loss=False))
    assert _rel_l2(guided, uncond) > 1e-3
