"""DDPM sampling (sample_method='ddpm') on CPU: the host tables, the package's torch composition of q_posterior_mean / p_sample_ddpm /
the step-wise ddpm_sample and the oracle (oracle/ddpm_port.py) against tests/golden/reference_ddpm_v1.npz, which
tests/golden/make_golden_ddpm.py produced by EXECUTING the reference's own GaussianDiffusion; and argument refusals.

Bars are those of the DDIM pins (tests/test_reference_pin_cpu.py): single steps to round-off, chains 5e-5, guided chains 2e-4."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import ddpm_port as dp
from oracle import unet_port as up
from tests.common import GOLDEN, parse_shapes, seeded_weights

SMALL = dict(image_size=16, in_channels=18, base_channels=32, channels_cfg=(1, 2, 2), resblocks_per_downsample=2,
             attention_res=(8, 4), num_heads=2)
TEST_CFG = dict(num_timesteps=10, clip_range=[-2, 2], guidance_gain=37.5, snr_weight_power=0.25)


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_ddpm_v1.npz'))


def _close(a, b, atol=2e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.abs(a - b).max() <= atol, float(np.abs(a - b).max())


def _noises(ref, key, n):
    g = torch.Generator().manual_seed(int(ref[key]))
    return [torch.randn(1, 18, 16, 16, generator=g) for _ in range(n)]


def _sd(ref):
    return seeded_weights(ref['unet_keys'].tolist(), parse_shapes(ref['unet_shapes']), int(ref['weight_seed']))


class _OracleUNet(torch.nn.Module):
    """oracle UNet behind the nn.Module interface `GaussianDiffusion` drives (CPU stand-in for the CUDA engine)"""

    def __init__(self, ref):
        super().__init__()
        self.spec, sd = up.unet_spec(**SMALL), _sd(ref)
        self.sd = torch.nn.ParameterDict({k.replace('.', '/'): torch.nn.Parameter(v) for k, v in sd.items()})

    def forward(self, x_t, t, label=None, concat_cond=None):
        return up.unet_forward({k.replace('/', '.'): v for k, v in self.sd.items()}, self.spec, x_t, t)


def _diffusion(ref, **kw):
    from ssdnerf_b200.diffusion import GaussianDiffusion
    return GaussianDiffusion(denoising=_OracleUNet(ref), betas_cfg=dict(type='linear'), num_timesteps=1000, sample_method='ddpm',
                             test_cfg=dict(TEST_CFG), **kw)


def _guide(ref):
    target = torch.randn(1, 18, 16, 16, generator=torch.Generator().manual_seed(int(ref['guide_seed'])))
    return lambda x0: 0.5 * ((x0 - target) ** 2).mean() * x0.size(0)


def test_coefficient_rows_are_the_reference_tables_in_float32():
    """rows {sqrt(ab_t), sqrt(1-ab_t), coef1_t, coef2_t, (t != 0) sqrt(var_t)}: float32 of the float64 tables, FIXED_LARGE one off"""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    dv = up.diffusion_vars(up.linear_betas())
    c1, c2 = dp.posterior_coefs(dv)
    for mode in ('FIXED_LARGE', 'FIXED_SMALL'):
        d = GaussianDiffusion(torch.nn.Identity(), betas_cfg=dict(type='linear'), denoising_var_mode=mode)
        np.testing.assert_array_equal(d.tilde_mu_t_coef1, c1)
        np.testing.assert_array_equal(d.tilde_mu_t_coef2, c2)
        for n in (10, 50, 1000):
            ts = d.ddim_timesteps(n)
            rows = d.ddpm_coefficients(ts).numpy()
            assert rows.dtype == np.float32 and rows.shape == (n, 5)
            t = ts.numpy()
            var = np.append(dv['tilde_betas_t'][1], dv['betas'])[t] if mode == 'FIXED_LARGE' else dv['tilde_betas_t'][t]
            expect = np.stack([dv['sqrt_alphas_bar'][t].astype(np.float32), dv['sqrt_one_minus_alphas_bar'][t].astype(np.float32),
                               c1[t].astype(np.float32), c2[t].astype(np.float32),
                               np.where(t != 0, np.sqrt(var.astype(np.float32)), np.float32(0))], axis=1)
            assert np.array_equal(rows, expect)
        rows = d.ddpm_coefficients([999, 500, 1, 0]).numpy()
        assert rows[-1, 4] == 0.0 and rows[-2, 4] > 0.0
        if mode == 'FIXED_LARGE':
            assert rows[1, 4] == np.sqrt(np.float32(dv['betas'][499])) and rows[2, 4] == np.sqrt(np.float32(dv['betas'][0]))
        else:
            assert rows[1, 4] == np.sqrt(np.float32(dv['tilde_betas_t'][500]))
    assert GaussianDiffusion(torch.nn.Identity(), betas_cfg=dict(type='linear')).ddim_timesteps(50)[-1] == 19       # strided: last step adds noise


def test_package_posterior_step_matches_reference(ref):
    """q_posterior_mean and single p_sample_ddpm steps at t = 600, 1, 0 for both variance modes and all three mean modes"""
    d = _diffusion(ref)
    x_t, x0 = torch.from_numpy(ref['x_t']), torch.from_numpy(ref['qpm_x0'])
    z = _noises(ref, 'step_noise_seed', 1)[0]
    for t in (600, 1, 0):
        _close(d.q_posterior_mean(x0, x_t, torch.tensor(t)), ref[f'qpm_t{t}'], 0)
    for var_mode in ('FIXED_LARGE', 'FIXED_SMALL'):
        for mean_mode in ('V', 'EPS', 'START_X'):
            d.denoising_var_mode, d.denoising_mean_mode = var_mode, mean_mode
            for t in (600, 1, 0):
                xp, _ = d.p_sample_ddpm(x_t.clone(), t, noise=z, cfg=TEST_CFG)
                # EPS divides by sqrt(ab_t) ~ 0.06 at t = 600: round-off of the UNet output is amplified there
                _close(xp, ref[f'step_{var_mode}_{mean_mode}_t{t}'], 2e-4 if mean_mode == 'EPS' else 2e-5)


def test_package_stepwise_chains_match_reference(ref):
    """the step-wise ddpm_sample (injected noise): 10 strided steps, all 1000 steps, and guided 10-step chains through the UNet and
    w.r.t. x_0, reached through GaussianDiffusion.forward as val_uncond / val_guide reach it"""
    d = _diffusion(ref)
    x_t = torch.from_numpy(ref['x_t'])
    _close(d(x_t.clone(), return_loss=False, ddpm_noises=iter(_noises(ref, 'chain10_noise_seed', 10))), ref['ddpm10'], 5e-5)
    d.test_cfg = dict(TEST_CFG, num_timesteps=1000)
    _close(d(x_t.clone(), return_loss=False, ddpm_noises=iter(_noises(ref, 'chain1000_noise_seed', 1000))), ref['ddpm1000'], 5e-5)
    for through, tag in ((True, 'thru'), (False, 'x0')):
        d.test_cfg = dict(TEST_CFG, grad_through_unet=through)
        out = d(x_t.clone(), return_loss=False, grad_guide_fn=_guide(ref), ddpm_noises=iter(_noises(ref, 'chain10_noise_seed', 10)))
        _close(out, ref[f'guided_ddpm10_{tag}'], 2e-4)


def test_oracle_ddpm_sample_matches_reference(ref):
    spec, sd = up.unet_spec(**SMALL), _sd(ref)
    den = lambda x, t: up.unet_forward(sd, spec, x, t)
    dv = up.diffusion_vars(up.linear_betas())
    x_t = torch.from_numpy(ref['x_t'])
    kw = dict(clip_range=(-2, 2))
    _close(dp.ddpm_sample(den, x_t, dv, iter(_noises(ref, 'chain10_noise_seed', 10)), num_timesteps=10, **kw), ref['ddpm10'], 5e-5)
    _close(dp.ddpm_sample(den, x_t, dv, iter(_noises(ref, 'chain1000_noise_seed', 1000)), num_timesteps=1000, **kw), ref['ddpm1000'], 5e-5)
    for through, tag in ((True, 'thru'), (False, 'x0')):
        out = dp.ddpm_sample(den, x_t, dv, iter(_noises(ref, 'chain10_noise_seed', 10)), num_timesteps=10, grad_guide_fn=_guide(ref),
                             guidance_gain=37.5, snr_weight_power=0.25, grad_through_unet=through, **kw)
        _close(out, ref[f'guided_ddpm10_{tag}'], 2e-4)


def test_unknown_var_mode_and_save_intermediates_are_refused():
    from ssdnerf_b200.diffusion import GaussianDiffusion
    d = GaussianDiffusion(torch.nn.Identity(), betas_cfg=dict(type='linear'), sample_method='ddpm', denoising_var_mode='LEARNED')
    x = torch.zeros(1, 18, 8, 8)
    with pytest.raises(AttributeError, match=r'Unknown denoising var output type \[LEARNED\]'):
        d(x, return_loss=False)
    with pytest.raises(AttributeError, match='Unknown denoising var output type'):
        d.p_sample_ddpm(x, 10)
    with pytest.raises(AttributeError, match='Unknown denoising var output type'):
        d.ddpm_coefficients([10])
    d.denoising_var_mode = 'FIXED_SMALL'
    with pytest.raises(TypeError, match='save_intermediates'):
        d(x, return_loss=False, save_intermediates=True)
    with pytest.raises(NotImplementedError, match='concat_cond'):
        d(x, return_loss=False, concat_cond=torch.zeros(1, 1, 3, 8, 8))
    # the captured path runs on the native kernels only
    from ssdnerf_b200._lib import SSDNeRFNativeError
    with pytest.raises(SSDNeRFNativeError):
        d(x, return_loss=False)


def test_ddpm_update_rejects_bad_arguments_before_any_launch():
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    u32 = ctypes.c_uint32
    fake = ctypes.c_void_p(1 << 20)                  # never dereferenced: validation fails first

    def call(x_t=fake, v=fake, C=18, Cv=24, coef=fake, step=fake, seed=fake, next_in=fake, Cpad=24):
        return L.ssdnerf_ddpm_update(x_t, v, u32(2), u32(C), u32(16), u32(16), u32(Cv), coef, step, seed, ctypes.c_int(1), ctypes.c_float(-1),
                                     ctypes.c_float(1), next_in, u32(Cpad), None)
    for bad in (dict(x_t=None), dict(v=None), dict(coef=None), dict(step=None), dict(seed=None), dict(Cv=16), dict(Cpad=20), dict(Cpad=16),
                dict(next_in=ctypes.c_void_p((1 << 20) + 8))):
        assert call(**bad) == -2, bad
        assert b'ddpm_update' in L.ssdnerf_last_error()
