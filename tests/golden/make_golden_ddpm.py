"""Generates tests/golden/reference_ddpm_v1.npz by RUNNING THE REFERENCE'S OWN GaussianDiffusion DDPM sampler (build container only:
`python tests/golden/make_golden_ddpm.py`; the fixture is committed).

It loads lib/models/diffusions/gaussian_diffusion.py and the UNet of lib/models/architecture/ddpm/ from the reference with mmcv / mmgen
stubbed exactly as tests/golden/make_golden_ref.py does (same stubs, same [mmgen-memory] caveat for the inner block bodies), builds the
small UNET_CFG UNet with seeded weights, and records what q_posterior_mean (:156-164), p_sample_ddpm (:333-365) and ddpm_sample
(:367-386) compute.  The noise the reference would draw with `_get_noise_batch` is patched to a seeded iterator.

Stored: the UNet key / shape lists and weight seed (tests/common.py:seeded_weights regenerates the weights), the input x_t, the
generator seeds of every noise sequence and of the guidance target (the tests regenerate them), and the outputs:
  q_posterior_mean at t in {600, 1, 0};
  single p_sample_ddpm steps at t in {600, 1, 0} x {FIXED_LARGE, FIXED_SMALL} x {V, EPS, START_X};
  unguided ddpm_sample over 10 strided steps (last t = 99, noise added) and over all 1000 steps (last t = 0, none added);
  guided ddpm_sample over 10 steps, with grad_through_unet True and False.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden_ref import MODULES, UNET_CFG, _NullLoss, load_reference, seeded_state_dict  # noqa: E402

SHAPE = (1, 18, 16, 16)
WEIGHT_SEED, INPUT_SEED, STEP_NOISE_SEED, CHAIN10_SEED, CHAIN1000_SEED, GUIDE_SEED = 11, 5, 6, 7, 8, 9
TEST_CFG = dict(num_timesteps=10, clip_range=[-2, 2], guidance_gain=37.5, snr_weight_power=0.25)


def noises(seed, n):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(SHAPE, generator=g) for _ in range(n)]


def main():
    mods, den, gd, sm = load_reference()
    MODULES.register_module(name='NullLoss', module=_NullLoss)
    torch.manual_seed(0)
    unet = den.DenoisingUnetMod(**UNET_CFG)
    sd = seeded_state_dict(unet, seed=WEIGHT_SEED)
    unet.load_state_dict(sd)
    unet.eval()
    out = dict(unet_keys=np.array(list(sd.keys())), unet_shapes=np.array([','.join(map(str, v.shape)) for v in sd.values()]),
               weight_seed=np.array(WEIGHT_SEED), step_noise_seed=np.array(STEP_NOISE_SEED), chain10_noise_seed=np.array(CHAIN10_SEED),
               chain1000_noise_seed=np.array(CHAIN1000_SEED), guide_seed=np.array(GUIDE_SEED))
    diff = gd.GaussianDiffusion(denoising=unet, ddpm_loss=dict(type='NullLoss'), betas_cfg=dict(type='linear'), num_timesteps=1000,
                                timestep_sampler=dict(type='SNRWeightedTimeStepSampler', power=0.25), sample_method='ddpm',
                                denoising_var_mode='FIXED_LARGE', denoising_mean_mode='V', test_cfg=dict(TEST_CFG))
    x_t = torch.randn(SHAPE, generator=torch.Generator().manual_seed(INPUT_SEED)) * 1.3
    out['x_t'] = x_t.numpy()
    x0 = x_t.clamp(-1, 1) * 0.7
    out['qpm_x0'] = x0.numpy()
    mod = sys.modules['ref_gaussian_diffusion']
    with torch.no_grad():
        for t in (600, 1, 0):
            out[f'qpm_t{t}'] = diff.q_posterior_mean(x0, x_t, torch.tensor(t)).numpy()
        z = noises(STEP_NOISE_SEED, 1)[0]
        for var_mode in ('FIXED_LARGE', 'FIXED_SMALL'):
            for mean_mode in ('V', 'EPS', 'START_X'):
                diff.denoising_var_mode, diff.denoising_mean_mode = var_mode, mean_mode
                for t in (600, 1, 0):
                    xp, _ = diff.p_sample_ddpm(x_t.clone(), torch.tensor(t), noise=z, cfg=TEST_CFG)
                    out[f'step_{var_mode}_{mean_mode}_t{t}'] = xp.numpy()
        diff.denoising_var_mode, diff.denoising_mean_mode = 'FIXED_LARGE', 'V'
        it = iter(noises(CHAIN10_SEED, 10))
        mod._get_noise_batch = lambda *a, **k: next(it)
        out['ddpm10'] = diff.ddpm_sample(x_t.clone()).numpy()
        diff.test_cfg = dict(TEST_CFG, num_timesteps=1000)
        it = iter(noises(CHAIN1000_SEED, 1000))
        mod._get_noise_batch = lambda *a, **k: next(it)
        out['ddpm1000'] = diff.ddpm_sample(x_t.clone()).numpy()
        diff.test_cfg = dict(TEST_CFG)
    target = torch.randn(SHAPE, generator=torch.Generator().manual_seed(GUIDE_SEED))

    def guide(x0):
        return 0.5 * ((x0 - target) ** 2).mean() * x0.size(0)

    for through, tag in ((True, 'thru'), (False, 'x0')):
        diff.test_cfg = dict(TEST_CFG, grad_through_unet=through)
        it = iter(noises(CHAIN10_SEED, 10))
        mod._get_noise_batch = lambda *a, **k: next(it)
        with torch.no_grad():
            out[f'guided_ddpm10_{tag}'] = diff.ddpm_sample(x_t.clone(), grad_guide_fn=guide).numpy()
    np.savez_compressed(os.path.join(HERE, 'reference_ddpm_v1.npz'), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
