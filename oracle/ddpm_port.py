"""fp32 / float64 restatement of the reference's DDPM sampler -- TEST INFRASTRUCTURE ONLY.

gaussian_diffusion.py:131-164 (posterior tables, q_posterior_mean), :333-386 (p_sample_ddpm, ddpm_sample) and mmgen's var_to_tensor
(the float64 table entry rounded to float32).  It sits beside oracle/unet_port.py's ddim_sample / ddim_sample_guided and reuses their
timesteps and pred_x_0, so guidance follows the same restatement.  V parameterisation.

PINNING: tests/test_ddpm_cpu.py against tests/golden/reference_ddpm_v1.npz, which tests/golden/make_golden_ddpm.py produced by EXECUTING
the reference's own GaussianDiffusion.ddpm_sample with the noise draws injected.
"""
import numpy as np

from .unet_port import ddim_timesteps, pred_x_0


def posterior_coefs(dv):
    """tilde_mu_t_coef1 / tilde_mu_t_coef2 (gaussian_diffusion.py:151-154), float64"""
    betas, ab, ab_prev = dv['betas'], dv['alphas_bar'], dv['alphas_bar_prev']
    return np.sqrt(ab_prev) / (1 - ab) * betas, np.sqrt(1.0 - betas) * (1 - ab_prev) / (1 - ab)


def ddpm_var(dv, var_mode='FIXED_LARGE'):
    """gaussian_diffusion.py:343-349: FIXED_LARGE = [tilde_beta_1, betas...] indexed at t (betas[t - 1] for t >= 1); FIXED_SMALL = tilde_beta_t"""
    if var_mode == 'FIXED_LARGE':
        return np.append(dv['tilde_betas_t'][1], dv['betas'])
    if var_mode == 'FIXED_SMALL':
        return dv['tilde_betas_t']
    raise AttributeError(f'Unknown denoising var output type [{var_mode}].')


def ddpm_sample(denoise_fn, noise, dv, noises, num_timesteps=1000, T=1000, var_mode='FIXED_LARGE', grad_guide_fn=None, clip_denoised=True,
                clip_range=(-1, 1), guidance_gain=1.0, grad_through_unet=True, snr_weight_power=0.5):
    """gaussian_diffusion.py:367-386: at each strided t, x_prev = coef1_t x0 + coef2_t x_t + (t != 0) sqrt(var_t) z with z = next(noises)
    (the tensors the reference draws with _get_noise_batch); coefficients are float32 table entries, sqrt taken in float32"""
    coef1, coef2 = posterior_coefs(dv)
    var = ddpm_var(dv, var_mode)
    x_t = noise
    for t in [int(t) for t in ddim_timesteps(T, num_timesteps)]:
        x0, _ = pred_x_0(denoise_fn, x_t, t, dv, grad_guide_fn=grad_guide_fn, clip_denoised=clip_denoised, clip_range=clip_range,
                         guidance_gain=guidance_gain, grad_through_unet=grad_through_unet, snr_weight_power=snr_weight_power)
        mean = float(np.float32(coef1[t])) * x0 + float(np.float32(coef2[t])) * x_t
        sigma = float(np.sqrt(np.float32(var[t]))) if t != 0 else 0.0
        x_t = mean + sigma * next(noises)
    return x_t
