"""Pins the oracle (oracle/unet_port.py) and the package's host-side diffusion logic to fixtures produced by EXECUTING the
reference's own denoising.py / modules.py / gaussian_diffusion.py / sampler.py (tests/golden/make_golden_ref.py, run in the build
container; which lines ran from /root/reference and which were mmgen stubs is listed in that file's header).

Bars: float64 schedule tables bit-exact; fp32 tensors to 2e-5 absolute on O(1) values (same arithmetic, different op order)."""
import os

import numpy as np
import pytest
import torch

from oracle import unet_port as up
from oracle.render_port import get_cam_rays as rp_get_cam_rays
from tests.common import GOLDEN, parse_shapes, seeded_weights


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_v1.npz'))


SMALL = dict(image_size=16, in_channels=18, base_channels=32, channels_cfg=(1, 2, 2), resblocks_per_downsample=2,
             attention_res=(8, 4), num_heads=2)
TEST_CFG = dict(num_timesteps=10, clip_range=[-2, 2], guidance_gain=37.5, snr_weight_power=0.25, langevin_steps=2, langevin_delta=0.4)


def _small(ref):
    keys, shapes = ref['unet_keys'].tolist(), parse_shapes(ref['unet_shapes'])
    sd = seeded_weights(keys, shapes, int(ref['unet_weight_seed']))
    assert abs(sum(float(v.double().sum()) for v in sd.values()) - float(ref['unet_weight_checksum'])) < 1e-6
    return up.unet_spec(**SMALL), sd


def _close(a, b, atol=2e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.abs(a - b).max() <= atol, float(np.abs(a - b).max())


def test_state_dict_layout_matches_reference_constructor(ref):
    """keys + shapes the REFERENCE constructor produces (denoising.py:106-187) == the oracle's enumeration == the package's module"""
    spec = up.unet_spec()
    sd = up.random_state_dict(spec, seed=0)
    ref_keys, ref_shapes = ref['full_keys'].tolist(), parse_shapes(ref['full_shapes'])
    assert sorted(sd.keys()) == sorted(ref_keys)
    for k, s in zip(ref_keys, ref_shapes):
        assert tuple(sd[k].shape) == s, k
    assert int(ref['full_numel']) == sum(v.numel() for v in sd.values()) == 122434194
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
                         use_scale_shift_norm=True, num_heads=4, attention_res=[32, 16, 8])
    msd = m.state_dict()
    assert list(msd.keys()) == ref_keys                      # same ORDER too (checkpoint loaders may rely on it)
    assert [tuple(v.shape) for v in msd.values()] == ref_shapes
    md = DenoisingUnetMod(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
                          dropout=0.1, use_scale_shift_norm=True, num_heads=4, attention_res=[32, 16, 8])
    assert list(md.state_dict().keys()) == ref['full_dropout_keys'].tolist()     # conv_2.2 when dropout > 0


def test_unet_forward_and_input_gradient(ref):
    spec, sd = _small(ref)
    assert sorted(sd.keys()) == sorted(up.random_state_dict(spec).keys())
    x, t = torch.from_numpy(ref['unet_x']), torch.from_numpy(ref['unet_t'])
    _close(up.unet_forward(sd, spec, x, t), ref['unet_y'])
    xr = x.clone().requires_grad_(True)
    (up.unet_forward(sd, spec, xr, t) * torch.from_numpy(ref['unet_r'])).sum().backward()
    _close(xr.grad, ref['unet_dx'])


def test_schedule_tables_bit_exact(ref):
    dv = up.diffusion_vars(up.linear_betas())
    for k in ('betas', 'alphas_bar', 'alphas_bar_prev', 'sqrt_alphas_bar', 'sqrt_one_minus_alphas_bar', 'tilde_betas_t'):
        assert np.array_equal(dv[k], ref['lin_' + k]), k
    from ssdnerf_b200.diffusion import GaussianDiffusion
    d = GaussianDiffusion(denoising=torch.nn.Identity(), betas_cfg=dict(type='linear'), num_timesteps=1000)
    for k in ('betas', 'alphas_bar', 'alphas_bar_prev', 'sqrt_alphas_bar', 'sqrt_one_minus_alphas_bar', 'sqrt_recip_alplas_bar',
              'sqrt_recipm1_alphas_bar', 'tilde_betas_t', 'log_tilde_betas_t_clipped', 'tilde_mu_t_coef1', 'tilde_mu_t_coef2'):
        assert np.array_equal(np.asarray(getattr(d, k), np.float64), ref['lin_' + k]), k
    dc = GaussianDiffusion(denoising=torch.nn.Identity(), betas_cfg=dict(type='cosine'), num_timesteps=1000)
    assert np.array_equal(dc.alphas_bar, ref['cos_alphas_bar'])
    assert np.array_equal(up.snr_weighted_loss_weight(dv, 0.25, 'V').numpy(), ref['snr_weight_p025_V'])


def _oracle_denoiser(ref):
    spec, sd = _small(ref)
    return lambda x, t: up.unet_forward(sd, spec, x, t)


def test_oracle_sampler_algebra(ref):
    den = _oracle_denoiser(ref)
    dv = up.diffusion_vars(up.linear_betas())
    x_t = torch.from_numpy(ref['x_t'])
    x0, v = up.pred_x_0(den, x_t, 600, dv, clip_range=(-2, 2))
    _close(x0, ref['pred_x0_t600']); _close(v, ref['pred_v_t600'])
    _close(up.ddim_sample(den, x_t, dv, num_timesteps=10, clip_range=(-2, 2)), ref['ddim10'], 5e-5)
    target = torch.from_numpy(ref['guide_target'])
    guide = lambda x0: 0.5 * ((x0 - target) ** 2).mean() * x0.size(0)
    for through, tag in ((True, 'thru'), (False, 'x0')):
        x0, v = up.pred_x_0(den, x_t, 600, dv, grad_guide_fn=guide, clip_range=(-2, 2), guidance_gain=37.5, snr_weight_power=0.25,
                            grad_through_unet=through, update_denoising_output=True)
        _close(x0, ref[f'guided_x0_{tag}']); _close(v, ref[f'guided_v_{tag}'], 1e-4)
    g2 = torch.Generator().manual_seed(int(ref['langevin_noise_seed']))
    noises = iter([torch.randn(2, 18, 16, 16, generator=g2) for _ in range(18)])
    out = up.ddim_sample_guided(den, x_t, dv, dict(TEST_CFG, langevin_t_range=[0, 1000]), grad_guide_fn=guide, langevin_noises=noises)
    _close(out, ref['guided_langevin_ddim10'], 2e-4)


class _OracleUNet(torch.nn.Module):
    """oracle UNet behind the nn.Module interface `GaussianDiffusion` drives (CPU stand-in for the CUDA engine)"""

    def __init__(self, ref):
        super().__init__()
        self.spec, sd = _small(ref)
        self.sd = torch.nn.ParameterDict({k.replace('.', '/'): torch.nn.Parameter(v) for k, v in sd.items()})

    def forward(self, x_t, t, label=None, concat_cond=None):
        sd = {k.replace('/', '.'): v for k, v in self.sd.items()}
        return up.unet_forward(sd, self.spec, x_t, t)


def test_package_sampler_host_logic_matches_reference(ref):
    """ssdnerf_b200.GaussianDiffusion's step-wise loop (pred_x_0 both guidance routes, p_sample_ddim incl. eta, langevin,
    save_intermediates) on CPU with the oracle UNet as denoiser == what the reference's own loop produced."""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    d = GaussianDiffusion(denoising=_OracleUNet(ref), betas_cfg=dict(type='linear'), num_timesteps=1000, test_cfg=dict(TEST_CFG))
    x_t = torch.from_numpy(ref['x_t'])
    with torch.no_grad():           # unguided pred_x_0 follows the ambient autograd mode (forward_train differentiates through it)
        x0, v = d.pred_x_0(x_t.clone(), torch.tensor(600), cfg=TEST_CFG)
    _close(x0, ref['pred_x0_t600']); _close(v, ref['pred_v_t600'])
    xp, _ = d.p_sample_ddim(x_t.clone(), 600, 500, cfg=TEST_CFG)
    _close(xp, ref['ddim_prev_600_500'])
    xp, _ = d.p_sample_ddim(x_t.clone(), 99, -1, cfg=TEST_CFG)
    _close(xp, ref['ddim_prev_99_last'])
    r = torch.from_numpy(ref['unet_r'])
    xp, _ = d.p_sample_ddim(x_t.clone(), 600, 500, noise=r, cfg=dict(TEST_CFG, eta=0.7))
    _close(xp, ref['ddim_prev_600_500_eta07'])
    _close(d.p_sample_langevin(x_t.clone(), 500, noise=r, cfg=TEST_CFG), ref['langevin_500'])
    d.test_cfg = dict(TEST_CFG, langevin_steps=0)
    inter = d.ddim_sample(x_t.clone(), save_intermediates=True)
    assert len(inter) == 20
    _close(torch.stack([inter[i] for i in (0, 1, 2, 3, 18, 19)]), ref['ddim10_intermediates_0_1_2_3_18_19'], 5e-5)
    _close(inter[-1], ref['ddim10'], 5e-5)
    target = torch.from_numpy(ref['guide_target'])
    guide = lambda x0: 0.5 * ((x0 - target) ** 2).mean() * x0.size(0)
    for through, tag in ((True, 'thru'), (False, 'x0')):
        cfg = dict(TEST_CFG, grad_through_unet=through)
        with torch.no_grad():
            x0, v = d.pred_x_0(x_t.clone(), torch.tensor(600), grad_guide_fn=guide, cfg=cfg, update_denoising_output=True)
        _close(x0, ref[f'guided_x0_{tag}']); _close(v, ref[f'guided_v_{tag}'], 1e-4)
    g2 = torch.Generator().manual_seed(int(ref['langevin_noise_seed']))
    noises = [torch.randn(2, 18, 16, 16, generator=g2) for _ in range(18)]
    d.test_cfg = dict(TEST_CFG, langevin_t_range=[0, 1000])
    out = d.ddim_sample(x_t.clone(), grad_guide_fn=guide, langevin_noises=iter(noises))
    _close(out, ref['guided_langevin_ddim10'], 2e-4)
    eps = torch.from_numpy(ref['q_eps'])
    xq, mean, std = d.q_sample(target, torch.tensor([10, 900]), noise=eps)
    _close(xq, ref['q_sample'])


def test_diffusion_prior_loss_matches_reference(ref):
    """forward_train as val_optim calls it (SNR-weighted v-loss, weight_scale, scale_norm) with the timestep draw and the noise injected:
    loss value and d loss / d x_0 == the reference's GaussianDiffusion.forward_train + DDPMMSELossMod"""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    d = GaussianDiffusion(denoising=_OracleUNet(ref).requires_grad_(False), betas_cfg=dict(type='linear'), num_timesteps=1000,
                          timestep_sampler=dict(type='SNRWeightedTimeStepSampler', power=0.25),
                          ddpm_loss=dict(type='DDPMMSELossMod', rescale_mode='timestep_weight', data_info=dict(pred='v_t_pred', target='v_t'),
                                         weight_scale=4.0, scale_norm=True,
                                         log_cfgs=dict(type='quartile', prefix_name='loss_mse', total_timesteps=1000)))
    d.eval()
    d.ddpm_loss.norm_factor.fill_(0.37)
    assert np.array_equal(d.sampler.weight.numpy(), ref['snr_weight_p025_V'])
    x0 = torch.from_numpy(ref['guide_target']).clone().requires_grad_(True)
    loss, log_vars = d(x0, return_loss=True, cfg=dict(clip_range=[-2, 2]), t=torch.from_numpy(ref['train_t']), noise=torch.from_numpy(ref['q_eps']))
    loss.backward()
    assert abs(float(loss) - float(ref['train_loss'])) <= 1e-5 * abs(float(ref['train_loss']))
    _close(x0.grad, ref['train_dx0'], 1e-6 + 1e-4 * float(np.abs(ref['train_dx0']).max()))
    assert 'loss_ddpm_mse' in log_vars
    # override_cfg semantics of BaseNeRF.train(): eval mode swaps the configured attributes, train mode restores them
    import json, os
    import ssdnerf_b200 as S
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_chairs_recons1v.py']
    c['model']['diffusion']['denoising'].update(base_channels=64, channels_cfg=[1, 2], attention_res=[])      # keep the CPU test light
    m = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg'])
    assert m.diffusion_ema.ddpm_loss.weight_scale == 4.0
    m.eval()
    assert m.diffusion_ema.ddpm_loss.weight_scale == 1.0 and m.diffusion.ddpm_loss.weight_scale == 4.0
    m.train()
    assert m.diffusion_ema.ddpm_loss.weight_scale == 4.0


def test_host_helpers_match_reference_executed(ref):
    """fixtures produced by executing the reference's nerf_utils.get_cam_rays, activation._trunc_exp, RegLoss / TVLoss, TanhCode /
    NormalizedTanhCode and BaseNeRF.ray_sample / get_raybatch_inds (seeded CPU randperm draws)"""
    from oracle import render_port as rp
    from ssdnerf_b200.activation import trunc_exp
    from ssdnerf_b200.nerf import BaseNeRF, NormalizedTanhCode, RegLoss, TanhCode, TVLoss
    # cameras -> rays: the oracle restatement the GPU kernel (ssdnerf_cam_rays / in-kernel make_ray) is tested against
    ro, rd = rp.get_cam_rays(torch.from_numpy(ref['cam_c2w']), torch.from_numpy(ref['cam_intr']), 6, 5)
    assert np.array_equal(ro.numpy(), ref['cam_rays_o'])
    _close(rd, ref['cam_rays_d'], 2e-7)
    # trunc_exp: exp forward (no clamp), gradient clamped to [1e-6, 1e6]
    x = torch.from_numpy(ref['trunc_exp_x']).clone().requires_grad_(True)
    y = trunc_exp(x)
    y.backward(torch.ones_like(y))
    assert np.array_equal(y.detach().numpy(), ref['trunc_exp_y']) and np.array_equal(x.grad.numpy(), ref['trunc_exp_grad'])
    # regularisers of the latent
    code = torch.from_numpy(ref['loss_code'])
    assert abs(float(RegLoss(power=2, loss_weight=3e-3)(code)) - float(ref['reg_loss_p2'])) < 1e-9
    assert abs(float(RegLoss(power=1, loss_weight=0.5)(code)) - float(ref['reg_loss_p1'])) < 1e-7
    assert abs(float(TVLoss(power=1.5, loss_weight=1.0)(code)) - float(ref['tv_loss_p15'])) < 1e-6
    # code activations
    z = torch.from_numpy(ref['act_z'])
    t2 = TanhCode(scale=2)
    _close(t2(z), ref['tanh2_fwd'], 1e-6); _close(t2.inverse(t2(z) * 0.9), ref['tanh2_inv'], 1e-5)
    nt = NormalizedTanhCode(mean=0.0, std=0.5, clip_range=2)
    nt.running_mean.fill_(0.1); nt.running_var.fill_(0.3)
    _close(nt(z), ref['ntanh_fwd'], 1e-6); _close(nt.inverse(nt(z) * 0.9), ref['ntanh_inv'], 1e-5)
    nt.train()
    nt(z, update_stats=True)
    _close(nt.running_mean, ref['ntanh_running_mean_after'], 1e-7); _close(nt.running_var, ref['ntanh_running_var_after'], 1e-7)
    # ray batches: same randperm draws in the same order as the reference
    imgs, rays_o, rays_d = (torch.from_numpy(ref[k]) for k in ('rb_imgs', 'rb_rays_o', 'rb_rays_d'))
    torch.manual_seed(123)
    inds, nb = BaseNeRF.get_raybatch_inds(imgs, 20)
    assert nb == int(ref['rb_num']) and np.array_equal(torch.cat(list(inds), dim=1).numpy(), ref['rb_inds'])
    torch.manual_seed(321)
    o, d, t = BaseNeRF.ray_sample(rays_o, rays_d, imgs, 10)
    assert np.array_equal(o.numpy(), ref['rs_o']) and np.array_equal(d.numpy(), ref['rs_d']) and np.array_equal(t.numpy(), ref['rs_t'])
    o, d, t = BaseNeRF.ray_sample(rays_o, rays_d, imgs, 20, sample_inds=inds[1])
    assert np.array_equal(o.numpy(), ref['rs_o_given']) and np.array_equal(t.numpy(), ref['rs_t_given'])


def test_stage2_train_step_matches_reference_execution(ref):
    """`DiffusionNeRF.train_step` (stage 2: stored scenes, denoiser optimizer only) for two consecutive iterations vs the fixture produced
    by executing the reference's own train_step / forward_train / DDPMMSELossMod (training mode) / load_scene
    (tests/golden/make_golden_train_step.py): loss, log_vars, running norm factor and the SGD-updated denoiser weights.  The oracle UNet stands
    in for the CUDA engine (same seeded weights as the reference UNet of the fixture); timestep draw and noise are injected on both sides."""
    import ssdnerf_b200 as S
    tr = np.load(os.path.join(GOLDEN, 'reference_train_step_v1.npz'))
    m = S.build_model(dict(
        type='DiffusionNeRF', code_size=(3, 6, 16, 16), code_reshape=(18, 16, 16), grid_size=8, diffusion_use_ema=False, decoder_use_ema=True,
        freeze_decoder=True, decoder=dict(type='TriPlaneDecoder', base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3],
                                          use_dir_enc=True, dir_layers=[16, 64]),
        diffusion=dict(type='GaussianDiffusion', num_timesteps=1000, betas_cfg=dict(type='linear'), denoising_mean_mode='V',
                       denoising=dict(type='DenoisingUnetMod', image_size=16, in_channels=18, base_channels=64, channels_cfg=[1],
                                      resblocks_per_downsample=1, use_scale_shift_norm=True, attention_res=[]),
                       timestep_sampler=dict(type='SNRWeightedTimeStepSampler', power=0.5),
                       ddpm_loss=dict(type='DDPMMSELossMod', rescale_mode='timestep_weight', data_info=dict(pred='v_t_pred', target='v_t'),
                                      weight_scale=4.0, scale_norm=True, loss_name='loss_ddpm_mse'))), train_cfg=dict(), test_cfg=dict())
    unet = _OracleUNet(ref)
    m.diffusion.denoising = unet
    m.train()
    assert all(p.requires_grad for p in unet.parameters()) and not any(p.requires_grad for p in m.decoder.parameters())
    opt = dict(diffusion=torch.optim.SGD(m.diffusion.parameters(), lr=float(tr['lr'])))
    data = dict(scene_id=[0, 1], scene_name=['a', 'b'], code=[dict(param=dict(code=torch.from_numpy(c))) for c in tr['codes']])
    plain = m.diffusion.forward_train
    for it in range(2):
        t, noise = torch.from_numpy(tr['t'][it]), torch.from_numpy(tr['noise'][it])
        m.diffusion.forward_train = lambda x0, t=t, noise=noise, **kw: plain(x0, t=t, noise=noise, **kw)
        res = m.train_step(data, opt)
        lv = res['log_vars']
        assert sorted(lv.keys()) == list(tr[f'it{it}_log_keys']) and res['num_samples'] == int(tr[f'it{it}_num_samples'])
        assert abs(lv['loss_ddpm_mse'] - float(tr[f'it{it}_loss'])) <= 2e-5 * abs(float(tr[f'it{it}_loss'])), (it, lv)
        _close(m.diffusion.ddpm_loss.norm_factor, tr[f'it{it}_norm_factor'], 1e-7)
        sd = {k.replace('/', '.'): v.detach() for k, v in unet.sd.items()}
        for k in tr['probe_names']:
            ref_w = tr[f'it{it}_{k}']
            _close(sd[str(k)], ref_w, 2e-6 + 2e-5 * float(np.abs(ref_w).max()))
        chk = sum(float(v.double().abs().sum()) for v in sd.values())
        assert abs(chk - float(tr[f'it{it}_param_checksum'])) <= 1e-6 * float(tr[f'it{it}_param_checksum'])


def _replay_checks(jt, tag, model, res, decoder, atol=2e-6):
    lv = res['log_vars']
    assert sorted(lv.keys()) == list(jt[f'{tag}_log_keys']), (sorted(lv.keys()), list(jt[f'{tag}_log_keys']))
    got = np.array([lv[k] for k in sorted(lv.keys())], np.float64)
    np.testing.assert_allclose(got, jt[f'{tag}_log_vals'], rtol=5e-5, atol=1e-7, err_msg=f'{tag} log_vars {sorted(lv.keys())}')
    assert res['num_samples'] == int(jt[f'{tag}_num_samples'])
    for k, v in decoder.state_dict().items():
        _close(v, jt[f'{tag}_dec_{k}'], atol)
    _close(model.init_code, jt[f'{tag}_init_code'], atol)
    for sid, e in model.cache.items():
        assert (e is not None) == bool(jt[f'{tag}_cache{sid}_filled']), (tag, sid)
        if e is not None:
            assert e['param']['code_'].dtype == torch.float16
            _close(e['param']['code_'].float(), jt[f'{tag}_cache{sid}_code'], 1e-3)          # fp16 storage: one ulp at |x| <= 2 is 9.8e-4
            assert float(e['optimizer']['state'][0]['step']) == float(jt[f'{tag}_cache{sid}_step'])
            _close(e['optimizer']['state'][0]['exp_avg'].float(), jt[f'{tag}_cache{sid}_exp_avg'], 2e-3)


def test_joint_train_steps_match_reference_execution(ref, monkeypatch):
    """`MultiSceneNeRF.train_step` (stage 1) and `DiffusionNeRF.train_step` (single stage), two iterations each over overlapping scene sets,
    vs the fixture produced by executing the reference's own train_steps through their real constructors
    (tests/golden/make_golden_joint_step.py).  Both sides use tests/common.py:ToyDecoder as the renderer and skip the occupancy update (the
    reference's needs its CUDA extension); log_vars, decoder weights after Adam, the running mean code, every cache entry (latent, Adam
    step count and first moment) and, for the single-stage step, the SGD-updated denoiser and its loss normaliser are compared."""
    import ssdnerf_b200 as S
    from ssdnerf_b200 import nerf as nerf_mod
    from tests.common import ToyDecoder
    jt = np.load(os.path.join(GOLDEN, 'reference_joint_step_v1.npz'))
    tr = np.load(os.path.join(GOLDEN, 'reference_train_step_v1.npz'))
    if 'ToyDecoder' not in S.MODULES._module_dict:
        S.MODULES.register_module(name='ToyDecoder', module=ToyDecoder)
    monkeypatch.setattr(nerf_mod.R, 'get_cam_rays', lambda c2w, intr, h, w: rp_get_cam_rays(c2w, intr, h, w))
    train1 = dict(optimizer=dict(type='Adam', lr=0.01, weight_decay=0.0), n_decoder_rays=40, n_inverse_rays=48, extra_scene_step=3,
                  loss_coef=0.01, dt_gamma_scale=0.5, density_thresh=0.1)
    model1 = dict(code_size=(3, 6, 8, 8), grid_size=8, code_activation=dict(type='TanhCode', scale=2), bg_color=1, init_from_mean=True,
                  pixel_loss=dict(type='MSELoss', loss_weight=20.0), reg_loss=dict(type='TVLoss', power=1.5, loss_weight=1.0),
                  decoder=dict(type='ToyDecoder'), decoder_use_ema=False, cache_size=3, cache_16bit=True)
    imgs, poses, intr = (torch.from_numpy(jt[k]) for k in ('s1_imgs', 's1_poses', 's1_intr'))

    def batch(ids):
        return dict(scene_id=ids, scene_name=[f's{i}' for i in ids], cond_imgs=imgs[ids], cond_poses=poses[ids], cond_intrinsics=intr[ids])
    # ---- stage 1
    m1 = S.build_model(dict(type='MultiSceneNeRF', **model1), train_cfg=dict(train1), test_cfg=dict())
    m1.update_extra_state = lambda *a, **k: None
    m1.train()
    opt = dict(decoder=torch.optim.Adam(m1.decoder.parameters(), lr=1e-3))
    torch.manual_seed(123)
    for it, ids in enumerate(([2, 0], [0, 1])):
        _replay_checks(jt, f's1_it{it}', m1, m1.train_step(batch(ids), opt), m1.decoder)
    # ---- single stage
    m2 = S.build_model(dict(
        type='DiffusionNeRF', **dict(model1, code_size=(3, 6, 16, 16)), code_reshape=(18, 16, 16), freeze_decoder=False, diffusion_use_ema=False,
        diffusion=dict(type='GaussianDiffusion', num_timesteps=1000, betas_cfg=dict(type='linear'), denoising_mean_mode='V',
                       denoising=dict(type='DenoisingUnetMod', image_size=16, in_channels=18, base_channels=64, channels_cfg=[1],
                                      resblocks_per_downsample=1, use_scale_shift_norm=True, attention_res=[]),
                       timestep_sampler=dict(type='SNRWeightedTimeStepSampler', power=0.5),
                       ddpm_loss=dict(type='DDPMMSELossMod', rescale_mode='timestep_weight', data_info=dict(pred='v_t_pred', target='v_t'),
                                      weight_scale=4.0, scale_norm=True, loss_name='loss_ddpm_mse'))),
        train_cfg=dict(train1, optimizer=dict(type='Adam', lr=0.005, weight_decay=0.0), extra_scene_step=2), test_cfg=dict())
    unet = _OracleUNet(ref)
    m2.diffusion.denoising = unet
    m2.update_extra_state = lambda *a, **k: None
    m2.train()
    opt = dict(diffusion=torch.optim.SGD(m2.diffusion.parameters(), lr=0.05), decoder=torch.optim.Adam(m2.decoder.parameters(), lr=1e-3))
    plain = m2.diffusion.forward_train
    torch.manual_seed(321)
    for it, ids in enumerate(([2, 0], [0, 1])):
        t, noise = torch.from_numpy(jt['s2_t'][it]), torch.from_numpy(jt['s2_noise'][it])
        m2.diffusion.forward_train = lambda x0, t=t, noise=noise, **kw: plain(x0, t=t, noise=noise, **kw)
        tag = f's2_it{it}'
        _replay_checks(jt, tag, m2, m2.train_step(batch(ids), opt), m2.decoder)
        _close(m2.diffusion.ddpm_loss.norm_factor, jt[f'{tag}_norm_factor'], 1e-7)
        sd = {k.replace('/', '.'): v.detach() for k, v in unet.sd.items()}
        for k in tr['probe_names']:
            w = jt[f'{tag}_unet_{k}']
            _close(sd[str(k)], w, 2e-6 + 2e-5 * float(np.abs(w).max()))
        chk = sum(float(v.double().abs().sum()) for v in sd.values())
        assert abs(chk - float(jt[f'{tag}_unet_checksum'])) <= 1e-6 * float(jt[f'{tag}_unet_checksum'])


def test_val_paths_match_reference_execution(ref, monkeypatch):
    """BASELINE config 4's host logic: `val_guide` (render-loss guidance through the denoiser + langevin), `val_optim` (diffusion-prior
    gradient, inner render-loss Adam steps from that gradient, ExponentialLR) and `val_uncond` (intermediates list + prior-only refinement)
    vs the fixture produced by executing the reference's own methods through the real `DiffusionNeRF` constructor
    (tests/golden/make_golden_val.py; toy renderer and no-op occupancy calls on both sides, draws injected)."""
    import ssdnerf_b200 as S
    from ssdnerf_b200 import nerf as nerf_mod
    from tests.common import ToyDecoder
    vf = np.load(os.path.join(GOLDEN, 'reference_val_v1.npz'))
    if 'ToyDecoder' not in S.MODULES._module_dict:
        S.MODULES.register_module(name='ToyDecoder', module=ToyDecoder)
    monkeypatch.setattr(nerf_mod.R, 'get_cam_rays', lambda c2w, intr, h, w: rp_get_cam_rays(c2w, intr, h, w))
    test_cfg = dict(num_timesteps=4, clip_range=[-2, 2], guidance_gain=50.0, snr_weight_power=0.25, langevin_steps=1, langevin_delta=0.4,
                    n_inverse_rays=48, n_inverse_steps=3, extra_scene_step=2, optimizer=dict(type='Adam', lr=0.005, weight_decay=0.0),
                    lr_scheduler=dict(type='ExponentialLR', gamma=0.9), loss_coef=0.01, dt_gamma_scale=0.5, density_thresh=0.1)
    m = S.build_model(dict(
        type='DiffusionNeRF', code_size=(3, 6, 16, 16), grid_size=8, code_activation=dict(type='TanhCode', scale=2), bg_color=1,
        pixel_loss=dict(type='MSELoss', loss_weight=20.0), reg_loss=dict(type='TVLoss', power=1.5, loss_weight=1.0),
        decoder=dict(type='ToyDecoder'), decoder_use_ema=False, code_reshape=(18, 16, 16), freeze_decoder=True, diffusion_use_ema=False,
        diffusion=dict(type='GaussianDiffusion', num_timesteps=1000, betas_cfg=dict(type='linear'), denoising_mean_mode='V',
                       denoising=dict(type='DenoisingUnetMod', image_size=16, in_channels=18, base_channels=64, channels_cfg=[1],
                                      resblocks_per_downsample=1, use_scale_shift_norm=True, attention_res=[]),
                       timestep_sampler=dict(type='SNRWeightedTimeStepSampler', power=0.25),
                       ddpm_loss=dict(type='DDPMMSELossMod', rescale_mode='timestep_weight', data_info=dict(pred='v_t_pred', target='v_t'),
                                      weight_scale=4.0, scale_norm=True, loss_name='loss_ddpm_mse'))), train_cfg=dict(), test_cfg=dict(test_cfg))
    m.diffusion.denoising = _OracleUNet(ref)
    m.update_extra_state = lambda *a, **k: None
    m.get_density = lambda decoder, code, cfg=dict(): (torch.zeros(code.size(0), 8 ** 3), torch.zeros(code.size(0), 8 ** 3 // 8, dtype=torch.uint8))
    m.eval()
    m.diffusion.ddpm_loss.norm_factor.fill_(0.6)
    t = lambda k: torch.from_numpy(vf[k])
    lang, ts, eps = list(t('lang')), list(t('ts')), list(t('eps'))
    data = dict(scene_id=[0, 1], scene_name=['a', 'b'], cond_imgs=t('imgs'), cond_poses=t('poses'), cond_intrinsics=t('intr'), noise=t('noise'))
    plain = m.diffusion.forward_train

    def inject(t_list, n_list):
        it_t, it_n = iter(t_list), iter(n_list)
        m.diffusion.forward_train = lambda x0, **kw: plain(x0, t=next(it_t), noise=next(it_n), **kw)
    # ---- guided sampling
    torch.manual_seed(77)
    with torch.no_grad():
        code, _, _ = m.val_guide(data, langevin_noises=iter(lang[:3]))
    err = float((code - t('guide_code')).abs().max())
    print('val_guide max abs diff vs reference execution', err)
    _close(code, vf['guide_code'], 2e-4)
    # ---- code optimisation with the diffusion prior
    inject(ts, eps)
    torch.manual_seed(78)
    with torch.no_grad():
        code, _, _ = m.val_optim(data, code_=t('code0').clone().requires_grad_(True))
    print('val_optim max abs diff', float((code - t('optim_code')).abs().max()))
    _close(code, vf['optim_code'], 5e-5)
    # ---- unconditional sampling with intermediates + prior-only refinement (the fixture's draw order: 3 langevin, then 3 loss noises)
    assert int(vf['uncond_noise_calls']) == 6
    inject(ts[3:], [lang[3], eps[3], eps[4]])
    torch.manual_seed(79)
    with torch.no_grad():
        codes, grids, bits = m.val_uncond(dict(scene_id=[0, 1], noise=t('noise')), save_intermediates=True, langevin_noises=iter(lang[:3]))
    assert len(codes) == int(vf['uncond_len']) == len(grids) == len(bits)
    _close(codes[0], vf['uncond_first'], 5e-5)
    _close(codes[-1], vf['uncond_last'], 2e-4)


def test_renderer_oracle_matches_reference_decoder_execution():
    """The oracle restatements every GPU parity test of the fused renderers is measured against -- `render_port.point_decode`,
    `render_port.render_eval_scene` (host loop of base_volume_renderer.py:79-123) and `train_port.render_train_scene` (train branch + K7 / K8
    through autograd) -- vs the fixture produced by executing the reference's OWN `TriPlaneDecoder` and op wrappers over a `_backend` that
    forwards to the kernel-exact C oracle (tests/golden/make_golden_decoder.py).  Also: our TriPlaneDecoder's state-dict layout."""
    import ssdnerf_b200 as S
    from oracle import render_port as rp
    from oracle import train_port as tp
    from tests.common import spiral_poses
    D = np.load(os.path.join(GOLDEN, 'reference_decoder_v1.npz'))
    res = 24
    f = 131.25 * res / 128
    poses = torch.from_numpy(spiral_poses(2)).float()
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(2, 4).contiguous()
    ro, rd = rp.get_cam_rays(poses, intr, res, res)
    ro, rd = ro.reshape(2, -1, 3).contiguous(), rd.reshape(2, -1, 3).contiguous()
    bits = np.stack([rp.sphere_bitfield(radius=0.7), rp.sphere_bitfield(radius=0.5)])
    dt_gamma = [0.0, 0.004]
    cfgs = dict(P=dict(type='TriPlaneDecoder', base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3], use_dir_enc=True,
                       dir_layers=[16, 64], max_steps=256), S=dict(type='TriPlaneDecoder', max_steps=256))
    for variant in ('P', 'S'):
        C = 6 if variant == 'P' else 32
        g = torch.Generator().manual_seed(int(D[f'{variant}_code_seed']))
        code = (torch.randn(2, 3, C, 128, 128, generator=g) * 0.7).clamp(-2, 2)
        params = rp.make_decoder_params(variant, 4)
        params['density_net.0.bias'] = params['density_net.0.bias'] + 1.0
        assert list(S.build_module(cfgs[variant]).state_dict().keys()) == list(D[f'{variant}_state_keys'])
        # point_decode on the fixture's explicit points
        xyz, dirs, counts = torch.from_numpy(D[f'{variant}_pd_xyz']), torch.from_numpy(D[f'{variant}_pd_dirs']), D[f'{variant}_pd_counts']
        o = 0
        for b, n in enumerate(counts):
            sig, rgb = rp.point_decode(params, xyz[o:o + n], dirs[o:o + n], code[b])
            _close(sig, D[f'{variant}_pd_sigma'][o:o + n], 1e-5 * float(np.abs(D[f'{variant}_pd_sigma']).max()))
            _close(rgb, D[f'{variant}_pd_rgb'][o:o + n], 2e-6)
            o += n
        # eval branch
        for b in range(2):
            r = rp.render_eval_scene(params, ro[b].numpy(), rd[b].numpy(), code[b], bits[b], max_steps=256, dt_gamma=dt_gamma[b])
            for k in ('weights_sum', 'depth', 'image'):
                err = float(np.abs(r[k] - D[f'{variant}_eval_{k}'][b]).max())
                assert err <= 2e-6, (variant, b, k, err)
            assert float(D[f'{variant}_eval_weights_sum'][b].max()) > 0.5          # the rays do hit something
    # train branch (variant P): forward, d loss / d code, d loss / d decoder weights
    g = torch.Generator().manual_seed(int(D['P_code_seed']))
    code = (torch.randn(2, 3, 6, 128, 128, generator=g) * 0.7).clamp(-2, 2)
    params = rp.make_decoder_params('P', 4)
    params['density_net.0.bias'] = params['density_net.0.bias'] + 1.0
    pref = {k: torch.as_tensor(v).double().requires_grad_(True) for k, v in params.items()}
    cref = code.double().requires_grad_(True)
    sel = torch.from_numpy(D['P_train_sel'])
    gi, gw = torch.from_numpy(D['P_train_gi']).double(), torch.from_numpy(D['P_train_gw']).double()
    tot = 0
    for b in range(2):
        ws, dep, img = tp.render_train_scene(pref, cref[b], ro[b][sel[b]].numpy(), rd[b][sel[b]].numpy(), bits[b], None, dt_gamma=dt_gamma[b])
        for k, v in (('weights_sum', ws), ('depth', dep), ('image', img)):
            _close(v.detach(), D[f'P_train_{k}'][b], 5e-6)
        tot = tot + (img * gi[b]).sum() + (ws * gw[b]).sum()
    names = [k for k in pref if f'P_train_grad_{k}' in D.files]
    assert len(names) == 8
    grads = torch.autograd.grad(tot, [cref] + [pref[k] for k in names])
    rel = lambda a, b: float((a - torch.from_numpy(b).double()).norm() / np.linalg.norm(b))
    assert rel(grads[0], D['P_train_grad_code']) < 2e-5, rel(grads[0], D['P_train_grad_code'])
    for k, gk in zip(names, grads[1:]):
        assert rel(gk, D[f'P_train_grad_{k}']) < 2e-5, (k, rel(gk, D[f'P_train_grad_{k}']))
    assert bool(D['P_train_decoder_reg_loss_is_none'])


def test_density_oracle_matches_reference_execution():
    """`render_port.get_density` / `update_extra_state` (the restatement the GPU occupancy-grid kernels are measured against) vs the fixture
    produced by executing the reference's own `BaseNeRF.get_density` / `update_extra_state` + `point_density_decode` + morton / packbits
    wrappers over the kernel-exact C backend (tests/golden/make_golden_density.py): bitfields bit-exact, grid values to fp16 / fp32 round-off."""
    from oracle import render_port as rp
    D = np.load(os.path.join(GOLDEN, 'reference_density_v1.npz'))
    g = torch.Generator().manual_seed(21)
    code = (torch.randn(2, 3, 6, 128, 128, generator=g) * 0.7).clamp(-2, 2)
    params = rp.make_decoder_params('P', 6)
    params['density_net.0.bias'] = params['density_net.0.bias'] - 2.5
    torch.manual_seed(5)
    rands = [torch.rand(64 ** 3, 3) for _ in range(3)]                  # the reference draws torch.rand_like(xyzs) once per iteration
    grid, bits = rp.get_density(params, code, rands, density_thresh=0.1)
    assert str(grid.dtype) == str(D['gd_grid_dtype']) == 'torch.float16'
    diff = np.unpackbits(bits) != np.unpackbits(D['gd_bits'])
    assert diff.mean() <= 2e-5, diff.mean()                              # a voxel exactly at the threshold may flip with 1-ulp decode differences
    _close(grid.float()[:, ::37], D['gd_grid_sub'], 2e-3 * float(D['gd_grid_sub'].max()))
    assert abs(float(grid.double().sum()) - float(D['gd_grid_sum'])) <= 1e-4 * float(D['gd_grid_sum'])
    assert 0.2 < np.unpackbits(D['gd_bits']).mean() < 0.8
    grid2 = torch.zeros(2, 64 ** 3)
    torch.manual_seed(6)
    for i in range(2):
        bits2, _ = rp.update_extra_state(params, code * (1.0 if i == 0 else 0.5), grid2, torch.rand(64 ** 3, 3), density_thresh=0.08, decay=0.9)
        _close(grid2[:, ::37], D[f'ue_grid_sub_{i}'], 2e-6 * float(D[f'ue_grid_sub_{i}'].max()) + 1e-7)
        diff = np.unpackbits(bits2) != np.unpackbits(D[f'ue_bits_{i}'])
        assert diff.mean() <= 2e-5, (i, diff.mean())


def _train_edges_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_golden_decoder', os.path.join(GOLDEN, 'make_golden_decoder.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize('name', ['floor', 'ones', 'plane96x160', 'budget32'])
def test_train_oracle_matches_reference_at_the_edges(name):
    """`train_port.render_train_scene` vs the reference's own `TriPlaneDecoder` train branch (tests/golden/make_golden_decoder.py
    --train-edges) where its edge rules act: TruncExp's gradient floor (density bias -22), the plane borders (all-ones grid), 96 x 160
    planes and a binding sample budget (max_steps 32).  Forward to 5e-6, code and all eight decoder-parameter gradients to relative L2
    2e-5.  At the floor the reference's float32 alpha is exactly 0 and the density path is the floor alone; the float64 oracle's alpha is
    not, and it differs from float32 by about 1e-4 there, so that case is pinned with the oracle run in float32, the reference's own
    precision."""
    from oracle import train_port as tp
    M = _train_edges_module()
    D = np.load(os.path.join(GOLDEN, 'reference_train_edges_v1.npz'))
    inp = M.train_edge_inputs(name)
    dtype = torch.float32 if name == 'floor' else torch.float64
    sel = torch.from_numpy(D[f'{name}_sel'].astype(np.int64))
    gi, gw = torch.from_numpy(D[f'{name}_gi']).to(dtype), torch.from_numpy(D[f'{name}_gw']).to(dtype)
    gcode = np.zeros(inp['code'].numel(), np.float32)
    gcode[np.cumsum(D[f'{name}_grad_code_idx_diff'])] = D[f'{name}_grad_code_val']
    gcode = gcode.reshape(inp['code'].shape)

    def run(trunc_exp):
        pref = {k: torch.as_tensor(v).to(dtype).requires_grad_(True) for k, v in inp['params'].items()}
        cref = inp['code'].to(dtype).requires_grad_(True)
        tot, outs = 0, []
        for b in range(2):
            ws, dep, img, smp = tp.render_train_scene(pref, cref[b], inp['rays_o'][b][sel[b]].numpy(), inp['rays_d'][b][sel[b]].numpy(), inp['bits'][b],
                                                      None, dt_gamma=M.TRAIN_EDGE_DT_GAMMA[b], max_steps=inp['max_steps'], dtype=dtype,
                                                      trunc_exp=trunc_exp, return_samples=True)
            outs.append((ws, dep, img, smp))
            tot = tot + (img * gi[b]).sum() + (ws * gw[b]).sum()
        names = [k for k in pref if f'{name}_grad_{k}' in D.files]
        return outs, dict(zip(['code'] + names, torch.autograd.grad(tot, [cref] + [pref[k] for k in names])))

    def rel(a, b):
        nb = float(np.linalg.norm(b))
        return float((a.double() - torch.from_numpy(b).double()).norm()) / max(nb, 1e-30)

    outs, grads = run(True)
    assert len(grads) == 9
    for b, (ws, dep, img, smp) in enumerate(outs):
        for k, v in (('weights_sum', ws), ('depth', dep), ('image', img)):
            _close(v.detach(), D[f'{name}_{k}'][b], 5e-6)
    assert rel(grads['code'], gcode) < 2e-5, rel(grads['code'], gcode)
    for k in list(grads)[1:]:
        assert rel(grads[k], D[f'{name}_grad_{k}']) < 2e-5, (k, rel(grads[k], D[f'{name}_grad_{k}']))
    # each case is in the regime it is named for
    counts = np.concatenate([smp['counts'] for *_, smp in outs])
    if name == 'budget32':
        assert (counts == 32).mean() >= 0.25, (counts == 32).mean()
    else:
        assert counts.max() < inp['max_steps']
    if name == 'floor':
        assert float(np.abs(D['floor_weights_sum']).max()) == 0.0          # float32 alpha underflows to 0: the floor drives every gradient
        _, grads_exp = run(False)                                        # plain exp's gradient misses the reference by far
        k = 'density_net.0.bias'
        assert rel(grads_exp[k], D[f'{name}_grad_{k}']) > 0.5, rel(grads_exp[k], D[f'{name}_grad_{k}'])
    if name in ('ones', 'budget32'):
        assert float(D[f'{name}_weights_sum'].max()) > 0.5
    if name == 'ones':                                                   # samples within half a texel of a plane edge
        xyzs = np.concatenate([smp['xyzs'] for *_, smp in outs])
        assert (np.abs(xyzs) > 1 - 1 / 128).any(axis=1).mean() >= 0.01


def test_oracle_trunc_exp_matches_reference_executed(ref):
    """the oracle's TruncExp (render_port.point_decode's density activation) is bit-equal to the reference's _trunc_exp, forward and
    backward, on the fixture's inputs, which straddle both clamp bounds of the gradient"""
    from oracle.render_port import TruncExp
    x = torch.from_numpy(ref['trunc_exp_x']).clone().requires_grad_(True)
    y = TruncExp.apply(x)
    y.backward(torch.ones_like(y))
    assert np.array_equal(y.detach().numpy(), ref['trunc_exp_y']) and np.array_equal(x.grad.numpy(), ref['trunc_exp_grad'])
    assert (ref['trunc_exp_x'] < np.log(1e-6)).any() and (ref['trunc_exp_x'] > np.log(1e6)).any()
