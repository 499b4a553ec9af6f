"""`ssdnerf_cars_recons1v_tiled` (reference config, resolved fixture) through the public entry point: `DiffusionNeRF.val_step`
unconditionally and in its own test mode `guide_optim`, at reduced sizes (one scene, fewer views, DDIM / inverse / inner steps).
The denoiser runs on the 6 x 128 x 384 latent that `code_permute` / `code_reshape` make of the 3 x 6 x 128 x 128 code; the
unconditional sample is compared with the fp32 oracle chain (tests/unet_tiled_oracle.py) on the same noise.  Training this model
raises NotImplementedError."""
import json
import os

import pytest
import torch

from oracle import unet_port as up
from tests import unet_tiled_oracle as uto
from tests.common import GOLDEN, spiral_poses

pytestmark = pytest.mark.gpu

NAME = 'configs/new_cfgs/ssdnerf_cars_recons1v_tiled.py'


def _rel_l2(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _spec():
    return up.unet_spec(image_size=128, in_channels=6, base_channels=80, channels_cfg=(1, 1, 2, 2, 4, 4), resblocks_per_downsample=2,
                        attention_res=(16, 8, 4), num_heads=4)


def _model(cuda, test_over, seed=7, cache_size=0, **train_over):
    import ssdnerf_b200 as S
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))[NAME]
    dcfg = c['model']['diffusion']
    assert dcfg['num_timesteps'] == 1000 and dcfg['betas_cfg'] == dict(type='linear')
    assert c['model']['code_reshape'] == [6, 128, 384] and c['model']['diffusion']['denoising']['norm_cfg']['num_groups'] == 16
    test_cfg = dict(c['test_cfg'], **test_over)
    torch.manual_seed(0)
    train_cfg = {k: v for k, v in c['train_cfg'].items() if k != 'cache_load_from'}
    train_cfg.update(train_over)
    model = S.build_model(dict(c['model'], cache_size=cache_size), train_cfg=train_cfg, test_cfg=test_cfg)
    sd = up.random_state_dict(_spec(), seed=seed, std=0.02)
    for diff in (model.diffusion, model.diffusion_ema):
        diff.denoising.load_state_dict(sd, strict=True)
    return model.to(cuda).eval(), sd, c


def _capture(model, name):
    """record what model.<name> returns while val_step runs"""
    seen = []
    orig = getattr(model, name)

    def wrapped(*a, **k):
        out = orig(*a, **k)
        seen.append(out)
        return out
    setattr(model, name, wrapped)
    return seen


def test_tiled_val_step_unconditional_vs_oracle_chain(cuda):
    model, sd, c = _model(cuda, dict(num_timesteps=8, n_inverse_steps=0))
    B, res = 1, 128                     # test_cfg img_size: the views are rendered at 128 x 128
    g = torch.Generator().manual_seed(3)
    noise = torch.randn(B, 3, 6, 128, 128, generator=g)
    poses = torch.from_numpy(spiral_poses(2))[None].to(cuda)
    f = 131.25 * res / 128
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(B, 2, 4).contiguous().to(cuda)
    seen = _capture(model, 'val_uncond')
    out = model.val_step(dict(scene_id=[0], scene_name=['a'], noise=noise.to(cuda), test_poses=poses, test_intrinsics=intr))
    assert out['num_samples'] == B and out['pred_imgs'].shape == (B, 2, 3, res, res) and torch.isfinite(out['pred_imgs']).all()
    code = seen[-1][0]
    assert code.shape == (B, 3, 6, 128, 128)
    diff_layout = model.code_diff_pr(code)
    assert diff_layout.shape == (B, 6, 128, 384)
    assert torch.equal(model.code_diff_pr_inv(diff_layout), code)
    # the same chain in fp32 on the denoiser's layout, mapped back
    up.fp32_reference_mode()
    sdg = up.state_dict_to(sd, cuda)
    dv = up.diffusion_vars(up.linear_betas())
    with torch.no_grad():
        x = model.code_diff_pr(noise.to(cuda)).contiguous()
        ref = up.ddim_sample(lambda x, t: uto.unet_forward(sdg, _spec(), x, t.to(x.device)), x, dv, num_timesteps=8,
                             clip_range=tuple(c['test_cfg']['clip_range']))
        ref = model.code_diff_pr_inv(ref)
    err = _rel_l2(code, ref)
    print('tiled val_step unconditional code rel l2', err)
    assert err < 1e-3


def test_tiled_val_step_guide_optim(cuda):
    """guided DDIM with the gradient through the UNet's input-gradient pass, then val_optim (diffusion prior + render loss)"""
    model, sd, c = _model(cuda, dict(num_timesteps=3, n_inverse_steps=2, extra_scene_step=1, n_inverse_rays=2 ** 12))
    assert model.test_cfg['cond_mode'] == 'guide_optim'
    B, res = 1, 128                     # test_cfg img_size: the views are rendered at 128 x 128
    g = torch.Generator().manual_seed(4)
    poses = torch.from_numpy(spiral_poses(3))[None].to(cuda)
    f = 131.25 * res / 128
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(B, 3, 4).contiguous().to(cuda)
    code0 = (torch.randn(B, 3, 6, 128, 128, generator=g) * 0.5).to(cuda)
    with torch.no_grad():
        _, bits0 = model.get_density(model.decoder_ema, code0, cfg=dict(density_thresh=0.1))
        img0, _ = model.render(model.decoder_ema, code0, bits0, res, res, intr[:, :1].contiguous(), poses[:, :1].contiguous(), cfg=model.test_cfg)
    guided = _capture(model, 'val_guide')
    optimd = _capture(model, 'val_optim')
    data = dict(scene_id=[0], scene_name=['a'], cond_imgs=img0, cond_intrinsics=intr[:, :1].contiguous(), cond_poses=poses[:, :1].contiguous(),
                test_poses=poses[:, 1:].contiguous(), test_intrinsics=intr[:, 1:].contiguous(),
                noise=torch.randn(B, 3, 6, 128, 128, generator=g).to(cuda))
    out = model.val_step(data)
    assert out['num_samples'] == B and out['pred_imgs'].shape == (B, 2, 3, res, res)
    assert torch.isfinite(out['pred_imgs']).all() and float(out['pred_imgs'].std()) > 0
    for seen in (guided, optimd):
        code = seen[-1][0]
        assert code.shape == (B, 3, 6, 128, 128) and torch.isfinite(code).all()
        assert torch.equal(model.code_diff_pr_inv(model.code_diff_pr(code)), code)
    assert not torch.equal(guided[-1][0], optimd[-1][0])           # val_optim moved the guided code


def test_tiled_train_step_is_refused(cuda):
    model, sd, c = _model(cuda, {}, cache_size=4, extra_scene_step=1, n_decoder_rays=1024, n_inverse_rays=1024)
    model.train()
    B, res = 1, 32
    poses = torch.from_numpy(spiral_poses(2))[None].to(cuda)
    f = 131.25 * res / 128
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(B, 2, 4).contiguous().to(cuda)
    imgs = torch.rand(B, 2, res, res, 3, device=cuda)
    opt = dict(diffusion=torch.optim.Adam(model.diffusion.parameters(), lr=1e-4), decoder=torch.optim.Adam(model.decoder.parameters(), lr=1e-3))
    data = dict(scene_id=[0], scene_name=['s0'], cond_imgs=imgs, cond_poses=poses, cond_intrinsics=intr)
    with pytest.raises(NotImplementedError, match='GroupNorm\\(16\\)'):
        model.train_step(data, opt)
