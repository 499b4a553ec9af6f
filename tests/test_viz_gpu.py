"""PNG files on the device (csrc/png.cu): every file passes the stdlib reader (tests/png_check.py) and decodes to exactly the pixels of the
reference's formulas composed in torch; edge sizes, the stored fallback, back-references across segments, determinism, the size bar
against zlib level 6 on the same filtered stream, and the viz_dir outputs of val_step and interp_diffusion_nerf_ddim."""
import io
import json
import os
import zlib

import numpy as np
import pytest
import torch

from tests import png_check
from tests.common import GOLDEN

pytestmark = pytest.mark.gpu


def _expect_views(pred, real=None):
    """base_nerf.py:551-553, 580-584 composed in torch: uint8 [n, h, w', 4]"""
    p = torch.round(torch.round(pred.clamp(0, 1) * 255) / 255 * 255).to(torch.uint8)
    if real is not None:
        p = torch.cat([(real * 255).to(torch.uint8), p], dim=2)
    return torch.cat([p, torch.full_like(p[..., :1], 255)], dim=-1).cpu().numpy()


def _expect_maps(maps, vmin, vmax):
    """matplotlib's Normalize + Colormap index rule in float32, through the shipped viridis table"""
    from ssdnerf_b200 import viz
    x = maps.cpu().float()
    xa = (x - np.float32(vmin)) / np.float32(np.float32(vmax - vmin)) * 256
    xa = torch.where(xa == 256, torch.full_like(xa, 255), xa)
    idx = torch.where(xa < 0, torch.zeros_like(xa), torch.where(xa >= 256, torch.full_like(xa, 255), xa))
    idx = torch.nan_to_num(idx, nan=0.0).to(torch.int64)          # NaN -> bad colour below
    rgb = torch.from_numpy(viz.viridis())[idx]
    out = torch.cat([rgb, torch.full_like(rgb[..., :1], 255)], dim=-1)
    out[torch.isnan(x)] = 0
    return out.numpy()


def _check(files, expect):
    assert len(files) == len(expect)
    for data, exp in zip(files, expect):
        px, _, _ = png_check.decode(data)
        assert np.array_equal(px, exp)
        for lib in ('PIL', 'cv2'):
            try:
                mod = __import__(lib)
            except ImportError:
                continue
            if lib == 'PIL':
                from PIL import Image
                other = np.asarray(Image.open(io.BytesIO(data)).convert('RGBA'))
            else:
                bgra = mod.imdecode(np.frombuffer(data, np.uint8), mod.IMREAD_UNCHANGED)
                other = bgra[..., [2, 1, 0, 3]] if bgra.ndim == 3 else None
            if other is not None:
                assert np.array_equal(other, exp), lib


def _render_like(n, h, w, seed, cuda):
    """smooth shaded blobs on a white background with a little noise: the statistics of rendered views"""
    g = torch.Generator().manual_seed(seed)
    y, x = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing='ij')
    imgs = torch.ones(n, h, w, 3)
    for i in range(n):
        c = torch.rand(3, generator=g) * 0.6 - 0.3
        r = 0.4 + 0.4 * torch.rand(1, generator=g)
        d = ((x - c[0]) ** 2 + (y - c[1]) ** 2).sqrt()
        inside = d < r
        shade = (0.5 + 0.5 * torch.cos(6 * x + 4 * y + 10 * c[2]))[..., None] * torch.rand(3, generator=g)
        imgs[i][inside] = shade[inside] + 0.01 * torch.randn(int(inside.sum()), 3, generator=g)
    return imgs.to(cuda)


def test_views_match_reference_formula(cuda):
    from ssdnerf_b200 import viz
    pred = _render_like(5, 64, 48, 0, cuda) * 1.2 - 0.1          # out of [0, 1] too: clamped
    real = _render_like(5, 64, 48, 1, cuda)
    _check(viz.encode_png(pred=pred, real=real), _expect_views(pred, real))
    _check(viz.encode_png(pred=pred), _expect_views(pred))


@pytest.mark.parametrize('h,w', [(1, 1), (1, 2), (3, 5), (7, 33), (2, 4095), (600, 3)])
def test_edge_sizes(cuda, h, w):
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(h * 7919 + w)
    pred = torch.rand(3, h, w, 3, generator=g).to(cuda)
    pred[1] = 0.5                                                 # solid: runs of 258
    _check(viz.encode_png(pred=pred), _expect_views(pred))


def test_noise_takes_stored_blocks(cuda):
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(2)
    pred = torch.randint(0, 256, (2, 128, 256, 3), generator=g).float().div(255).to(cuda)
    files = viz.encode_png(pred=pred)
    _check(files, _expect_views(pred))
    for data in files:
        _, raw, payload = png_check.decode(data)
        assert payload <= len(raw) + 5 * -(-len(raw) // 65535), (payload, len(raw))


def test_colormap_mode_and_multi_segment_triplane(cuda):
    """a 384 x 768 map (3 planes of 128 rows, 6 channels of 128): 5 rows per segment, back-references across segment boundaries"""
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(3)
    code = torch.tanh(torch.randn(2, 3, 6, 16, 16, generator=g)).to(cuda)
    code = torch.nn.functional.interpolate(code.reshape(2, 18, 16, 16), size=(128, 128), mode='bilinear').reshape(2, 3, 6, 128, 128)
    maps = viz.code_maps(code)
    maps[0, :3, :5] = torch.tensor([-1.0, 1.0, -2.0, 2.0, float('nan')], device=cuda)   # both range ends, under, over, bad
    assert maps.shape == (2, 384, 768)
    _check(viz.encode_png(maps=maps.contiguous(), vmin=-1, vmax=1), _expect_maps(maps, -1, 1))
    _check(viz.encode_png(maps=maps.contiguous(), vmin=-0.7, vmax=0.9), _expect_maps(maps, -0.7, 0.9))


@pytest.mark.parametrize('w,period', [(4095, 2), (1024, 8)])
def test_repeats_at_the_window_limit(cuda, w, period):
    """noise rows repeating every `period` rows: 32762 bytes back (w = 4095, inside the 32768-byte window, 6 bytes short of its end)
    and 32776 bytes back (w = 1024, just outside: must not be referenced)"""
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(4)
    base = torch.rand(period, w, 3, generator=g)
    pred = base.repeat(16 // period, 1, 1)[None].to(cuda)
    files = viz.encode_png(pred=pred)
    _check(files, _expect_views(pred))
    if w == 4095:
        _, raw, payload = png_check.decode(files[0])
        assert payload < 0.6 * len(raw)


def test_repeat_exactly_32768_back(cuda):
    """the longest legal distance: w = 2047 (rows of 8189 bytes), row k = row k - 4 shifted right by 3 pixels, so the filtered bytes
    repeat 4 * 8189 + 12 = 32768 bytes back.  Pixel bytes are small signed values (0..40, 216..255) with high entropy, so the None filter
    wins every row and the 3-byte strings are nearly unique.  Against the same rows drawn independently, the file must shrink by half:
    without the match at exactly 32768 it would not shrink at all."""
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(6)
    vals = torch.cat([torch.arange(0, 41), torch.arange(216, 256)])
    draw = lambda *s: vals[torch.randint(0, len(vals), s, generator=g)]
    h, w = 16, 2047
    rep = draw(h, w, 3)
    for k in range(4, h):
        rep[k, 3:] = rep[k - 4, :-3]
    ind = draw(h, w, 3)
    pred = torch.stack([rep, ind]).float().div(255).to(cuda)
    files = viz.encode_png(pred=pred)
    _check(files, _expect_views(pred))
    (_, raw, p_rep), (_, _, p_ind) = png_check.decode(files[0]), png_check.decode(files[1])
    assert raw[0] == 0 and all(raw[r * (4 * w + 1)] == 0 for r in range(h))         # None filter on every row
    print(f'repeat {p_rep} B, independent {p_ind} B')
    assert p_rep < 0.5 * p_ind


def test_deterministic_across_runs_and_batches(cuda):
    from ssdnerf_b200 import viz
    a = _render_like(6, 96, 80, 5, cuda)
    b = _render_like(3, 96, 80, 6, cuda)
    f1 = viz.encode_png(pred=a)
    f2 = viz.encode_png(pred=a)
    f3 = viz.encode_png(pred=torch.cat([b, a[2:4]]))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        f4 = viz.encode_png(pred=a[3:])
    assert f1 == f2 and f3[3:] == f1[2:4] and f4 == f1[3:]


def test_size_within_ten_percent_of_zlib6(cuda):
    from ssdnerf_b200 import viz
    pred = _render_like(24, 128, 128, 7, cuda)
    real = _render_like(24, 128, 128, 8, cuda)
    native = ref = 0
    for data in viz.encode_png(pred=pred, real=real):
        _, raw, payload = png_check.decode(data)
        native += payload
        ref += len(zlib.compress(raw, 6)) - 6
    print(f'native {native} B, zlib-6 {ref} B, ratio {native / ref:.4f}')
    assert native <= 1.10 * ref


def test_bad_arguments_raise(cuda):
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import viz
    L = N.lib()
    x = torch.rand(1, 4, 4, 3, device=cuda)
    ws = torch.empty(L.ssdnerf_png_workspace_bytes(1, 4, 4), dtype=torch.uint8, device=cuda)
    out = torch.empty(L.ssdnerf_png_output_bound(1, 4, 4), dtype=torch.uint8, device=cuda)
    off = torch.empty(2, dtype=torch.int64, device=cuda)
    args = lambda n, h, w, wsb, ob: (N.ptr(x), None, n, h, w, N.ptr(ws), wsb, N.ptr(out), ob, N.ptr(off), N.stream_ptr())
    for bad, msg in [((0, 4, 4, ws.numel(), out.numel()), 'n, h, w'), ((1, 4, 4096, ws.numel(), out.numel()), 'row'),
                     ((1, 4, 4, ws.numel() - 1, out.numel()), 'workspace'), ((1, 4, 4, ws.numel(), out.numel() - 1), 'out')]:
        with pytest.raises(N.SSDNeRFNativeError, match=msg):
            N.check(L.ssdnerf_png_encode_views(*args(*bad)))
    with pytest.raises(ValueError):
        viz.encode_png(pred=torch.rand(1, 4, 4097, 3, device=cuda))
    with pytest.raises(ValueError):
        viz.encode_png(maps=torch.rand(1, 4, 4, device=cuda), vmin=1, vmax=0)


def test_encoder_replays_reference_arrays(cuda):
    """tests/golden/reference_viz_v1.npz: the u8 arrays the reference's eval_and_viz handed to plt.imsave, from the renders it made;
    the device encoder, given the same renders and test images, decodes to exactly those pixels"""
    from ssdnerf_b200 import viz
    z = np.load(os.path.join(GOLDEN, 'reference_viz_v1.npz'))
    for tag, real in (('eval', z['test_imgs']), ('noimg', None)):
        n, v, h, w, _ = z[f'{tag}_image'].shape
        pred = torch.from_numpy(z[f'{tag}_image']).reshape(n * v, h, w, 3).to(cuda)
        real_t = None if real is None else torch.from_numpy(real).reshape(n * v, h, w, 3).to(cuda)
        u8 = z[f'{tag}_u8']
        _check(viz.encode_png(pred=pred, real=real_t), np.concatenate([u8, np.full(u8.shape[:-1] + (1,), 255, np.uint8)], -1))


# ------------------------------------------------------------------------------------------------ model paths
def _cars_model(cuda, **test_over):
    import ssdnerf_b200 as S
    from oracle import unet_port as up
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=dict(c['test_cfg'], **test_over))
    sd = up.random_state_dict(up.unet_spec(), seed=7, std=0.02)
    for diff in (model.diffusion, model.diffusion_ema):
        diff.denoising.load_state_dict(sd, strict=True)
    return model.to(cuda).eval(), c


def _poses(n, cuda):
    from tests.test_ddpm_gpu import spiral_poses
    return torch.from_numpy(spiral_poses(n)).to(cuda)


def test_val_step_writes_reference_files(cuda, tmp_path):
    model, c = _cars_model(cuda, num_timesteps=2, n_inverse_steps=0, img_size=(64, 64))
    B, V, res = 2, 3, 64
    poses = _poses(V, cuda)[None].expand(B, -1, -1, -1).contiguous()
    intr = torch.tensor([65.625, 65.625, 32.0, 32.0], device=cuda).expand(B, V, 4).contiguous()
    noise = torch.randn(B, 3, 6, 128, 128, generator=torch.Generator().manual_seed(3)).to(cuda)
    # val_uncond with test_poses: scene_<name>_{:03d}.png per view, then the triplane maps
    d_u = tmp_path / 'uncond'
    out = model.val_step(dict(scene_id=[0, 1], scene_name=['a', 'b'], noise=noise, test_poses=poses, test_intrinsics=intr), viz_dir=str(d_u))
    names = sorted(os.listdir(d_u))
    assert names == sorted([f'scene_{s}_{v:03d}.png' for s in 'ab' for v in range(V)] + ['scene_a.png', 'scene_b.png']
                           + (['scene_000_mean.png'] if model.init_code is not None else []))
    pred = out['pred_imgs'].permute(0, 1, 3, 4, 2).reshape(B * V, res, res, 3)       # already on the 8-bit grid
    for k, (s, v) in enumerate([(s, v) for s in 'ab' for v in range(V)]):
        px, _, _ = png_check.decode((d_u / f'scene_{s}_{v:03d}.png').read_bytes())
        assert np.array_equal(px, _expect_views(pred[k:k + 1])[0])
    # evaluation with test images (val_uncond plus test_imgs: the same eval_and_viz path a val_cond run takes): names from the
    # per-image metrics, stale files of the same view removed first
    d_c = tmp_path / 'cond'
    d_c.mkdir()
    (d_c / 'scene_a_v0_psnr1.0_ssim0.00_lpipsnan.png').write_bytes(b'stale')
    test_imgs = _render_like(B * V, res, res, 9, cuda).reshape(B, V, res, res, 3)
    paths = [[f'/data/{s}/v{v}.png' for v in range(V)] for s in 'ab']
    data = dict(scene_id=[0, 1], scene_name=['a', 'b'], noise=noise, test_poses=poses, test_intrinsics=intr, test_imgs=test_imgs,
                test_img_paths=paths)
    model.lpips = None
    out = model.val_step(data, viz_dir=str(d_c))
    pred = out['pred_imgs'].permute(0, 1, 3, 4, 2).reshape(B * V, res, res, 3)
    real = test_imgs.reshape(B * V, res, res, 3)
    mse = (pred - real).square().flatten(1).mean(1)
    psnr = (-10 * torch.log10(mse + 1e-6)).tolist()
    from ssdnerf_b200 import metrics as M
    ssim = M.ssim(pred.contiguous(), real.contiguous()).tolist()
    files = sorted(f for f in os.listdir(d_c) if f.startswith('scene_a_v') or f.startswith('scene_b_v'))
    expect = sorted(f'scene_{s}_v{v}_psnr{psnr[k]:02.1f}_ssim{ssim[k]:.2f}_lpipsnan.png'
                    for k, (s, v) in enumerate([(s, v) for s in 'ab' for v in range(V)]))
    assert files == expect
    exp_px = _expect_views(pred, real)
    for k, name in enumerate(f'scene_{s}_v{v}' for s in 'ab' for v in range(V)):
        (f,) = [x for x in files if x.startswith(name + '_')]
        px, _, _ = png_check.decode((d_c / f).read_bytes())
        assert np.array_equal(px, exp_px[k])
    assert (d_c / 'scene_a.png').is_file() and (d_c / 'scene_b.png').is_file()
    # skip_eval (base_nerf.py:542): test images are ignored, the prediction alone is written under the index names
    model.test_cfg['skip_eval'] = True
    d_s = tmp_path / 'skip'
    out = model.val_step(data, viz_dir=str(d_s))
    pred = out['pred_imgs'].permute(0, 1, 3, 4, 2).reshape(B * V, res, res, 3)
    for k, (s, v) in enumerate([(s, v) for s in 'ab' for v in range(V)]):
        px, _, _ = png_check.decode((d_s / f'scene_{s}_{v:03d}.png').read_bytes())
        assert np.array_equal(px, _expect_views(pred[k:k + 1])[0])


def test_val_step_without_test_poses_writes_maps(cuda, tmp_path):
    from ssdnerf_b200 import viz
    model, c = _cars_model(cuda, num_timesteps=2, n_inverse_steps=0, save_dir=str(tmp_path / 'save'))
    noise = torch.randn(1, 3, 6, 128, 128, generator=torch.Generator().manual_seed(5)).to(cuda)
    model.val_step(dict(scene_id=[0], scene_name=['z'], noise=noise), viz_dir=str(tmp_path / 'viz'))
    assert sorted(os.listdir(tmp_path / 'viz')) == ['scene_z.png']
    code = torch.load(str(tmp_path / 'save' / 'z.pth'))['param']['code'].to(cuda)[None].float()
    clip = c['test_cfg'].get('clip_range', [-1, 1])
    px, _, _ = png_check.decode((tmp_path / 'viz' / 'scene_z.png').read_bytes())
    assert np.array_equal(px, _expect_maps(viz.code_maps(code), clip[0], clip[1])[0])


def test_interp_diffusion_nerf_ddim_writes_views_and_maps(cuda, tmp_path):
    import ssdnerf_b200 as S
    model, c = _cars_model(cuda, num_timesteps=2, n_inverse_steps=0, img_size=(32, 32))
    V = 2
    poses = _poses(V, cuda).cpu()
    intr = torch.tensor([32.8, 32.8, 16.0, 16.0]).expand(V, 4).contiguous()
    torch.manual_seed(1)
    S.interp_diffusion_nerf_ddim(model, poses, intr, viz_dir=str(tmp_path), num_samples=3, batchsize=2, type='spherical_linear')
    names = sorted(os.listdir(tmp_path))
    expect = [f'scene_interp_{i:02d}_{v:03d}.png' for i in range(3) for v in range(V)] + [f'scene_interp_{i:02d}.png' for i in range(3)]
    expect += ['scene_000_mean.png'] if model.init_code is not None else []
    assert names == sorted(expect)
    for n in names:
        png_check.decode((tmp_path / n).read_bytes())


def test_guide_optim_writes_viz_dir_guide(cuda, tmp_path):
    """diffusion_nerf.py:418-425: in guide_optim the guided sample is evaluated into viz_dir_guide before the optimisation"""
    import ssdnerf_b200 as S
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_chairs_recons1v.py']
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'],
                          test_cfg=dict(c['test_cfg'], num_timesteps=2, n_inverse_steps=1, extra_scene_step=1, n_inverse_rays=2 ** 12,
                                        img_size=(64, 64)))
    g = torch.Generator().manual_seed(0)
    for p in model.diffusion_ema.denoising.parameters():
        if p.dim() > 1:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.02)
    model = model.to(cuda).eval()
    assert model.test_cfg['cond_mode'] == 'guide_optim'
    poses = _poses(3, cuda)[None]
    intr = torch.tensor([65.625, 65.625, 32.0, 32.0], device=cuda).expand(1, 3, 4).contiguous()
    cond = _render_like(1, 64, 64, 3, cuda)[None]
    test_imgs = _render_like(2, 64, 64, 4, cuda)[None]
    data = dict(scene_id=[0], scene_name=['c'], cond_imgs=cond, cond_intrinsics=intr[:, :1].contiguous(), cond_poses=poses[:, :1].contiguous(),
                test_poses=poses[:, 1:].contiguous(), test_intrinsics=intr[:, 1:].contiguous(), test_imgs=test_imgs,
                test_img_paths=[['r/0.png', 'r/1.png']], noise=torch.randn(1, 3, 6, 128, 128, generator=g).to(cuda))
    model.lpips = None
    model.val_step(data, viz_dir=str(tmp_path / 'final'), viz_dir_guide=str(tmp_path / 'guide'))
    for d in ('guide', 'final'):
        names = sorted(os.listdir(tmp_path / d))
        views = [n for n in names if n.startswith('scene_c_0_') or n.startswith('scene_c_1_')]
        assert len(views) == 2 and all('_lpipsnan.png' in n for n in views) and 'scene_c.png' in names, names
        for n in names:
            png_check.decode((tmp_path / d / n).read_bytes())
