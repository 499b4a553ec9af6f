"""SSIM kernel and LPIPS(VGG16) on the native convolutions against the CPU oracle (oracle/metrics_port.py), and the test_ssim /
test_lpips keys of val_step on a recons config.

Bars, fixed on the CPU before any GPU run (tests/test_eval_metrics_cpu.py):
  * SSIM: per image, no worse than the reference's own float32 error on the same inputs (float32 vs float64 oracle), floor 1e-5 absolute.
  * LPIPS: per image 1e-3 relative to the float64 oracle.  The fp16 storage probe (scaled input, conv weights and every post-ReLU map
    rounded to fp16, arithmetic in float64) moves LPIPS by at most 2.7e-4 relative on these inputs; the rest of the bar covers fp32
    accumulation and rounding-boundary flips of the stored maps."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import metrics_port as mp
from tests.common import GOLDEN, spiral_poses

pytestmark = pytest.mark.gpu

LPIPS_REL = 1e-3


@pytest.mark.parametrize('h,w', [(128, 128), (7, 7), (33, 65), (64, 96)])
@pytest.mark.parametrize('n', [1, 37, 4016])
def test_ssim_kernel_matches_float64_oracle(cuda, n, h, w):
    from ssdnerf_b200 import metrics as M
    if n == 4016 and (h, w) != (128, 128):
        pytest.skip('4016 images at the shipped size only')
    p, t = mp.synthetic_pairs(min(n, 64), h, w, seed=h * 1000 + w + n)
    idx = np.arange(n) % p.shape[0]                 # 4016 = the bench batch's 16 x 251 views, built from 64 distinct pairs
    p, t = p[idx], t[idx]
    pg, tg = torch.from_numpy(p).to(cuda), torch.from_numpy(t).to(cuda)
    got = M.ssim(pg, tg)
    again = M.ssim(pg, tg)
    assert torch.equal(got, again)
    k = min(n, 64)
    ref = mp.ssim_skimage(p[:k], t[:k], np.float64)
    bar = max(np.abs(mp.ssim_skimage(p[:k], t[:k], np.float32) - ref).max(), 1e-5)
    err = np.abs(got.cpu().numpy().astype(np.float64)[:k] - ref).max()
    assert err <= bar, (err, bar)
    if n > k:
        assert torch.equal(got[k:], got[idx[k:]])
    assert torch.equal(M.ssim(pg, pg), torch.ones(n, device=cuda))


def test_ssim_rejects_small_images(cuda):
    from ssdnerf_b200 import metrics as M
    from ssdnerf_b200._lib import SSDNeRFNativeError
    x = torch.rand(2, 6, 32, 3, device=cuda)
    with pytest.raises(SSDNeRFNativeError, match='7 x 7'):
        M.ssim(x, x)


def _lpips(tmp_path, seed=0, **kw):
    from ssdnerf_b200 import lpips as LP
    vgg, lin = mp.random_weights(seed)
    pv, pl = tmp_path / 'vgg16.pth', tmp_path / 'vgg.pth'
    torch.save(vgg, pv)
    torch.save(lin, pl)
    return LP.LPIPS(str(pv), str(pl), **kw), vgg, lin


def test_lpips_matches_float64_oracle_128(cuda, tmp_path):
    model, vgg, lin = _lpips(tmp_path)
    p, t = mp.synthetic_pairs(4, 128, 128, seed=1)
    got = model(torch.from_numpy(p).to(cuda), torch.from_numpy(t).to(cuda)).cpu().double()
    ref = mp.lpips_vgg(p, t, vgg, lin)
    rel = float(((got - ref).abs() / ref).max())
    assert rel < LPIPS_REL, (rel, got, ref)


def test_lpips_chunks_and_identity(cuda, tmp_path):
    """70 pairs at 32 x 32 with a 16-pair chunk (5 chunks, the last short) against the oracle and against one 70-pair chunk: a pair's
    result does not depend on its chunk; LPIPS(x, x) is exactly 0"""
    from ssdnerf_b200 import lpips as LP
    small, vgg, lin = _lpips(tmp_path, workspace_bytes=16 * LP.pair_bytes(32, 32))
    assert small.chunk(32, 32) == 16
    big = LP.LPIPS(small.vgg_path, small.lin_path)
    assert big.chunk(32, 32) >= 70
    p, t = mp.synthetic_pairs(70, 32, 32, seed=2)
    pg, tg = torch.from_numpy(p).to(cuda), torch.from_numpy(t).to(cuda)
    a = small(pg, tg)
    b = big(pg, tg)
    assert torch.equal(a, b)
    ref = mp.lpips_vgg(p, t, vgg, lin)
    rel = float(((a.cpu().double() - ref).abs() / ref).max())
    assert rel < LPIPS_REL, rel
    assert torch.equal(small(pg, pg), torch.zeros(70, device=cuda))
    assert torch.equal(small(pg, tg), a)


def test_lpips_rejects_unsupported_size(cuda, tmp_path):
    model, _, _ = _lpips(tmp_path)
    x = torch.rand(2, 96, 96, 3, device=cuda)
    with pytest.raises(NotImplementedError, match='96 x 96'):
        model(x, x)


def test_val_step_reports_ssim_and_lpips(cuda, tmp_path, monkeypatch):
    """a recons config (`ssdnerf_cars_recons1v`) evaluating stored codes against test_imgs: test_psnr as before, test_ssim equal to the
    oracle on the returned pred_imgs, test_lpips with a caller-supplied LPIPS; without weights only test_psnr and test_ssim"""
    import warnings
    import ssdnerf_b200 as S
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path / 'hub'))
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_recons1v.py']
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg']).to(cuda).eval()
    assert model.lpips == []
    B, V, res = 2, 3, 128
    g = torch.Generator().manual_seed(0)
    poses = torch.from_numpy(spiral_poses(V))[None].repeat(B, 1, 1, 1).to(cuda)
    intr = torch.tensor([131.25, 131.25, 64.0, 64.0]).expand(B, V, 4).contiguous().to(cuda)
    code = (torch.randn(B, 3, 6, 128, 128, generator=g) * 0.5).to(cuda)
    with torch.no_grad():
        _, bits = model.get_density(model.decoder_ema, code, cfg=dict(density_thresh=0.1))
        img, _ = model.render(model.decoder_ema, code, bits, res, res, intr, poses, cfg=model.test_cfg)
    p8, t8 = mp.synthetic_pairs(B * V, res, res, seed=5)
    test_imgs = (0.7 * img + 0.3 * torch.from_numpy(t8).to(cuda).view(B, V, res, res, 3)).clamp(0, 1).contiguous()
    stored = [dict(param=dict(code=code[i].cpu(), density_grid=torch.zeros(64 ** 3).half(), density_bitfield=bits[i].cpu())) for i in range(B)]
    data = dict(scene_id=[0, 1], scene_name=['a', 'b'], code=stored, test_poses=poses, test_intrinsics=intr, test_imgs=test_imgs)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        out = model.val_step(data)
        out2 = model.val_step(data)
    assert sum('LPIPS weights not found' in str(r.message) for r in rec) == 1
    lv = out['log_vars']
    assert sorted(lv) == ['test_psnr', 'test_ssim'] and out2['log_vars'] == lv
    pred = out['pred_imgs'].reshape(B * V, 3, res, res)
    target = test_imgs.permute(0, 1, 4, 2, 3).reshape(B * V, 3, res, res)
    mse = (pred - target).square().flatten(1).mean(dim=1)
    assert lv['test_psnr'] == float((-10 * torch.log10(mse + 1e-6)).mean())
    pred_cl = pred.permute(0, 2, 3, 1).cpu().numpy()
    tgt_cl = test_imgs.reshape(B * V, res, res, 3).cpu().numpy()
    ref_ssim = mp.ssim_skimage(pred_cl, tgt_cl, np.float64)
    assert abs(lv['test_ssim'] - ref_ssim.mean()) < 1e-5
    lp, vgg, lin = _lpips(tmp_path)
    model.lpips = lp
    lv2 = model.val_step(data)['log_vars']
    assert sorted(lv2) == ['test_lpips', 'test_psnr', 'test_ssim']
    assert lv2['test_psnr'] == lv['test_psnr'] and lv2['test_ssim'] == lv['test_ssim']
    ref_lp = mp.lpips_vgg(pred_cl, tgt_cl, vgg, lin)
    assert abs(lv2['test_lpips'] - float(ref_lp.mean())) < LPIPS_REL * float(ref_lp.mean())
