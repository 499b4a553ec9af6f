"""Evaluation metrics without a GPU: the SSIM / LPIPS oracle's fixed points and the float32 error of the reference's SSIM path, the LPIPS
weight loader on both on-disk key formats, default weight paths that never reach for the network, and the GEMM argument struct that
gained the ReLU flag."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import metrics_port as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_fixed_points():
    p, t = mp.synthetic_pairs(3, 32, 32, seed=0)
    np.testing.assert_allclose(mp.ssim_skimage(p, p), 1.0, rtol=0, atol=1e-12)
    assert (mp.ssim_skimage(p, t) < 0.99).all()
    vgg, lin = mp.random_weights(0)
    assert torch.equal(mp.lpips_vgg(p, p, vgg, lin), torch.zeros(3, dtype=torch.float64))
    assert (mp.lpips_vgg(p, t, vgg, lin) > 0).all()


@pytest.mark.parametrize('h,w', [(128, 128), (7, 7), (33, 65), (64, 96)])
def test_reference_float32_ssim_error(h, w):
    """the reference computes SSIM in float32 (its inputs are float32); its gap to the float64 value is what the GPU kernel's error is held
    to (with a 1e-5 floor).  On these inputs it stays below 1e-5 everywhere, so the floor is the effective GPU bar."""
    p, t = mp.synthetic_pairs(37, h, w, seed=h * 1000 + w)
    gap = np.abs(mp.ssim_skimage(p, t, np.float32) - mp.ssim_skimage(p, t, np.float64)).max()
    assert 0 < gap < 1e-5, gap


def test_lpips_fp16_storage_probe():
    """precision probe behind the GPU LPIPS bar: rounding what the native path stores in fp16 (scaled input, conv weights, every post-ReLU
    map) moves LPIPS by at most 2.7e-4 relative on these inputs (1.1e-6 absolute); the GPU test allows 1e-3 relative"""
    vgg, lin = mp.random_weights(0)
    for n, h, w, seed in [(4, 128, 128, 1), (70, 32, 32, 2)]:
        p, t = mp.synthetic_pairs(n, h, w, seed=seed)
        ref = mp.lpips_vgg(p, t, vgg, lin)
        probe = mp.lpips_vgg(p, t, vgg, lin, fp16_storage=True)
        assert float(((probe - ref).abs() / ref).max()) < 4e-4


def _write_weights(tmp_path, vgg, lin):
    pv, pl = tmp_path / 'vgg16.pth', tmp_path / 'vgg.pth'
    torch.save(vgg, pv)
    torch.save(lin, pl)
    return str(pv), str(pl)


def test_lpips_weight_loader(tmp_path):
    from ssdnerf_b200 import lpips as LP
    vgg, lin = mp.random_weights(0)
    vgg_full = dict(vgg, **{'classifier.0.weight': torch.zeros(2, 2)})          # torchvision's file also holds the classifier
    pv, pl = _write_weights(tmp_path, vgg_full, lin)
    m = LP.LPIPS(pv, pl)
    assert len(m._host['w']) == 13 and m._host['w'][0].shape == (9, 64, LP.IN_CHANNELS) and m._host['w'][12].shape == (9, 512, 512)
    assert torch.equal(m._host['lin'][4], lin['lin4.model.1.weight'].reshape(-1))
    bad = dict(vgg)
    del bad['features.17.bias']
    pv2, _ = _write_weights(tmp_path, bad, lin)
    with pytest.raises(ValueError, match=r"vgg16\.pth.*features\.17\.bias"):
        LP.LPIPS(pv2, pl)
    bad_lin = dict(lin, **{'lin2.model.1.weight': torch.zeros(1, 128, 1, 1)})
    _, pl2 = _write_weights(tmp_path, vgg, bad_lin)
    with pytest.raises(ValueError, match=r"vgg\.pth.*lin2\.model\.1\.weight.*\(1, 128, 1, 1\)"):
        LP.LPIPS(pv, pl2)
    with pytest.raises(FileNotFoundError, match='nowhere.pth'):
        LP.LPIPS(str(tmp_path / 'nowhere.pth'), pl)


def test_lpips_sizes():
    from ssdnerf_b200 import lpips as LP
    assert LP.supported(128, 128) and LP.supported(64, 64) and LP.supported(32, 32) and LP.supported(256, 256)
    assert not LP.supported(96, 96) and not LP.supported(40, 40) and not LP.supported(128, 384)


def test_default_weight_paths_never_download(tmp_path, monkeypatch):
    """no weights on disk and no lpips package: no LPIPS, no exception, `test_lpips` left out with one warning, and nothing asks torch.hub
    for a URL"""
    import importlib.util
    import warnings
    from ssdnerf_b200 import lpips as LP
    from ssdnerf_b200.nerf import BaseNeRF

    def no_url(*a, **k):
        raise AssertionError('LPIPS weights must never be downloaded')
    monkeypatch.setattr(torch.hub, 'load_state_dict_from_url', no_url)
    monkeypatch.setattr(torch.hub, 'download_url_to_file', no_url)
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path))
    real_find_spec = importlib.util.find_spec
    monkeypatch.setattr(importlib.util, 'find_spec', lambda name, *a: None if name == 'lpips' else real_find_spec(name, *a))
    vgg, lin = LP.default_paths()
    assert vgg == os.path.join(str(tmp_path), 'checkpoints', 'vgg16-397923af.pth') and lin is None
    assert not LP.default_files_exist()
    with pytest.raises(FileNotFoundError):
        LP.LPIPS()
    model = BaseNeRF()
    assert model.lpips == [] and not any('lpips' in k for k in model.state_dict())
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        assert model._lpips_metric() is None
        assert model._lpips_metric() is None
    assert len(rec) == 1 and 'LPIPS weights not found' in str(rec[0].message)
    assert model.lpips == []
    assert BaseNeRF(use_lpips_metric=False)._lpips_metric() is None


def test_default_weight_paths_with_files(tmp_path, monkeypatch):
    """both default files present: the model builds LPIPS from them on first use and keeps it in its list"""
    import importlib.machinery
    import importlib.util
    from ssdnerf_b200 import lpips as LP
    from ssdnerf_b200.nerf import BaseNeRF
    vgg, lin = mp.random_weights(0)
    (tmp_path / 'checkpoints').mkdir()
    torch.save(vgg, tmp_path / 'checkpoints' / 'vgg16-397923af.pth')
    pkg = tmp_path / 'site' / 'lpips'
    (pkg / 'weights' / 'v0.1').mkdir(parents=True)
    torch.save(lin, pkg / 'weights' / 'v0.1' / 'vgg.pth')
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path))
    real_find_spec = importlib.util.find_spec
    spec = importlib.machinery.ModuleSpec('lpips', None, origin=str(pkg / '__init__.py'))
    monkeypatch.setattr(importlib.util, 'find_spec', lambda name, *a: spec if name == 'lpips' else real_find_spec(name, *a))
    assert LP.default_files_exist()
    model = BaseNeRF()
    m = model._lpips_metric()
    assert isinstance(m, LP.LPIPS) and model.lpips == [m] and model._lpips_metric() is m
    own = LP.LPIPS(str(tmp_path / 'checkpoints' / 'vgg16-397923af.pth'), str(pkg / 'weights' / 'v0.1' / 'vgg.pth'))
    model.lpips = own
    assert model._lpips_metric() is own


def test_gemm_args_mirror_with_relu_flag(tmp_path):
    """`ssdnerf_gemm_args.relu` is the struct's last field and the ctypes mirror matches the header's layout"""
    from ssdnerf_b200 import unet_ops as U
    assert U.GemmArgs._fields_[-1][0] == 'relu'
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ssdnerf_b200.h"', 'int main(void) {',
             '    printf("%zu %zu\\n", sizeof(ssdnerf_gemm_args), offsetof(ssdnerf_gemm_args, relu));', '    return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines) + '\n')
    subprocess.run(['cc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(U.GemmArgs), U.GemmArgs.relu.offset]


def test_metric_entry_points_exported_and_validated():
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    u32 = ctypes.c_uint32
    fake = ctypes.c_void_p(1 << 20)                  # never dereferenced: validation fails first
    assert L.ssdnerf_ssim_f32(fake, fake, u32(1), u32(6), u32(32), fake, None) == -2
    assert b'7 x 7' in L.ssdnerf_last_error()
    assert L.ssdnerf_ssim_f32(fake, fake, u32(1), u32(32), u32(5), fake, None) == -2
    assert L.ssdnerf_lpips_tap_f16(fake, u32(1), u32(8), u32(8), u32(96), fake, fake, None, fake, None) == -2
    assert L.ssdnerf_lpips_tap_partials(u32(3), u32(128), u32(128), u32(64), ctypes.c_int(1)) == 3 * 4096 // 128
    assert L.ssdnerf_lpips_tap_partials(u32(3), u32(8), u32(8), u32(512), ctypes.c_int(0)) == 3 * 64 // 32
    assert L.ssdnerf_version() == 102
