"""CPU side of the viz_dir PNG files: the PNG reader the GPU tests rely on (against files built with zlib), the shipped viridis table,
the file names of eval_and_viz and the colormap layout of TriPlaneDecoder.visualize."""
import math
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from tests import png_check


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def _filter_row(t, cur, prev):
    out = []
    for i, x in enumerate(cur):
        a = cur[i - 4] if i >= 4 else 0
        b = prev[i]
        c = prev[i - 4] if i >= 4 else 0
        pr = [0, a, b, (a + b) // 2, _paeth(a, b, c)][t]
        out.append((x - pr) % 256)
    return bytes([t] + out)


def _png(rgba, types, level=6):
    h, w, _ = rgba.shape
    raw, prev = b'', [0] * (4 * w)
    for y in range(h):
        cur = [int(v) for v in rgba[y].reshape(-1)]
        raw += _filter_row(types[y % len(types)], cur, prev)
        prev = cur

    def chunk(kind, body):
        return struct.pack('>I', len(body)) + kind + body + struct.pack('>I', zlib.crc32(kind + body))
    return (png_check.SIGNATURE + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 6, 0, 0, 0))
            + chunk(b'IDAT', zlib.compress(raw, level)) + chunk(b'IEND', b'')), raw


@pytest.mark.parametrize('shape', [(1, 1), (5, 7), (9, 33)])
def test_checker_reads_zlib_built_files_with_every_filter(shape):
    g = np.random.default_rng(sum(shape))
    rgba = g.integers(0, 256, shape + (4,), dtype=np.uint8)
    rgba[..., 3] = 255
    data, raw = _png(rgba, types=[0, 1, 2, 3, 4])
    pixels, stream, _ = png_check.decode(data)
    assert np.array_equal(pixels, rgba) and stream == raw


def test_checker_rejects_corruption():
    rgba = np.full((4, 4, 4), 200, np.uint8)
    data, _ = _png(rgba, types=[4])
    with pytest.raises(AssertionError, match='CRC'):
        png_check.decode(data[:20] + bytes([data[20] ^ 1]) + data[21:])
    bad = bytearray(data)
    bad[-20] ^= 0xFF                                          # inside the zlib stream: Adler-32 / inflate fails before the CRC
    with pytest.raises((AssertionError, zlib.error)):
        png_check.decode(bytes(bad))


def test_viridis_table_is_opencv_viridis():
    cv2 = pytest.importorskip('cv2')
    from ssdnerf_b200 import viz
    ref = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(1, 256), cv2.COLORMAP_VIRIDIS)[0, :, ::-1]
    assert np.array_equal(viz.viridis(), ref)


def test_view_file_names():
    from ssdnerf_b200 import viz
    names, bases = viz.view_file_names(['a', 'b'], 2)
    assert names == ['scene_a_000.png', 'scene_a_001.png', 'scene_b_000.png', 'scene_b_001.png'] and bases is None
    paths = [['/x/rgb/000.png', '/x/rgb/001.jpg'], ['y/7.png', 'y/8.png']]
    psnr, ssim = [25.04, 9.96, 30.0, 31.25], [0.915, 0.5, 0.994, 0.995]
    names, bases = viz.view_file_names(['a', 'b'], 2, paths, psnr, ssim, None)
    assert bases == ['scene_a_000', 'scene_a_001', 'scene_b_7', 'scene_b_8']
    assert names[0] == 'scene_a_000_psnr25.0_ssim0.92_lpipsnan.png'
    assert names[1] == 'scene_a_001_psnr10.0_ssim0.50_lpipsnan.png'
    names, _ = viz.view_file_names(['a', 'b'], 2, paths, psnr, ssim, [0.1234, 0.5, 0.0, math.nan])
    assert names[0] == 'scene_a_000_psnr25.0_ssim0.92_lpips0.123.png' and names[3].endswith('_lpipsnan.png')


def test_code_maps_layout():
    """triplane_decoder.py:186-194: rows flipped unless flip_z, then [3, C, h, w] -> [3 h, C w]"""
    from ssdnerf_b200 import viz
    code = torch.arange(2 * 3 * 4 * 5 * 6, dtype=torch.float32).reshape(2, 3, 4, 5, 6)
    m = viz.code_maps(code)
    c = code.numpy()[..., ::-1, :]
    assert m.shape == (2, 15, 24)
    for p in range(3):
        for k in range(4):
            assert np.array_equal(m[:, 5 * p:5 * p + 5, 6 * k:6 * k + 6].numpy(), c[:, p, k])
    assert np.array_equal(viz.code_maps(code, flip_z=True)[:, :5, :6].numpy(), code[:, 0, 0].numpy())


def test_interp_noise_forms():
    """inference.py:70-84: the two draws of torch.randn, linear and spherical forms"""
    from ssdnerf_b200 import viz
    torch.manual_seed(5)
    ab = torch.randn(2, 3, 2, 4, 4)
    torch.manual_seed(5)
    lin = viz.interp_noise((3, 2, 4, 4), 5, 'linear')
    assert torch.equal(lin[0], ab[0]) and torch.equal(lin[-1], ab[1])
    torch.manual_seed(5)
    sph = viz.interp_noise((3, 2, 4, 4), 5, 'spherical_linear')
    theta = torch.acos((ab[0].flatten() / ab[0].norm()).dot(ab[1].flatten() / ab[1].norm()))
    mid = (math.sin(0.5 * theta) * (ab[0] + ab[1])) / torch.sin(theta)
    assert torch.allclose(sph[2], mid, atol=1e-5)
    with pytest.raises(AttributeError):
        viz.interp_noise((3, 2, 4, 4), 5, 'cubic')


def test_size_queries_refuse_bad_sizes():
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    assert L.ssdnerf_png_workspace_bytes(0, 4, 4) == 0 and L.ssdnerf_png_output_bound(1, 0, 4) == 0
    assert L.ssdnerf_png_workspace_bytes(1, 4, 4096) == 0 and L.ssdnerf_png_workspace_bytes(1, 4, 4095) > 0
    # 128 x 256 RGBA: 15 rows of 1025 bytes per segment, 9 segments
    assert L.ssdnerf_png_output_bound(2, 128, 256) == 2 * (63 + 128 * 1025 + 5 * 9)


# ------------------------------------------------------------------------------------------------ replay of the reference's execution
# tests/golden/reference_viz_v1.npz: the reference's own eval_and_viz, TriPlaneDecoder.visualize and interp_diffusion_nerf_ddim
# (tests/golden/make_golden_viz.py), with plt.imsave recording what it was given
def _fixture():
    from tests.common import GOLDEN
    return np.load(os.path.join(GOLDEN, 'reference_viz_v1.npz'))


def _pred_imgs(image):
    """base_nerf.py:551-553 as ssdnerf_b200.nerf computes it: [n, 3, h, w] on the 8-bit grid"""
    n, v, h, w, _ = image.shape
    p = torch.from_numpy(image).permute(0, 1, 4, 2, 3).reshape(n * v, 3, h, w).clamp(min=0, max=1)
    return torch.round(p * 255) / 255


def _names_and_files(z, tag, tmp_path):
    from oracle import metrics_port
    from ssdnerf_b200 import viz
    n_imgs = z['poses'].shape[1]
    paths = None
    psnr = ssim = None
    if tag == 'eval':
        pred = _pred_imgs(z['eval_image'])
        target = torch.from_numpy(z['test_imgs']).permute(0, 1, 4, 2, 3).reshape(pred.shape)
        psnr = (-10 * torch.log10((pred - target).square().flatten(1).mean(dim=1) + 1e-6)).tolist()
        ssim = metrics_port.ssim_skimage(pred.permute(0, 2, 3, 1), target.permute(0, 2, 3, 1)).tolist()
        paths = z['paths'].tolist()
    names, bases = viz.view_file_names(['a', 'b'], n_imgs, paths, psnr, ssim, None)
    d = tmp_path / tag
    d.mkdir()
    for f in z['stale']:
        (d / str(f)).write_bytes(b'')
    viz.write_view_files(str(d), names, bases, [b'png'] * len(names))
    for f in ('scene_a.png', 'scene_b.png', 'scene_000_mean.png'):           # TriPlaneDecoder.visualize, then init_code
        (d / f).write_bytes(b'png')
    return names, sorted(os.listdir(d))


@pytest.mark.parametrize('tag', ['eval', 'noimg'])
def test_view_files_replay_reference(tag, tmp_path):
    """names from the per-image metrics, and the directory after the reference's per-view delete-then-write (including a stem '1'
    that deletes the file written for stem '10')"""
    z = _fixture()
    names, files = _names_and_files(z, tag, tmp_path)
    assert names + ['scene_a.png', 'scene_b.png', 'scene_000_mean.png'] == z[f'{tag}_names'].tolist()
    assert files == z[f'{tag}_files'].tolist()


def test_view_pixels_replay_reference():
    """the u8 arrays the reference handed to plt.imsave = the formulas the device encoder implements (tests/test_viz_gpu.py replays the
    same arrays through the encoder)"""
    z = _fixture()
    for tag, real in (('eval', z['test_imgs']), ('noimg', None)):
        n, v, h, w, _ = z[f'{tag}_image'].shape
        p = torch.round(_pred_imgs(z[f'{tag}_image']).permute(0, 2, 3, 1) * 255).to(torch.uint8)
        if real is not None:
            p = torch.cat([(torch.from_numpy(real).reshape(n * v, h, w, 3) * 255).to(torch.uint8), p], dim=2)
        assert np.array_equal(p.numpy(), z[f'{tag}_u8'])


def test_maps_replay_reference():
    """the 2-D maps and ranges the reference's visualize handed to plt.imsave: code_maps of the codes and of init_code, clip_range"""
    from ssdnerf_b200 import viz
    z = _fixture()
    for tag in ('eval', 'noimg'):
        assert np.array_equal(viz.code_maps(torch.from_numpy(z['code'])).numpy(), z[f'{tag}_maps'])
        assert np.array_equal(viz.code_maps(torch.from_numpy(z['init_code'])[None])[0].numpy(), z[f'{tag}_mean_map'])
        assert (z[f'{tag}_vrange'] == [-1.5, 1.5]).all()


@pytest.mark.parametrize('typ', ['linear', 'spherical_linear'])
def test_interp_replay_reference(typ):
    """interp_diffusion_nerf_ddim's val_step data dicts: the noise bit for bit after the same seed, names, ids and batch split"""
    import types
    from ssdnerf_b200 import viz
    z = _fixture()
    rec = []
    model = types.SimpleNamespace(code_size=tuple(z['code'].shape[1:]), parameters=lambda: iter([torch.zeros(1)]),
                                  val_step=lambda data, **kw: rec.append((data, kw)))
    torch.manual_seed(17)
    viz.interp_diffusion_nerf_ddim(model, torch.from_numpy(z['poses'][0]), torch.from_numpy(z['intr'][0]), viz_dir='/v',
                                   num_samples=5, batchsize=2, type=typ)
    assert np.array_equal(torch.cat([r[0]['noise'] for r in rec]).numpy(), z[f'interp_{typ}_noise'])
    assert sum([r[0]['scene_name'] for r in rec], []) == z[f'interp_{typ}_names'].tolist()
    assert sum([list(r[0]['scene_id']) for r in rec], []) == z[f'interp_{typ}_ids'].tolist()
    assert [len(r[0]['scene_name']) for r in rec] == z[f'interp_{typ}_batch'].tolist()
    assert all(r[1] == dict(viz_dir='/v', show_pbar=True) for r in rec)
    assert all(r[0]['test_poses'].shape == (len(r[0]['scene_name']),) + z['poses'].shape[1:] for r in rec)
