"""Orbit videos on the device: the JPEG encoder (csrc/jpeg.cu) writes the fixture's cv2.imencode bytes for the whole corpus in mixed
batches, its fp32 prologue is numpy's round(x * 255), and `python -m ssdnerf_b200.orbit` on a small random-weight model writes one AVI
per scene whose payloads are encode_jpeg of model.render for the orbit's poses, draws the GUI's seed noise, round-trips --save-scene /
--scene and writes the meshes save_mesh writes."""
import json
import os
import struct

import numpy as np
import pytest
import torch

from oracle import jpeg_port as J
from tests.common import GOLDEN
from tests.test_orbit_cpu import FIXTURE, corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def items():
    return corpus(dict(np.load(FIXTURE)))


def _encode(imgs, q, dev):
    from ssdnerf_b200 import video
    return video.encode_jpeg(torch.from_numpy(np.stack(imgs)).to(dev), q)


def test_fixture_bytes_one_by_one(items, cuda):
    bad = [name for name, img, q, data in items if _encode([img], q, cuda)[0] != data]
    assert not bad, f'{len(bad)} of {len(items)} files differ, e.g. {bad[:5]}'


def test_fixture_bytes_in_batches(items, cuda):
    """every (size, quality) group of the corpus in one call, and each image again inside a batch of shuffled copies of its group"""
    groups = {}
    for name, img, q, data in items:
        groups.setdefault((img.shape, q), []).append((img, data))
    rng = np.random.default_rng(0)
    for (shape, q), members in groups.items():
        files = _encode([m[0] for m in members], q, cuda)
        assert files == [m[1] for m in members], (shape, q)
        order = rng.permutation(np.tile(np.arange(len(members)), 3))
        files = _encode([members[i][0] for i in order], q, cuda)
        assert files == [members[i][1] for i in order], (shape, q)


def test_large_batch_and_determinism(cuda):
    rng = np.random.default_rng(1)
    imgs = [rng.integers(0, 256, (40, 72, 3), dtype=np.uint8) for _ in range(5)]
    imgs += [np.full((40, 72, 3), v, np.uint8) for v in (0, 255)]
    imgs = imgs * 20
    a = _encode(imgs, 90, cuda)
    b = _encode(imgs, 90, cuda)
    assert a == b and len(a) == len(imgs)
    for k in (0, 3, 5, 6):
        assert a[k] == J.encode(imgs[k], 90)


def test_float_prologue_is_numpy_round(cuda):
    from ssdnerf_b200 import video
    rng = np.random.default_rng(2)
    h, w = 33, 47
    x = rng.uniform(-0.001, 1.001, (4, h, w, 3)).astype(np.float32)
    ties = (rng.integers(0, 255, (h, w, 3)).astype(np.float32) + 0.5) / np.float32(255)   # .5 ties after * 255 in fp32
    x[1] = ties
    x[2, :4] = np.float32(-0.001)
    x[2, 4:8] = np.float32(1.001)
    u8 = np.round(x * 255).astype(np.uint8)
    assert np.array_equal(u8, J.round_u8(x))
    for q in (50, 95):
        got = video.encode_jpeg(torch.from_numpy(x).to(cuda), q)
        assert got == video.encode_jpeg(torch.from_numpy(u8).to(cuda), q)
        assert got == [J.encode(u, q) for u in u8]


def test_refusals(cuda):
    from ssdnerf_b200 import video
    with pytest.raises(ValueError, match='uint8 or float32'):
        video.encode_jpeg(torch.zeros(1, 8, 8, 4, device=cuda))
    with pytest.raises(ValueError, match='uint8 or float32'):
        video.encode_jpeg(torch.zeros(1, 8, 8, 3, dtype=torch.float16, device=cuda))
    with pytest.raises(ValueError, match='quality'):
        video.encode_jpeg(torch.zeros(1, 8, 8, 3, device=cuda), 0)
    with pytest.raises(ValueError, match='unsupported size'):
        video.encode_jpeg(torch.zeros(1, 0, 8, 3, device=cuda))
    assert video.encode_jpeg(torch.zeros(0, 8, 8, 3, device=cuda)) == []


# ------------------------------------------------------------------------------------------------ the tool, end to end
CAM_RES = 64


def _camera_dir(root):
    """a ShapeNet SRN style camera directory: 70 poses on a spiral at the cars' distance, intrinsics of a CAM_RES^2 view"""
    from tests.common import spiral_poses
    os.makedirs(os.path.join(root, 'pose'))
    for i, p in enumerate(spiral_poses(70, radius=1.3, seed=0)):
        np.savetxt(os.path.join(root, 'pose', f'{i:06d}.txt'), p.reshape(1, 16), fmt='%.9g', delimiter=' ')
    f = 131.25 * CAM_RES / 128
    with open(os.path.join(root, 'intrinsics.txt'), 'w') as fh:
        fh.write(f'{f} {CAM_RES / 2} {CAM_RES / 2} 0.\n0. 0. 0.\n1.\n{CAM_RES} {CAM_RES}\n')
    return root


def _model_files(tmp_path):
    """a config file of the cars unconditional model (with its EMA hook) and a checkpoint with a seeded random denoiser"""
    import ssdnerf_b200 as S
    from oracle import unet_port as up
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    hooks = [dict(type='ExponentialMovingAverageHook', module_keys=('diffusion_ema', 'decoder_ema'), interp_mode='lerp')]
    cfg_path = str(tmp_path / 'cars_uncond.py')
    with open(cfg_path, 'w') as f:
        f.write(f'model = {c["model"]!r}\ntrain_cfg = {c["train_cfg"]!r}\ntest_cfg = {c["test_cfg"]!r}\ncustom_hooks = {hooks!r}\n')
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg'])
    sd = up.random_state_dict(up.unet_spec(), seed=7, std=0.02)
    for diff in (model.diffusion, model.diffusion_ema):
        diff.denoising.load_state_dict(sd, strict=True)
    ckpt = str(tmp_path / 'iter_1.pth')
    torch.save(dict(meta=dict(iter=1), state_dict=model.state_dict()), ckpt)
    return cfg_path, ckpt


def _avi_frames(path):
    """(width, height, frame count from avih, [00dc payloads]) of an AVI the writer made"""
    data = open(path, 'rb').read()
    assert data[:4] == b'RIFF' and data[8:12] == b'AVI '
    i = data.index(b'avih') + 8
    avih = struct.unpack('<14I', data[i:i + 56])
    movi = data.index(b'movi')
    frames, k = [], movi + 4
    while data[k:k + 4] == b'00dc':
        size = struct.unpack('<I', data[k + 4:k + 8])[0]
        frames.append(data[k + 8:k + 8 + size])
        k += 8 + size + (size & 1)
    return avih[8], avih[9], avih[4], frames


def _sof_size(jpeg):
    i = jpeg.index(b'\xff\xc0')
    return struct.unpack('>HH', jpeg[i + 5:i + 9])


def test_orbit_tool_end_to_end(cuda, tmp_path):
    from ssdnerf_b200 import orbit, video
    from ssdnerf_b200.config import Config
    cams = _camera_dir(str(tmp_path / 'cams'))
    cfg_path, ckpt = _model_files(tmp_path)
    out = str(tmp_path / 'out')
    common = ['--cameras', cams, '--res', '32', '--fps', '5', '--sec', '1.2', '--batch-frames', '4', '--quality', '90']
    written = orbit.main([cfg_path, ckpt, '--seed', '0', '1', '--steps', '2', '--batch-scenes', '2', '--out-dir', out, '--mesh',
                          '--mesh-resolution', '48', '--save-scene'] + common)
    assert list(written) == ['seed_0', 'seed_1']
    assert sorted(os.listdir(out)) == sorted(f'seed_{s}.{e}' for s in (0, 1) for e in ('avi', 'stl', 'pth'))

    # the same model, poses and sampling by hand
    model = orbit.init_model(Config.fromfile(cfg_path), ckpt, cuda)
    assert 'diffusion' not in model._modules and 'decoder' not in model._modules      # ema_only
    for s in (0, 1):                               # the GUI's draw: mmgen's set_random_seed, then torch.randn on the CPU
        torch.manual_seed(s)
        ref = torch.randn((1,) + tuple(model.code_size))
        assert torch.equal(orbit.seed_noise(s, model.code_size), ref)
    poses, intr, hw = orbit.orbit_geometry(cams, 64, 32, 5, 1.2)
    assert poses.shape == (6, 4, 4) and hw == (32, 32)
    pose, intr0, _ = video.gui_camera(cams, 64)
    assert torch.equal(poses, video.surround_views(pose, num_frames=6)) and torch.equal(intr, intr0 * 0.5)
    for s in (0, 1):
        scene = torch.load(os.path.join(out, f'seed_{s}.pth'), weights_only=True)
        code, bitfield = scene['param']['code'].to(cuda), scene['param']['density_bitfield'].to(cuda)
        w, h, count, frames = _avi_frames(written[f'seed_{s}']['avi'])
        assert (w, h, count, len(frames)) == (32, 32, 6, 6)
        assert all(_sof_size(f) == (32, 32) for f in frames)
        assert frames == video.encode_jpeg(orbit.render_frames(model, code, bitfield, poses, intr, hw), 90)
        # --mesh: the file save_mesh writes for the same code
        model.save_mesh(str(tmp_path / 'mesh'), model.decoder_ema, code[None], ['m'], 48, 10)
        assert open(written[f'seed_{s}']['stl'], 'rb').read() == open(tmp_path / 'mesh' / 'm.stl', 'rb').read()
    # the sampled codes are those of val_uncond on the GUI's noise: two sampling runs on the device agree to round-off (on an H100
    # they differed by up to 4e-3 here after 2 steps of a random-weight denoiser), while another seed's noise moves the code by O(1)
    code_ref, _ = orbit.sample_seeds(model, [0, 1], 2)
    for s in (0, 1):
        saved = torch.load(os.path.join(out, f'seed_{s}.pth'), weights_only=True)['param']['code']
        err = float((saved - code_ref[s].cpu()).abs().max())
        print(f'seed {s}: resampled code max |diff| {err:.3g}')
        assert err < 2e-2
    assert float((code_ref[0] - code_ref[1]).abs().max()) > 0.5

    # --scene on the saved file: the same code; the occupancy grid is rebuilt with fresh jitter (as the GUI's Load scene does), so
    # the payloads equal a hand render under the same generator state, and the frames agree with the sampled scene's up to the grid
    out2 = str(tmp_path / 'out2')
    torch.manual_seed(5)
    written2 = orbit.main([cfg_path, ckpt, '--scene', os.path.join(out, 'seed_0.pth'), '--out-dir', out2] + common)
    assert list(written2) == ['seed_0'] and os.listdir(out2) == ['seed_0.avi']
    torch.manual_seed(5)
    code, bitfield = orbit.load_scene(model, os.path.join(out, 'seed_0.pth'))
    frames2 = _avi_frames(written2['seed_0']['avi'])[3]
    assert frames2 == video.encode_jpeg(orbit.render_frames(model, code, bitfield, poses, intr, hw), 90)
    scene = torch.load(os.path.join(out, 'seed_0.pth'), weights_only=True)
    assert torch.equal(code.cpu(), scene['param']['code'])
    a = orbit.render_frames(model, code, scene['param']['density_bitfield'].to(cuda), poses, intr, hw)
    b = orbit.render_frames(model, code, bitfield, poses, intr, hw)
    diff = (a - b).abs()
    print(f'--scene vs --seed frames: max |diff| {float(diff.max()):.3g}, mean {float(diff.mean()):.3g}')
    assert float(diff.mean()) < 2e-2


def test_scene_file_with_pre_activation_code(cuda, tmp_path):
    """test.py's save_dir files and the GUI's: code_ only -> code_activation(code_), applied to the loaded CPU tensor as the GUI does"""
    from ssdnerf_b200 import orbit
    from ssdnerf_b200.config import Config
    cfg_path, ckpt = _model_files(tmp_path)
    model = orbit.init_model(Config.fromfile(cfg_path), ckpt, cuda)
    code_ = torch.randn(model.code_size) * 0.5
    torch.save(dict(scene_name='x', param=dict(code_=code_)), tmp_path / 'x.pth')
    code, bitfield = orbit.load_scene(model, str(tmp_path / 'x.pth'))
    assert torch.equal(code.cpu(), model.code_activation(code_))
    assert bitfield.dtype == torch.uint8 and bitfield.numel() == model.grid_size ** 3 // 8
    torch.save(dict(param=dict(other=code_)), tmp_path / 'bad.pth')
    with pytest.raises(ValueError, match='not a scene file'):
        orbit.load_scene(model, str(tmp_path / 'bad.pth'))
