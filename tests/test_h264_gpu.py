"""The device H.264 encoder (csrc/h264.cu) against the numpy encoder (oracle/h264_port.py): the bytes of the MP4 corpus one frame at a
time and in mixed, shuffled batches, u8 and fp32, determinism over a 120-frame batch, the C ABI's refusals and the orbit tool's mp4."""
import os
import struct

import numpy as np
import pytest
import torch

from oracle import h264_port as H
from tests.golden.make_golden_h264 import FPS, corpus
from tests.test_h264_cpu import FIXTURE, boxes, child

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def items():
    return corpus()


def mp4_parts(data):
    """(sps, pps, samples) of a one-track MP4 file written by video.write_mp4"""
    top = boxes(data)
    moov, mdat = top[1], top[2]
    mdia = child(data, child(data, moov, b'trak'), b'mdia')
    stbl = child(data, child(data, mdia, b'minf'), b'stbl')
    stsz = child(data, stbl, b'stsz')
    n = struct.unpack('>I', data[stsz[1] + 8:stsz[1] + 12])[0]
    sizes = struct.unpack(f'>{n}I', data[stsz[1] + 12:stsz[1] + 12 + 4 * n])
    avcc = child(data, child(data, child(data, stbl, b'stsd'), b'avc1', skip=8), b'avcC', skip=78)
    rec = data[avcc[1]:avcc[2]]
    ls = struct.unpack('>H', rec[6:8])[0]
    lp = struct.unpack('>H', rec[9 + ls:11 + ls])[0]
    samples, k = [], mdat[1]
    for s in sizes:
        samples.append(data[k:k + s])
        k += s
    return rec[8:8 + ls], rec[11 + ls:11 + ls + lp], samples


def test_corpus_bytes_whole_and_one_by_one(items):
    from ssdnerf_b200 import video
    z = np.load(FIXTURE)
    for name, qp, frames in items:
        sps, pps, samples = mp4_parts(z[f'{name}/mp4'].tobytes())
        got = video.encode_h264(torch.from_numpy(frames).cuda(), qp, FPS)
        assert got == (sps, pps, samples), name
        for i in range(len(frames)):
            s1, p1, a1 = video.encode_h264(torch.from_numpy(frames[i:i + 1]).cuda(), qp, FPS, first_frame=i)
            assert (s1, p1, a1) == (sps, pps, samples[i:i + 1]), (name, i)


def test_mixed_shuffled_batches(items):
    from ssdnerf_b200 import video
    rng = np.random.default_rng(11)
    groups = {}
    for name, qp, frames in items:
        if frames.shape[1] * frames.shape[2] <= 128 * 128:
            groups.setdefault(frames.shape[1:3], []).append(frames)
    for hw, fl in groups.items():
        frames = np.concatenate(fl)
        frames = frames[rng.permutation(len(frames))]
        for qp in (H.MIN_QP, 20, 30, 51):
            for first in (0, 1):
                got = video.encode_h264(torch.from_numpy(frames).cuda(), qp, FPS, first_frame=first)
                assert got == H.encode(frames, qp, FPS, first_frame=first), (hw, qp, first)


def test_float_prologue_is_numpy_round():
    from ssdnerf_b200 import video
    g = torch.Generator().manual_seed(5)
    x = torch.rand(3, 18, 34, 3, generator=g) * 1.004 - 0.002
    x[0, 0, :4, 0] = torch.tensor([0.5 / 255, 1.5 / 255, 2.5 / 255, float('nan')])
    got = video.encode_h264(x.cuda(), 23, FPS)
    assert got == H.encode(H.round_u8(x.numpy()), 23, FPS)


def test_large_batch_deterministic():
    from ssdnerf_b200 import video
    from tests.golden.make_golden_h264 import gradient
    rng = np.random.default_rng(3)
    frames = torch.from_numpy(np.stack([gradient(256, 256, rng) for _ in range(120)])).cuda().float() / 255
    a = video.encode_h264(frames, 20, FPS)
    b = video.encode_h264(frames, 20, FPS)
    assert a == b
    for i in (0, 1, 57, 119):
        assert video.encode_h264(frames[i:i + 1], 20, FPS, first_frame=i)[2][0] == a[2][i]
    ref = H.encode(H.round_u8(frames[:2].cpu().numpy()), 20, FPS)
    assert a[:2] == ref[:2] and a[2][:2] == ref[2]


def test_capi_refusals():
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    n, h, w = 2, 32, 48
    ws, ob = L.ssdnerf_h264_workspace_bytes(n, h, w), L.ssdnerf_h264_output_bound(n, h, w)
    assert ws > 0 and ob > 0
    for bad in ((0, h, w), (n, 31, w), (n, h, 47), (n, 1, w), (n, 16 * 544, 16), (n, 16 * 200, 16 * 200)):
        assert L.ssdnerf_h264_workspace_bytes(*bad) == 0 and L.ssdnerf_h264_output_bound(*bad) == 0
    rgb = torch.zeros(n, h, w, 3, dtype=torch.uint8, device='cuda')
    rgbf = torch.zeros(n * h * w * 3 + 1, dtype=torch.float32, device='cuda')
    work = torch.empty(ws + 512, dtype=torch.uint8, device='cuda')
    out = torch.empty(ob, dtype=torch.uint8, device='cuda')
    off = torch.empty(n + 4, dtype=torch.int64, device='cuda')
    p = lambda t: N.ptr(t).value
    base = dict(rgb=p(rgb), n=n, h=h, w=w, qp=20, num=30, den=1, first=0, work=p(work), ws=ws, out=p(out), ob=ob, off=p(off))
    cases = [dict(rgb=0), dict(n=0), dict(h=31), dict(w=47), dict(qp=H.MIN_QP - 1), dict(qp=52), dict(num=0), dict(den=0),
             dict(work=p(work) + 128), dict(ws=ws - 1), dict(work=0), dict(ob=ob - 1), dict(out=0), dict(off=0), dict(off=p(off) + 4)]
    torch.cuda.synchronize()
    for c in cases:
        a = dict(base, **c)
        r = L.ssdnerf_h264_encode_u8(a['rgb'], a['n'], a['h'], a['w'], a['qp'], a['num'], a['den'], a['first'], a['work'], a['ws'],
                                     a['out'], a['ob'], a['off'], N.stream_ptr())
        assert r == -2, c
    r = L.ssdnerf_h264_encode_f32(p(rgbf) + 2, n, h, w, 20, 30, 1, 0, p(work), ws, p(out), ob, p(off), N.stream_ptr())
    assert r == -2
    assert 'aligned' in L.ssdnerf_last_error().decode()
    with pytest.raises(ValueError):
        from ssdnerf_b200 import video
        video.encode_h264(rgb[:, :31], 20)
    with pytest.raises(ValueError):
        video.encode_h264(rgb, 9)
    with pytest.raises(ValueError):
        video.encode_h264(rgb[:0], 20)


def test_orbit_tool_mp4(cuda, tmp_path):
    from tests.test_orbit_gpu import _camera_dir, _model_files
    from ssdnerf_b200 import orbit, video
    from ssdnerf_b200.config import Config
    cams = _camera_dir(str(tmp_path / 'cams'))
    cfg_path, ckpt = _model_files(tmp_path)
    out = str(tmp_path / 'out')
    written = orbit.main([cfg_path, ckpt, '--cameras', cams, '--seed', '3', '--steps', '2', '--out-dir', out, '--res', '32', '--fps',
                          '5', '--sec', '1.4', '--batch-frames', '3', '--format', 'mp4', '--qp', '24', '--save-scene'])
    assert sorted(os.listdir(out)) == ['seed_3.mp4', 'seed_3.pth']
    sps, pps, samples = mp4_parts(open(written['seed_3']['mp4'], 'rb').read())
    model = orbit.init_model(Config.fromfile(cfg_path), ckpt, cuda)
    scene = torch.load(os.path.join(out, 'seed_3.pth'), weights_only=True)
    code, bitfield = scene['param']['code'].to(cuda), scene['param']['density_bitfield'].to(cuda)
    poses, intr, hw = orbit.orbit_geometry(cams, 64, 32, 5, 1.4)
    frames = orbit.render_frames(model, code, bitfield, poses, intr, hw)
    assert len(samples) == poses.size(0) == 7
    assert (sps, pps, samples) == video.encode_h264(frames, 24, 5)
    try:
        import cv2
    except ImportError:
        return
    cap = cv2.VideoCapture(written['seed_3']['mp4'])
    if not cap.isOpened():
        return                                      # an OpenCV build without an H.264 decoder
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    u8 = H.round_u8(frames.cpu().numpy())
    for i in range(len(samples)):
        ok, d = cap.read()
        assert ok
        y, _, _ = H.decoded_planes(u8[i], 24, i & 1)
        assert np.array_equal(d.reshape(-1)[:y.size].reshape(y.shape), y)
