"""H.264 orbit videos without a GPU: the numpy encoder (oracle/h264_port.py) against FFmpeg's decoder (the decode pinned in
reference_h264_v1.npz, and live cv2 when it imports), the MP4 box structure of video.write_mp4, and the refusals."""
import os
import struct
from fractions import Fraction

import numpy as np
import pytest

from oracle import h264_port as H
from tests.common import GOLDEN
from tests.golden.make_golden_h264 import FPS, WINDOW, corpus, digest

FIXTURE = os.path.join(GOLDEN, 'reference_h264_v1.npz')
# decoded RGB against the source, on the render-like (gradient) frames' stored windows: 4:2:0 and the quantiser are the only losses
PSNR_BAR = {20: 42.0, 30: 37.0}
# cv2's BGR against BT.601 limited-range YCbCr -> RGB of the decoded planes with nearest chroma upsampling, in float and rounded:
# swscale works in fixed point (a rounding step of up to 1) and interpolates chroma between neighbours where we repeat it, which
# moves a sample by at most the neighbouring chroma difference times the matrix gain; on this corpus the largest difference is 3
BGR_TOL = 3


@pytest.fixture(scope='module')
def fixture():
    return np.load(FIXTURE)


@pytest.fixture(scope='module')
def items():
    return corpus()


def bgr_of(y, cb, cr):
    cb = np.repeat(np.repeat(cb, 2, 0), 2, 1).astype(np.float64) - 128
    cr = np.repeat(np.repeat(cr, 2, 0), 2, 1).astype(np.float64) - 128
    yy = (y.astype(np.float64) - 16) * 255 / 219
    k = 255 / 224
    r = yy + k * 1.402 * cr
    g = yy - k * (1.772 * 0.114 / 0.587 * cb + 1.402 * 0.299 / 0.587 * cr)
    b = yy + k * 1.772 * cb
    return np.clip(np.rint(np.stack([b, g, r], -1)), 0, 255)


def boxes(data, start=0, end=None):
    """[(type, payload start, payload end)] of the boxes in data[start:end]"""
    end = len(data) if end is None else end
    out = []
    while start < end:
        size, kind = struct.unpack('>I4s', data[start:start + 8])
        assert size >= 8 and start + size <= end
        out.append((kind, start + 8, start + size))
        start += size
    return out


def child(data, parent, kind, skip=0):
    for k, s, e in boxes(data, parent[1] + skip, parent[2]):
        if k == kind:
            return k, s, e
    raise AssertionError(f'no {kind} box')


def test_min_qp_derivation():
    assert H.MIN_QP == 10
    assert H.level_bound(H.MIN_QP) <= H.MAX_LEVEL < H.level_bound(H.MIN_QP - 1)
    assert all(H.level_bound(q) <= H.MAX_LEVEL for q in range(H.MIN_QP, 52))


def test_oracle_files_equal_fixture(fixture, items, tmp_path):
    from ssdnerf_b200.video import write_mp4
    for name, qp, frames in items:
        sps, pps, aus = H.encode(frames, qp, FPS)
        path = tmp_path / (name + '.mp4')
        write_mp4(path, sps, pps, aus, frames.shape[2], frames.shape[1], FPS)
        assert path.read_bytes() == fixture[f'{name}/mp4'].tobytes(), name


def test_decoded_luma_is_deblocked_reconstruction(fixture, items):
    """the whole decoded luma plane through its digest, the top-left window sample by sample, and the window's BGR"""
    for name, qp, frames in items:
        for i, f in enumerate(frames):
            y, cb, cr = H.decoded_planes(f, qp, i & 1)
            assert np.array_equal(digest(y), fixture[f'{name}/y_sha256'][i]), (name, i)
            assert np.array_equal(y[:WINDOW, :WINDOW], fixture[f'{name}/y'][i]), (name, i)
            d = np.abs(bgr_of(y, cb, cr)[:WINDOW, :WINDOW] - fixture[f'{name}/bgr'][i])
            assert d.max() <= BGR_TOL, (name, i, d.max())


def test_quality(fixture, items):
    for name, qp, frames in items:
        if qp not in PSNR_BAR or not (name.startswith('r128') or name.startswith('r256') or name.startswith('big')):
            continue
        for i, f in enumerate(frames):
            if f.min() == f.max():
                continue
            rgb = fixture[f'{name}/bgr'][i][..., ::-1].astype(np.float64)
            psnr = 10 * np.log10(255 ** 2 / ((rgb - f[:WINDOW, :WINDOW]) ** 2).mean())
            assert psnr >= PSNR_BAR[qp], (name, i, psnr)


def test_live_decoder(items, tmp_path):
    cv2 = pytest.importorskip('cv2')
    from ssdnerf_b200.video import write_mp4
    for name, qp, frames in items[:12]:
        sps, pps, aus = H.encode(frames, qp, FPS)
        path = str(tmp_path / (name + '.mp4'))
        write_mp4(path, sps, pps, aus, frames.shape[2], frames.shape[1], FPS)
        cap = cv2.VideoCapture(path)
        if not cap.isOpened():
            pytest.skip('this OpenCV build has no H.264 decoder')
        cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
        h, w = frames.shape[1:3]
        for i, f in enumerate(frames):
            ok, d = cap.read()
            assert ok, (name, i)
            y, _, _ = H.decoded_planes(f, qp, i & 1)
            assert np.array_equal(d.reshape(-1)[:h * w].reshape(h, w), y), (name, i)


def test_emulation_prevention_in_corpus(items):
    from tests.golden.make_golden_h264 import unescape
    name, qp, frames = next(it for it in items if it[0] == 'epb_q10')
    _, _, aus = H.encode(frames, qp, FPS)
    assert sum(len(a) - 5 - len(unescape(a[4:])) for a in aus) > 0
    assert H.ep_bytes(b'\0\0\0\0\1\0\0\3\0\0\4') == b'\0\0\3\0\0\3\1\0\0\3\3\0\0\4'


@pytest.mark.parametrize('fps', [30, Fraction(30000, 1001), 12.5])
def test_mp4_structure(fps, tmp_path):
    from ssdnerf_b200.video import write_mp4
    frames = np.random.default_rng(7).integers(0, 256, (5, 34, 18, 3), dtype=np.uint8)
    sps, pps, aus = H.encode(frames, 24, fps)
    path = tmp_path / 'v.mp4'
    write_mp4(path, sps, pps, aus, 18, 34, fps)
    data = path.read_bytes()
    top = boxes(data)
    assert [k for k, _, _ in top] == [b'ftyp', b'moov', b'mdat']
    moov, mdat = top[1], top[2]
    trak = child(data, moov, b'trak')
    mdia = child(data, trak, b'mdia')
    fr = Fraction(fps).limit_denominator(1_000_000)
    mdhd = child(data, mdia, b'mdhd')
    assert struct.unpack('>II', data[mdhd[1] + 12:mdhd[1] + 20]) == (fr.numerator, 5 * fr.denominator)
    assert data[child(data, mdia, b'hdlr')[1] + 8:][:4] == b'vide'
    stbl = child(data, child(data, mdia, b'minf'), b'stbl')
    assert b'stss' not in [k for k, _, _ in boxes(data, stbl[1], stbl[2])]
    stsz = child(data, stbl, b'stsz')
    n = struct.unpack('>I', data[stsz[1] + 8:stsz[1] + 12])[0]
    assert n == 5 and list(struct.unpack('>5I', data[stsz[1] + 12:stsz[1] + 32])) == [len(a) for a in aus]
    stts = child(data, stbl, b'stts')
    assert struct.unpack('>III', data[stts[1] + 4:stts[1] + 16]) == (1, 5, fr.denominator)
    stco = child(data, stbl, b'stco')
    off = struct.unpack('>I', data[stco[1] + 8:stco[1] + 12])[0]
    assert off == mdat[1] and data[off:mdat[2]] == b''.join(aus)
    stsd = child(data, stbl, b'stsd')
    avc1 = child(data, stsd, b'avc1', skip=8)
    avcc = child(data, avc1, b'avcC', skip=78)
    rec = data[avcc[1]:avcc[2]]
    ls = struct.unpack('>H', rec[6:8])[0]
    assert rec[:4] == bytes([1, 66, 0xC0, sps[3]]) and rec[8:8 + ls] == sps
    lp = struct.unpack('>H', rec[9 + ls:11 + ls])[0]
    assert rec[8 + ls] == 1 and rec[11 + ls:11 + ls + lp] == pps
    try:
        import cv2
    except ImportError:
        return
    cap = cv2.VideoCapture(str(path))
    if not cap.isOpened():
        return                                      # an OpenCV build without an H.264 decoder
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 5
    assert abs(cap.get(cv2.CAP_PROP_FPS) - float(fr)) < 1e-6


def test_refusals(tmp_path):
    from ssdnerf_b200 import video
    f = np.zeros((1, 16, 16, 3), np.uint8)
    for h, w in ((15, 16), (16, 17), (1, 2), (16 * 544, 16), (16 * 200, 16 * 200)):
        with pytest.raises(ValueError):
            H.check_args(h, w, 20)
    for qp in (H.MIN_QP - 1, 52):
        with pytest.raises(ValueError):
            H.encode(f, qp)
    sps, pps, aus = H.encode(f, 20)
    with pytest.raises(ValueError, match='no frames'):
        video.write_mp4(tmp_path / 'a.mp4', sps, pps, [], 16, 16, 30)
    with pytest.raises(ValueError, match='4 GB'):
        video.write_mp4(tmp_path / 'b.mp4', sps, pps, [b'\0' * (1 << 20)] * 4096, 16, 16, 30)
    assert not (tmp_path / 'b.mp4').exists()


def test_levels():
    assert H.level_idc(256, 256, 30) == 13              # 256 macroblocks at 30 fps: 7680 per second
    assert H.level_idc(16, 16, 30) == 10
    assert H.level_idc(1080, 1920, 30) == 40
    assert H.level_idc(1080, 1920, 60) == 42
    assert H.level_idc(8688, 8688, 1000) == 52
