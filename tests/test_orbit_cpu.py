"""Orbit videos without a GPU: the numpy JPEG encoder (oracle/jpeg_port.py) reproduces every cv2.imencode file of the fixture byte for
byte (and live cv2 output when cv2 imports), the camera path and the GUI camera match the reference's, the Motion-JPEG AVI writer's
structure, and the argument refusals of the Python surface and of the C ABI (host-side checks, no device touched)."""
import ctypes
import os
import struct

import numpy as np
import pytest
import torch

from oracle import jpeg_port as J
from tests.common import GOLDEN

FIXTURE = os.path.join(GOLDEN, 'reference_video_v1.npz')


@pytest.fixture(scope='module')
def fx():
    return dict(np.load(FIXTURE))


def corpus(fx):
    """(name, rgb u8 [h, w, 3], quality, cv2 bytes) of the fixture"""
    out = []
    for i, name in enumerate(fx['jpeg_names']):
        h, w = (int(v) for v in fx['jpeg_shapes'][i])
        img = fx['jpeg_pixels'][fx['jpeg_pixel_offsets'][i]:fx['jpeg_pixel_offsets'][i + 1]].reshape(h, w, 3)
        data = fx['jpeg_files'][fx['jpeg_file_offsets'][i]:fx['jpeg_file_offsets'][i + 1]].tobytes()
        out.append((str(name), img, int(fx['jpeg_quality'][i]), data))
    return out


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


# ------------------------------------------------------------------------------------------------ JPEG oracle
def test_corpus_covers_the_edge_cases(fx):
    items = corpus(fx)
    shapes = {img.shape[:2] for _, img, _, _ in items}
    assert {(1, 1), (8, 8), (7, 9), (16, 15), (17, 33), (128, 128), (256, 256), (255, 257)} <= shapes
    assert {q for _, _, q, _ in items} == {1, 25, 50, 75, 95, 100}
    assert any(b'\xff\x00' in data[623:-2] for *_, data in items), 'no stuffed 0xFF byte in the corpus'
    # a DC difference of category 11 and a ZRL: re-derive from the oracle's coefficients
    cat11 = zrl = False
    for name, img, q, _ in items:
        if not name.startswith('zrl_dc11') or img.shape[0] < 16:
            continue
        coef = J.mcu_coefficients(img, q).reshape(-1, 6, 64)
        dc = coef[:, :4, 0].reshape(-1)
        cat11 |= bool((np.abs(np.diff(dc)) >= 1024).any())
        for blk in coef.reshape(-1, 64):
            nz = np.flatnonzero(blk[1:])
            zrl |= bool(len(nz) and (np.diff(np.concatenate([[-1], nz])) > 16).any())
    assert cat11 and zrl


def test_oracle_reproduces_every_fixture_file(fx):
    bad = [name for name, img, q, data in corpus(fx) if J.encode(img, q) != data]
    assert not bad, f'{len(bad)} files differ, e.g. {bad[:5]}'


def test_oracle_matches_live_cv2():
    cv2 = _cv2()
    if cv2 is None:
        pytest.skip('cv2 not importable')
    rng = np.random.default_rng(3)
    for h, w in [(3, 5), (23, 31), (40, 24), (33, 17)]:
        for q in (10, 60, 90):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            img[: h // 2] = img[: h // 2] // 32 * 32                  # some flat runs next to noise
            ref = cv2.imencode('.jpg', np.ascontiguousarray(img[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
            assert J.encode(img, q) == ref, (h, w, q)


def test_oracle_header_layout():
    hdr = J.header(255, 257, 95)
    assert len(hdr) == 623
    markers = []
    i = 2
    while i < len(hdr):
        assert hdr[i] == 0xFF
        markers.append(hdr[i + 1])
        i += 2 + struct.unpack('>H', hdr[i + 2:i + 4])[0]
    assert hdr[:2] == b'\xff\xd8' and markers == [0xE0, 0xDB, 0xDB, 0xC0, 0xC4, 0xC4, 0xC4, 0xC4, 0xDA]
    assert hdr[6:11] == b'JFIF\0' and hdr[11:13] == b'\x01\x01'


def test_quality_scaling():
    assert (J.quant_tables(50)[0] == J.LUMA_Q).all() and (J.quant_tables(50)[1] == J.CHROMA_Q).all()
    assert (J.quant_tables(100)[0] == 1).all()
    assert J.quant_tables(1)[0].max() == 255 and J.quant_tables(1)[0].min() == 255
    for q in (0, 101):
        with pytest.raises(ValueError):
            J.quant_tables(q)


def test_round_u8_is_numpy_round_over_the_render_range():
    x = np.concatenate([np.linspace(-0.001, 1.001, 100001, dtype=np.float32),
                        (np.arange(255, dtype=np.float32) + 0.5) / np.float32(255)])    # .5 ties after * 255
    assert np.array_equal(J.round_u8(x), np.round(x * 255).astype(np.uint8))


# ------------------------------------------------------------------------------------------------ camera path
def test_surround_views_match_the_reference(fx):
    from ssdnerf_b200 import video
    pose = torch.from_numpy(fx['gui_pose'])
    for key in [k for k in fx if k.startswith('surround_')]:
        _, num, amp = key.split('_')
        got = video.surround_views(pose, angle_amp=float(amp), num_frames=int(num))
        ref = fx[key]
        assert got.shape == ref.shape and got.dtype == torch.float32
        np.testing.assert_allclose(got.numpy(), ref, rtol=0, atol=2e-6)
    default = video.surround_views(pose)
    assert default.shape == (60, 4, 4)


def test_look_at_is_orthonormal():
    from ssdnerf_b200 import video
    pos = torch.tensor([[1.0, 2.0, 0.5], [-2.0, 0.3, -1.0]])
    rot = video.look_at(pos, torch.zeros_like(pos), torch.tensor([0.0, 0.0, 1.0]))
    eye = rot.transpose(-1, -2) @ rot
    np.testing.assert_allclose(eye.numpy(), np.broadcast_to(np.eye(3), eye.shape), atol=1e-6)
    np.testing.assert_allclose(rot[..., 2].numpy(), (-pos / pos.norm(dim=-1, keepdim=True)).numpy(), atol=1e-6)


def test_gui_camera_reads_an_srn_scene_directory(fx, tmp_path):
    from ssdnerf_b200 import video
    pose_dir = tmp_path / 'pose'
    pose_dir.mkdir()
    cid = int(fx['camera_id'])
    for i in range(cid + 3):                       # the listing is sorted: decoys around the chosen name
        (pose_dir / f'{i:06d}.txt').write_text(' '.join(['0.5'] * 16))
    (pose_dir / str(fx['camera_pose_name'])).write_text(str(fx['camera_pose_text']))
    (tmp_path / 'intrinsics.txt').write_text(str(fx['camera_intrinsics_text']))
    pose, intr, hw = video.gui_camera(str(tmp_path), cid)
    assert np.array_equal(pose.numpy(), fx['gui_pose'])
    assert intr.dtype == torch.float32 and intr.tolist() == [131.25, 131.25, 64.0, 64.0] and hw == (128, 128)
    with pytest.raises(ValueError, match='out of range'):
        video.gui_camera(str(tmp_path), cid + 3)


# ------------------------------------------------------------------------------------------------ AVI
def _riff_chunks(data, start, end):
    """(fourcc, payload offset, size) of the chunks in data[start:end]"""
    out, i = [], start
    while i < end:
        fourcc, size = data[i:i + 4], struct.unpack('<I', data[i + 4:i + 8])[0]
        out.append((fourcc, i + 8, size))
        i += 8 + size + (size & 1)
    assert i == end
    return out


def _frames(n, seed=0):
    rng = np.random.default_rng(seed)
    return [J.encode(rng.integers(0, 256, (24, 40, 3), dtype=np.uint8), 80) for _ in range(n)]


def test_avi_structure(tmp_path):
    from ssdnerf_b200 import video
    jpegs = _frames(5)
    jpegs[2] = jpegs[2] + b'\0'                   # force one odd-length payload
    if len(jpegs[2]) % 2 == 0:
        jpegs[2] = jpegs[2] + b'\0'
    path = tmp_path / 'a.avi'
    video.write_avi(str(path), jpegs, 40, 24, 30)
    data = path.read_bytes()
    assert data[:4] == b'RIFF' and data[8:12] == b'AVI ' and struct.unpack('<I', data[4:8])[0] == len(data) - 8
    top = _riff_chunks(data, 12, len(data))
    assert [c[0] for c in top] == [b'LIST', b'LIST', b'idx1']
    hdrl, movi, idx1 = top
    assert data[hdrl[1]:hdrl[1] + 4] == b'hdrl' and data[movi[1]:movi[1] + 4] == b'movi'
    h = _riff_chunks(data, hdrl[1] + 4, hdrl[1] + hdrl[2])
    assert [c[0] for c in h] == [b'avih', b'LIST'] and h[0][2] == 56
    avih = struct.unpack('<14I', data[h[0][1]:h[0][1] + 56])
    assert avih[0] == 33333 and avih[3] == 0x10 and avih[4] == 5 and avih[6] == 1 and avih[8:10] == (40, 24)
    strl = _riff_chunks(data, h[1][1] + 4, h[1][1] + h[1][2])
    assert data[h[1][1]:h[1][1] + 4] == b'strl' and [c[0] for c in strl] == [b'strh', b'strf']
    strh = data[strl[0][1]:strl[0][1] + strl[0][2]]
    assert strh[:8] == b'vidsMJPG' and struct.unpack('<II', strh[20:28]) == (1, 30) and struct.unpack('<I', strh[32:36])[0] == 5
    strf = struct.unpack('<IiiHH4sI', data[strl[1][1]:strl[1][1] + 24])
    assert strf == (40, 40, 24, 1, 24, b'MJPG', 40 * 24 * 3)
    frames = _riff_chunks(data, movi[1] + 4, movi[1] + movi[2])
    assert len(frames) == 5
    for (fourcc, off, size), j in zip(frames, jpegs):
        assert fourcc == b'00dc' and size == len(j) and data[off:off + size] == j
        if size & 1:
            assert data[off + size] == 0
    index = [struct.unpack('<4sIII', data[idx1[1] + 16 * k:idx1[1] + 16 * k + 16]) for k in range(idx1[2] // 16)]
    assert len(index) == 5
    for (ck, flags, off, size), (_, payload, fsize) in zip(index, frames):
        assert ck == b'00dc' and flags == 0x10 and size == fsize
        assert movi[1] + off == payload - 8                     # offsets count from the 'movi' fourcc


def test_avi_fractional_rate(tmp_path):
    from ssdnerf_b200 import video
    video.write_avi(str(tmp_path / 'b.avi'), _frames(2), 40, 24, 29.97)
    data = (tmp_path / 'b.avi').read_bytes()
    i = data.index(b'strh') + 8
    assert struct.unpack('<II', data[i + 20:i + 28]) == (100, 2997)


def test_avi_reads_back_with_cv2(tmp_path):
    cv2 = _cv2()
    if cv2 is None:
        pytest.skip('cv2 not importable')
    from ssdnerf_b200 import video
    jpegs = _frames(7, seed=1)
    path = str(tmp_path / 'c.avi')
    video.write_avi(path, jpegs, 40, 24, 30)
    # OpenCV's own Motion-JPEG reader decodes the payloads with imdecode: equal pixels; ffmpeg's (when built in) decodes with its own
    # IDCT and chroma upsampling, so only the frame count, size and rate are compared there
    for backend in (cv2.CAP_OPENCV_MJPEG, cv2.CAP_FFMPEG):
        cap = cv2.VideoCapture(path, backend)
        if not cap.isOpened():
            assert backend != cv2.CAP_OPENCV_MJPEG, 'OpenCV MJPEG reader refused the file'
            continue
        assert cap.get(cv2.CAP_PROP_FPS) == 30
        got = []
        while True:
            ok, frame = cap.read()
            if not ok:
                break
            got.append(frame)
        cap.release()
        assert len(got) == 7 and all(f.shape == (24, 40, 3) for f in got)
        if backend == cv2.CAP_OPENCV_MJPEG:
            for frame, j in zip(got, jpegs):
                assert np.array_equal(frame, cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR))


def test_avi_refusals(tmp_path, monkeypatch):
    from ssdnerf_b200 import video
    p = str(tmp_path / 'd.avi')
    with pytest.raises(ValueError, match='no frames'):
        video.write_avi(p, [], 8, 8, 30)
    with pytest.raises(ValueError, match='fps'):
        video.write_avi(p, _frames(1), 40, 24, 0)
    with pytest.raises(ValueError, match='width and height'):
        video.write_avi(p, _frames(1), 0, 24, 30)
    monkeypatch.setattr(video, 'AVI_MAX_BYTES', 1000)
    with pytest.raises(ValueError, match='1 GB'):
        video.write_avi(p, _frames(3), 40, 24, 30)
    assert not os.path.exists(p)


# ------------------------------------------------------------------------------------------------ refusals
def test_encode_jpeg_refuses_bad_input():
    from ssdnerf_b200 import _lib, video
    with pytest.raises(_lib.SSDNeRFNativeError, match='CUDA'):
        video.encode_jpeg(torch.zeros(1, 8, 8, 3, dtype=torch.uint8))


def test_abi_sizes_and_host_validation():
    from ssdnerf_b200 import _lib
    L = _lib.lib()
    assert L.ssdnerf_jpeg_workspace_bytes(0, 8, 8) == 0 and L.ssdnerf_jpeg_output_bound(1, 0, 8) == 0
    assert L.ssdnerf_jpeg_workspace_bytes(1, 65536, 8) == 0 and L.ssdnerf_jpeg_output_bound(1, 8, 65536) == 0
    assert L.ssdnerf_jpeg_workspace_bytes(1, 65535, 65535) > 0
    assert L.ssdnerf_jpeg_output_bound(3, 17, 33) == 3 * (623 + 2 + 2 * 1245 * 2 * 3)
    assert L.ssdnerf_jpeg_workspace_bytes(1, 16, 16) % 256 == 0
    fake = ctypes.c_void_p(1 << 20)
    ws, ob = L.ssdnerf_jpeg_workspace_bytes(2, 16, 16), L.ssdnerf_jpeg_output_bound(2, 16, 16)
    S = _lib.SSDNERF_ERR_ARG if hasattr(_lib, 'SSDNERF_ERR_ARG') else -2
    cases = [
        ((None, 2, 16, 16, 95, fake, ws, fake, ob, fake, None), 'rgb'),
        ((fake, 0, 16, 16, 95, fake, ws, fake, ob, fake, None), 'n >= 1'),
        ((fake, 2, 16, 70000, 95, fake, ws, fake, ob, fake, None), 'n >= 1'),
        ((fake, 2, 16, 16, 0, fake, ws, fake, ob, fake, None), 'quality'),
        ((fake, 2, 16, 16, 101, fake, ws, fake, ob, fake, None), 'quality'),
        ((fake, 2, 16, 16, 95, fake, ws - 1, fake, ob, fake, None), 'workspace'),
        ((fake, 2, 16, 16, 95, ctypes.c_void_p((1 << 20) + 16), ws, fake, ob, fake, None), 'workspace'),
        ((fake, 2, 16, 16, 95, fake, ws, fake, ob - 1, fake, None), 'output_bound'),
        ((fake, 2, 16, 16, 95, fake, ws, fake, ob, None, None), 'offsets'),
    ]
    for fn in (L.ssdnerf_jpeg_encode_u8, L.ssdnerf_jpeg_encode_f32):
        for args, msg in cases:
            assert fn(*args) == S, (fn, msg)
            assert msg in L.ssdnerf_last_error().decode()
    assert L.ssdnerf_jpeg_encode_f32(ctypes.c_void_p((1 << 20) + 2), 2, 16, 16, 95, fake, ws, fake, ob, fake, None) == S
