"""Orbit videos of scenes: the camera path and file writing of the reference GUI's "Export video" (lib/core/ssdnerf_gui.py,
lib/core/utils/camera_utils.py), without a window or ffmpeg.

Frames are encoded on the device as baseline JPEG (csrc/jpeg.cu, byte-identical to cv2.imencode with libjpeg-turbo's defaults); only
the compressed files are copied to the host, once per call, and written into a Motion-JPEG AVI that ffmpeg, VLC and mpv play.
Alternatively they are encoded as all-intra H.264 (csrc/h264.cu, oracle/h264_port.py) and written into an MP4 file that browsers
also play."""
import math
import os
import struct
from fractions import Fraction

import numpy as np
import torch

from . import _lib as N
from .datasets import load_intrinsics, load_pose

AVI_MAX_BYTES = 1 << 30         # AVI 1.0 (no OpenDML): one RIFF list, kept under 1 GB for players that read 32-bit offsets signed
AVIF_HASINDEX = 0x10
AVIIF_KEYFRAME = 0x10
MP4_MAX_BYTES = 1 << 32         # 32-bit stco chunk offsets and box sizes
H264_MIN_QP = 10                # SSDNERF_H264_MIN_QP: below it Baseline's level codes cannot hold every 8-bit residual


def encode_jpeg(frames, quality=95):
    """JPEG files (list of bytes) of CUDA RGB frames [n, h, w, 3], uint8 or float32; float samples become rint(x * 255) in float32,
    clamped to [0, 255] (np.round(x * 255).astype(np.uint8) over the renderer's range).  Each file equals
    cv2.imencode('.jpg', frame[..., ::-1], [IMWRITE_JPEG_QUALITY, quality]) of the u8 frame; 1 <= h, w <= 65535."""
    N.require_cuda(frames)
    if frames.dim() != 4 or frames.shape[-1] != 3 or frames.dtype not in (torch.uint8, torch.float32):
        raise ValueError(f'encode_jpeg: frames must be uint8 or float32 [n, h, w, 3], got {frames.dtype} {tuple(frames.shape)}')
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= int(quality) <= 100:
        raise ValueError(f'encode_jpeg: quality must be an int in [1, 100], got {quality!r}')
    n, h, w, _ = frames.shape
    if n == 0:
        return []
    L, dev, stream = N.lib(), frames.device, N.stream_ptr()
    ws_bytes, out_bytes = L.ssdnerf_jpeg_workspace_bytes(n, h, w), L.ssdnerf_jpeg_output_bound(n, h, w)
    if ws_bytes == 0:
        raise ValueError(f'encode_jpeg: unsupported size n={n} h={h} w={w} (1 <= h, w <= 65535)')
    frames = frames.contiguous()
    work = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    fn = L.ssdnerf_jpeg_encode_u8 if frames.dtype == torch.uint8 else L.ssdnerf_jpeg_encode_f32
    N.check(fn(N.ptr(frames), n, h, w, int(quality), N.ptr(work), ws_bytes, N.ptr(out), out_bytes, N.ptr(offsets), stream))
    off = offsets.cpu().tolist()
    data = out[:off[-1]].cpu().numpy().tobytes()
    return [data[off[i]:off[i + 1]] for i in range(n)]


def encode_h264(frames, qp=20, fps=30, first_frame=0):
    """(sps, pps, [access unit]) of CUDA RGB frames [n, h, w, 3], uint8 or float32 (float samples as in encode_jpeg): Constrained
    Baseline H.264, every frame one IDR access unit of I_16x16 macroblocks at the constant `qp` (header section 13).  sps / pps are
    NAL units without start code; each access unit is its slice NAL unit behind a 4-byte big-endian length (an MP4 sample).  `fps`
    only selects the SPS's level; frame i's idr_pic_id is (first_frame + i) & 1, so the batches of one
    video pass the index of their first frame.  Even h, w >= 2 within level 5.2 (36864 macroblocks, 543 per side); H264_MIN_QP <= qp <= 51."""
    N.require_cuda(frames)
    if frames.dim() != 4 or frames.shape[-1] != 3 or frames.dtype not in (torch.uint8, torch.float32):
        raise ValueError(f'encode_h264: frames must be uint8 or float32 [n, h, w, 3], got {frames.dtype} {tuple(frames.shape)}')
    if isinstance(qp, bool) or not isinstance(qp, (int, np.integer)) or not H264_MIN_QP <= int(qp) <= 51:
        raise ValueError(f'encode_h264: qp must be an int in [{H264_MIN_QP}, 51], got {qp!r}')
    fps = Fraction(fps).limit_denominator(1_000_000) if not isinstance(fps, Fraction) else fps
    if fps <= 0 or fps.numerator >= 1 << 32 or fps.denominator >= 1 << 32:
        raise ValueError(f'encode_h264: fps must be > 0, got {fps}')
    n, h, w, _ = frames.shape
    if n == 0:
        raise ValueError('encode_h264: no frames')
    L, dev, stream = N.lib(), frames.device, N.stream_ptr()
    ws_bytes, out_bytes = L.ssdnerf_h264_workspace_bytes(n, h, w), L.ssdnerf_h264_output_bound(n, h, w)
    if ws_bytes == 0:
        raise ValueError(f'encode_h264: unsupported size h={h} w={w} (even sizes >= 2 up to level 5.2: 36864 macroblocks, 543 per side)')
    frames = frames.contiguous()
    work = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
    offsets = torch.empty(n + 3, dtype=torch.int64, device=dev)
    fn = L.ssdnerf_h264_encode_u8 if frames.dtype == torch.uint8 else L.ssdnerf_h264_encode_f32
    N.check(fn(N.ptr(frames), n, h, w, int(qp), fps.numerator, fps.denominator, int(first_frame) & 1, N.ptr(work), ws_bytes, N.ptr(out), out_bytes,
               N.ptr(offsets), stream))
    off = offsets.cpu().tolist()
    data = out[:off[-1]].cpu().numpy().tobytes()
    return data[off[0]:off[1]], data[off[1]:off[2]], [data[off[i]:off[i + 1]] for i in range(2, n + 2)]


# ------------------------------------------------------------------------------------------------ MP4
def _box(kind, *payload):
    body = b''.join(payload)
    return struct.pack('>I', 8 + len(body)) + kind + body


def _full(kind, version, flags, *payload):
    return _box(kind, struct.pack('>I', version << 24 | flags), *payload)


def write_mp4(path, sps, pps, samples, width, height, fps):
    """an MP4 file of one H.264 video track: `samples` are access units with 4-byte NAL lengths (encode_h264), width x height, at
    `fps` frames per second (timescale and sample delta from Fraction(fps)).  Boxes: ftyp (isom, iso2, avc1, mp41), moov { mvhd,
    trak { tkhd, mdia { mdhd, hdlr vide, minf { vmhd, dinf { dref url }, stbl { stsd { avc1 { avcC } }, stts, stsc, stsz, stco } } } } },
    mdat; moov leads so a player can start before the whole file has arrived.  No stss: every sample is a sync sample.  Files over 4 GB
    (32-bit stco offsets) are refused."""
    samples = [bytes(s) for s in samples]
    sps, pps, width, height = bytes(sps), bytes(pps), int(width), int(height)
    if not samples:
        raise ValueError('write_mp4: no frames')
    if not (1 <= width <= 65535 and 1 <= height <= 65535):
        raise ValueError(f'write_mp4: width and height must be in [1, 65535], got {width} x {height}')
    if len(sps) < 4 or not pps:
        raise ValueError('write_mp4: an SPS of at least 4 bytes and a PPS are needed')
    fps = Fraction(fps).limit_denominator(1_000_000) if not isinstance(fps, Fraction) else fps
    if fps <= 0:
        raise ValueError(f'write_mp4: fps must be > 0, got {fps}')
    n = len(samples)
    timescale, delta = fps.numerator, fps.denominator
    duration = n * delta
    mdat_size = 8 + sum(len(s) for s in samples)
    ident = struct.pack('>9i', 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)
    avcc = _box(b'avcC', bytes([1, sps[1], sps[2], sps[3], 0xFF, 0xE1]), struct.pack('>H', len(sps)), sps, b'\x01',
                struct.pack('>H', len(pps)), pps)
    avc1 = _box(b'avc1', bytes(6), struct.pack('>H', 1), bytes(16), struct.pack('>HHIIIH', width, height, 0x480000, 0x480000, 0, 1),
                bytes(32), struct.pack('>Hh', 0x18, -1), avcc)

    def moov(mdat_start):
        stbl = _box(b'stbl', _full(b'stsd', 0, 0, struct.pack('>I', 1), avc1),
                    _full(b'stts', 0, 0, struct.pack('>III', 1, n, delta)),
                    _full(b'stsc', 0, 0, struct.pack('>IIII', 1, 1, n, 1)),
                    _full(b'stsz', 0, 0, struct.pack('>II', 0, n), b''.join(struct.pack('>I', len(s)) for s in samples)),
                    _full(b'stco', 0, 0, struct.pack('>II', 1, mdat_start + 8)))
        minf = _box(b'minf', _full(b'vmhd', 0, 1, bytes(8)),
                    _box(b'dinf', _full(b'dref', 0, 0, struct.pack('>I', 1), _full(b'url ', 0, 1))), stbl)
        mdia = _box(b'mdia', _full(b'mdhd', 0, 0, struct.pack('>IIIIHH', 0, 0, timescale, duration, 0x55C4, 0)),
                    _full(b'hdlr', 0, 0, bytes(4), b'vide', bytes(12), b'VideoHandler\0'), minf)
        tkhd = _full(b'tkhd', 0, 3, struct.pack('>IIIII', 0, 0, 1, 0, duration), bytes(8), struct.pack('>hhhH', 0, 0, 0, 0), ident,
                     struct.pack('>II', width << 16, height << 16))
        mvhd = _full(b'mvhd', 0, 0, struct.pack('>IIIIIH', 0, 0, timescale, duration, 0x10000, 0x100), bytes(10), ident, bytes(24),
                     struct.pack('>I', 2))
        return _box(b'moov', mvhd, _box(b'trak', tkhd, mdia))
    ftyp = _box(b'ftyp', b'isom', struct.pack('>I', 0x200), b'isomiso2avc1mp41')
    head = len(ftyp) + len(moov(0))
    total = head + mdat_size
    if total > MP4_MAX_BYTES - 1 or duration >= 1 << 32:
        raise ValueError(f'write_mp4: {total} bytes exceed the 4 GB limit of 32-bit MP4 offsets (stco); write fewer or smaller '
                         'frames per file')
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, 'wb') as f:
        f.write(ftyp + moov(head) + struct.pack('>I', mdat_size) + b'mdat')
        for s in samples:
            f.write(s)


# ------------------------------------------------------------------------------------------------ Motion-JPEG AVI
def _chunk(fourcc, payload):
    return fourcc + struct.pack('<I', len(payload)) + payload + (b'\0' if len(payload) & 1 else b'')


def _list(kind, payload):
    return b'LIST' + struct.pack('<I', len(payload) + 4) + kind + payload


def write_avi(path, jpegs, width, height, fps):
    """a Motion-JPEG AVI 1.0 file of the JPEG files `jpegs` (bytes, width x height each) at `fps` frames per second:
    RIFF AVI { LIST hdrl { avih, LIST strl { strh vids/MJPG, strf BITMAPINFOHEADER } }, LIST movi { 00dc ... }, idx1 }, every
    frame a key frame, each 00dc chunk padded to even length; idx1 offsets count from the `movi` fourcc.  Files over 1 GB are refused."""
    jpegs = [bytes(j) for j in jpegs]
    width, height = int(width), int(height)
    if not jpegs:
        raise ValueError('write_avi: no frames')
    if not (1 <= width <= 65535 and 1 <= height <= 65535):
        raise ValueError(f'write_avi: width and height must be in [1, 65535], got {width} x {height}')
    fps = Fraction(fps).limit_denominator(1_000_000) if not isinstance(fps, Fraction) else fps
    if fps <= 0:
        raise ValueError(f'write_avi: fps must be > 0, got {fps}')
    n = len(jpegs)
    movi_size = 4 + sum(8 + len(j) + (len(j) & 1) for j in jpegs)
    total = 12 + 200 + 8 + movi_size + 8 + 16 * n           # RIFF AVI, hdrl (12 + avih 64 + strl 12 + strh 64 + strf 48), movi, idx1
    if total > AVI_MAX_BYTES:
        raise ValueError(f'write_avi: {total} bytes exceed the 1 GB (2^30 bytes) limit of an AVI 1.0 RIFF file (no OpenDML); '
                         'write fewer or smaller frames per file')
    biggest = max(len(j) for j in jpegs)
    avih = struct.pack('<10I4I', int(round(1e6 / fps)), int(math.ceil(biggest * fps)), 0, AVIF_HASINDEX, n, 0, 1, biggest, width,
                       height, 0, 0, 0, 0)
    strh = b'vids' + b'MJPG' + struct.pack('<IHHIIIIIIiI4h', 0, 0, 0, 0, fps.denominator, fps.numerator, 0, n, biggest, -1, 0, 0, 0,
                                           width, height)
    strf = struct.pack('<IiiHH4sIiiII', 40, width, height, 1, 24, b'MJPG', width * height * 3, 0, 0, 0, 0)
    hdrl = _list(b'hdrl', _chunk(b'avih', avih) + _list(b'strl', _chunk(b'strh', strh) + _chunk(b'strf', strf)))
    index, movi, pos = [], [], 4
    for j in jpegs:
        index.append(struct.pack('<4sIII', b'00dc', AVIIF_KEYFRAME, pos, len(j)))
        movi.append(_chunk(b'00dc', j))
        pos += 8 + len(j) + (len(j) & 1)
    body = b'AVI ' + hdrl + _list(b'movi', b''.join(movi)) + _chunk(b'idx1', b''.join(index))
    assert 8 + len(body) == total
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, 'wb') as f:
        f.write(b'RIFF' + struct.pack('<I', len(body)) + body)


# ------------------------------------------------------------------------------------------------ camera path
def _unit(v):
    return v / torch.linalg.norm(v, dim=-1, keepdim=True)


def look_at(center, target, up):
    """camera-to-world rotations [..., 3, 3] with columns (right, -up, forward) of cameras at `center` looking at `target`:
    forward = unit(target - center), right = unit(forward x up), up' = unit(right x forward)"""
    fwd = _unit(target - center)
    right = _unit(torch.linalg.cross(fwd, up.expand_as(fwd)))
    cam_up = _unit(torch.linalg.cross(right, fwd))
    return torch.stack([right, -cam_up, fwd], dim=-1)


def surround_views(initial_pose, angle_amp=1.0, num_frames=60):
    """camera-to-world poses [num_frames, 4, 4] circling the origin at the distance of `initial_pose` [4, 4]: frame k turns the
    camera's azimuth by -2 pi k / num_frames and scales its elevation e0 to e0 (1 + angle_amp sin(2 pi k / num_frames)), looking at
    the origin with +z up (the reference's camera_utils.surround_views)"""
    initial_pose = torch.as_tensor(initial_pose, dtype=torch.float32)
    theta = torch.from_numpy(np.linspace(0, 2 * np.pi, num=num_frames, endpoint=False, dtype=np.float32))
    p0 = initial_pose[:3, 3]
    dist = torch.linalg.norm(p0)
    elev = torch.asin(p0[2] / dist) * (1 + angle_amp * torch.sin(theta))
    azim0 = p0[:2] / torch.linalg.norm(p0[:2])
    c, s = torch.cos(theta), torch.sin(theta)
    xy = torch.stack([azim0[0] * c + azim0[1] * s, azim0[1] * c - azim0[0] * s], dim=-1)       # azimuth turned by -theta
    pos = torch.cat([xy * torch.cos(elev)[:, None], torch.sin(elev)[:, None]], dim=-1) * dist
    rot = look_at(pos, torch.zeros_like(pos), pos.new_tensor([0.0, 0.0, 1.0]))
    poses = torch.zeros(num_frames, 4, 4)
    poses[:, :3, :3] = rot
    poses[:, :3, 3] = pos
    poses[:, 3, 3] = 1
    return poses


def gui_camera(camera_dir, camera_id=64):
    """the GUI's initial camera from a ShapeNet SRN style directory (`pose/*.txt`, `intrinsics.txt`): pose file `camera_id` of the
    sorted listing as cam_to_ndc = [R | 2 t] with the homogeneous row, fp32 [4, 4]; intrinsics fp32 [4] (fx, fy, cx, cy); (h, w)"""
    pose_dir = os.path.join(camera_dir, 'pose')
    names = sorted(os.listdir(pose_dir))
    if not 0 <= camera_id < len(names):
        raise ValueError(f'gui_camera: camera_id {camera_id} out of range: {pose_dir} holds {len(names)} poses')
    c2w = load_pose(os.path.join(pose_dir, names[camera_id]))
    pose = torch.eye(4)
    pose[:3, :3] = c2w[:3, :3]
    pose[:3, 3] = c2w[:3, 3] * 2
    fx, fy, cx, cy, h, w = load_intrinsics(os.path.join(camera_dir, 'intrinsics.txt'))
    return pose, torch.tensor([fx, fy, cx, cy], dtype=torch.float32), (h, w)
