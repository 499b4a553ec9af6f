"""Orbit videos of scenes: the camera path and file writing of the reference GUI's "Export video" (lib/core/ssdnerf_gui.py,
lib/core/utils/camera_utils.py), without a window or ffmpeg.

Frames are encoded on the device as baseline JPEG (csrc/jpeg.cu, byte-identical to cv2.imencode with libjpeg-turbo's defaults); only
the compressed files are copied to the host, once per call, and written into a Motion-JPEG AVI that ffmpeg, VLC and mpv play."""
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
