"""KITTI single-view reconstruction data without mmcv: the reference's tools/kitti_preproc.py, which cuts every fully visible
instance of KITTI's object training set out of its frame into the ShapeNet SRN layout `configs/supp_cfgs/ssdnerf_cars_reconskitti.py`
reads (`data/shapenet/cars_kitti`).

Labels, calibration, poses, `pad_tgt`, `scale` and the intrinsics text are computed on the host in numpy with the reference's
float32 / float64 mixing.  The pixel work runs on the device, a batch of frames at a time (csrc/kitti.cu, csrc/png_decode.cu,
csrc/png.cu, header section 10): one raw PNG decode of the frames and instance maps, one box pass, one crop / resize launch and one
PNG encode.  Decoded outputs equal the reference's bit for bit; the PNG bytes are this encoder's own.

    python -m ssdnerf_b200.kitti_preproc --kitti-dir data/kitti/training --out-dir data/shapenet/cars_kitti
"""
import argparse
import ctypes
import os
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib as N
from .datasets import STATUS_REASONS, png_chunks

_RAW_DESC = np.dtype([('stream_offset', '<u8'), ('work_offset', '<u8'), ('out_offset', '<u8'), ('stream_bytes', '<u4'), ('h', '<u4'),
                      ('w', '<u4'), ('color_type', '<i4'), ('bit_depth', '<i4'), ('reserved', '<u4')])
_FRAME = np.dtype([('seg_offset', '<u8'), ('h', '<u4'), ('w', '<u4'), ('box_offset', '<u4'), ('num_labels', '<u4')])
_CROP = np.dtype([('image_offset', '<u8'), ('seg_offset', '<u8'), ('crop_offset', '<u8'), ('view_offset', '<u8'), ('frame_w', '<u4'),
                  ('y0', '<u4'), ('x0', '<u4'), ('h', '<u4'), ('w', '<u4'), ('label', '<u4'), ('pad_tgt', '<u4'), ('pad_y', '<u4'),
                  ('pad_x', '<u4'), ('prior_first', '<u4'), ('prior_count', '<u4'), ('_pad', '<u4')])
_BGR_DESC = np.dtype([('src_offset', '<u8'), ('h', '<u4'), ('w', '<u4'), ('filt_offset', '<u8'), ('seg_first', '<u4'), ('reserved', '<u4')])
MAX_LABELS = 1024

# camera axes of the reference's c2w: x -> -z, y -> x, z -> -y
_ROT_CONVERSION = np.array([[0, 1, 0], [0, 0, -1], [-1, 0, 0]], dtype=np.float32)


# ------------------------------------------------------------------------------------------------ host parsing and geometry
def parse_labels(text, name):
    """label_2 lines -> [type, truncated, occluded, alpha, bbox(4), dims(3), location(3), rotation_y] as the reference parses them:
    field 2 int(float(.)), field 0 a string, the rest floats"""
    rows = []
    try:
        for line in text.splitlines(True):
            vals = line.strip().split(' ')
            rows.append([float(v) if i not in (0, 2) else int(float(v)) if i == 2 else v for i, v in enumerate(vals)])
            if len(rows[-1]) < 15:
                raise ValueError(f'{len(rows[-1])} fields')
    except ValueError as e:
        raise ValueError(f'{name}: malformed label line {len(rows)} ({e})') from None
    return rows


def parse_calib(text, name, cam=2):
    """camera `cam`'s 3 x 4 projection matrix, float32"""
    try:
        line = text.splitlines(True)[cam]
        return np.array([float(v) for v in line.strip().split(' ')[1:]], dtype=np.float32).reshape((3, 4))
    except (IndexError, ValueError) as e:
        raise ValueError(f'{name}: malformed calibration (camera {cam}: {e})') from None


def camera_offset(proj):
    """K^-1 t of the projection [K | t], float32 as scipy's solve_triangular returns it"""
    from scipy.linalg import solve_triangular
    return solve_triangular(proj[:, :3], proj[:, 3:], lower=False).squeeze(-1)


def yaw_rotation(yaw):
    s, c = np.sin(yaw), np.cos(yaw)
    r = np.zeros(np.shape(yaw) + (3, 3), dtype=np.float32)
    r[..., 0, 0] = c
    r[..., 2, 2] = c
    r[..., 0, 2] = s
    r[..., 2, 0] = -s
    r[..., 1, 1] = 1
    return r


def instance_geometry(label, cam_t, proj, y_min, y_max, x_min, x_max, out_size=128, out_border=4):
    """one instance's c2w [4, 4], pad_tgt, scale, pad offsets (x, y) and intrinsics.txt text.  The box bounds are numpy integers, as
    the reference's nonzero() gives them, so every float32 / float64 promotion is the reference's."""
    K = proj[:, :3]
    resize_tgt = out_size - out_border * 2
    h, w = y_max - y_min, x_max - x_min
    box = np.array(label[8:], dtype=np.float32)
    box[[0, 1, 2]] = box[[2, 0, 1]]                           # h w l -> l h w
    diag = np.linalg.norm(box[:3])
    box[3:6] += cam_t
    box[4] -= box[1] / 2
    box[:6] /= diag
    rot = yaw_rotation(box[6]) @ _ROT_CONVERSION
    c2w = np.concatenate([rot.T, rot.T @ (-box[3:6])[:, None]], axis=1)
    c2w = np.concatenate([c2w, [[0, 0, 0, 1]]], axis=0)
    pad_tgt = max(round(np.linalg.norm(box[:3]) * K[0, 0] / box[5]), max(h, w))
    scale = resize_tgt / pad_tgt
    pad_x = (pad_tgt - w) // 2
    pad_y = (pad_tgt - h) // 2
    text = '{:.6f} {:.6f} {:.6f} 0.\n0. 0. 0.\n1.\n{} {}\n'.format(
        K[0, 0] * scale, (K[0, 2] - x_min + pad_x) * scale + out_border, (K[1, 2] - y_min + pad_y) * scale + out_border, out_size, out_size)
    return c2w, int(pad_tgt), scale, int(pad_x), int(pad_y), text


def pose_text(c2w):
    """np.savetxt of the flattened c2w, as a string"""
    import io
    f = io.BytesIO()
    np.savetxt(f, c2w.reshape(1, -1))
    return f.getvalue().decode()


# ------------------------------------------------------------------------------------------------ PNG chunks (8 and 16 bits)
def parse_png_raw(data, name):
    """(h, w, colour type, bit depth, zlib stream) of a non-interlaced PNG; ValueError naming the file when malformed"""
    ihdr, idat = None, []
    for ctype, body in png_chunks(data, name):
        if ctype == b'IHDR':
            ihdr = struct.unpack('>IIBBBBB', body)
        elif ctype == b'IDAT':
            idat.append(bytes(body))
    w, h, depth, ct, comp, filt, interlace = ihdr
    if not idat or comp or filt or interlace or w == 0 or h == 0:
        raise ValueError(f'{name}: unsupported or malformed PNG header / data')
    return h, w, ct, depth, b''.join(idat)


def decode_png_raw_host(data, name='<bytes>'):
    """one file decoded on the CPU like cv2.imread(IMREAD_UNCHANGED) (8-bit grey / BGR, 16-bit grey): (array, status)"""
    h, w, ct, depth, stream = parse_png_raw(data, name)
    ch, dt = {(0, 8): (1, np.uint8), (2, 8): (3, np.uint8), (0, 16): (1, np.uint16)}.get((ct, depth), (0, None))
    if not ch:
        raise ValueError(f'{name}: colour type {ct} at {depth} bits is not supported')
    out = np.empty((h, w, ch) if ch == 3 else (h, w), dt)
    status = ctypes.c_int32(-1)
    N.check(N.lib().ssdnerf_png_decode_raw_host(stream, len(stream), h, w, ct, depth, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(status)))
    return out, status.value


def resize_host(img, dh, dw):
    """cv2.resize(img, (dw, dh), interpolation=INTER_LINEAR) of a u8 [h, w, 3] image by the views' own arithmetic (CPU)"""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    out = np.empty((dh, dw, 3), np.uint8)
    N.check(N.lib().ssdnerf_kitti_resize_host(img.ctypes.data_as(ctypes.c_void_p), img.shape[0], img.shape[1], dh, dw,
                                              out.ctypes.data_as(ctypes.c_void_p)))
    return out


def _align(x, a):
    return (x + a - 1) // a * a


def decode_png_raw(files, names, device):
    """files (bytes) -> list of cuda u8 tensors: [h, w, 3] BGR for 8-bit RGB, int16-viewed uint16 [h, w] for 16-bit grey,
    decoded in one launch; ValueError naming the first bad file"""
    parsed = [parse_png_raw(f, nm) for f, nm in zip(files, names)]
    bpp = {(0, 8): 1, (2, 8): 3, (0, 16): 2}
    desc = np.zeros(len(files), _RAW_DESC)
    off = work = out = 0
    for i, ((h, w, ct, depth, stream), nm) in enumerate(zip(parsed, names)):
        if (ct, depth) not in bpp:
            raise ValueError(f'{nm}: colour type {ct} at {depth} bits is not supported (8-bit grey / RGB or 16-bit grey)')
        desc[i] = (off, work, out, len(stream), h, w, ct, depth, 0)
        off = _align(off + len(stream), 16)
        work += N.lib().ssdnerf_png_decode_raw_workspace_bytes(h, w, ct, depth)
        out = _align(out + h * w * bpp[(ct, depth)], 16)
    desc_off = _align(off, 16)
    host = torch.empty(desc_off + desc.nbytes, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for i, p in enumerate(parsed):
        o = int(desc[i]['stream_offset'])
        hv[o:o + len(p[4])] = np.frombuffer(p[4], np.uint8)
    hv[desc_off:] = desc.view(np.uint8)
    dev = host.to(device, non_blocking=True)
    ws = torch.empty(max(work, 1), dtype=torch.uint8, device=device)
    buf = torch.empty(max(out, 1), dtype=torch.uint8, device=device)
    status = torch.empty(len(files), dtype=torch.int32, device=device)
    N.check(N.lib().ssdnerf_png_decode_raw(N.ptr(dev), desc_off, ctypes.c_void_p(dev.data_ptr() + desc_off), len(files), N.ptr(ws),
                                           ws.numel(), N.ptr(buf), buf.numel(), N.ptr(status), N.stream_ptr(device)))
    st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if bad.size:
        k = int(st[bad[0]])
        raise ValueError(f'{names[bad[0]]}: corrupt PNG data ({STATUS_REASONS.get(k, f"status {k}")})')
    return buf, desc


def encode_bgr(images, shapes, offsets, device):
    """BGR u8 images in one device buffer (image i at byte offsets[i], shape shapes[i] = (h, w)) -> list of PNG files (bytes)"""
    n = len(shapes)
    if n == 0:
        return []
    desc = np.zeros(n, _BGR_DESC)
    desc['src_offset'] = offsets
    desc['h'] = [s[0] for s in shapes]
    desc['w'] = [s[1] for s in shapes]
    ws_bytes, out_bytes = ctypes.c_size_t(), ctypes.c_size_t()
    L = N.lib()
    N.check(L.ssdnerf_png_bgr_layout(desc.ctypes.data_as(ctypes.c_void_p), n, ctypes.byref(ws_bytes), ctypes.byref(out_bytes)))
    d_desc = torch.from_numpy(desc.view(np.uint8).copy()).to(device)
    work = torch.empty(ws_bytes.value, dtype=torch.uint8, device=device)
    out = torch.empty(out_bytes.value, dtype=torch.uint8, device=device)
    off = torch.empty(n + 1, dtype=torch.int64, device=device)
    N.check(L.ssdnerf_png_encode_bgr(N.ptr(images), N.ptr(d_desc), desc.ctypes.data_as(ctypes.c_void_p), n, N.ptr(work), ws_bytes.value,
                                     N.ptr(out), out_bytes.value, N.ptr(off), N.stream_ptr(device)))
    o = off.cpu().tolist()
    data = out[:o[-1]].cpu().numpy().tobytes()
    return [data[o[i]:o[i + 1]] for i in range(n)]


# ------------------------------------------------------------------------------------------------ the tool
def _read(path):
    with open(path, 'rb') as f:
        return f.read()


def _frame_inputs(kitti_dir, stem):
    paths = (os.path.join(kitti_dir, 'label_2', stem + '.txt'), os.path.join(kitti_dir, 'calib', stem + '.txt'),
             os.path.join(kitti_dir, 'image_2', stem + '.png'), os.path.join(kitti_dir, 'instance_2', stem + '.png'))
    return paths, [_read(p) for p in paths]


def process_batch(frames, out_dir, out_size, out_border, device, pool=None):
    """frames: list of (stem, paths, (label bytes, calib bytes, image png, instance png)) -> the reference's files under out_dir.
    Returns the number of instances written."""
    resize_tgt = out_size - 2 * out_border
    metas = []
    for stem, paths, (lab, cal, _, _) in frames:
        labels = parse_labels(lab.decode(), paths[0])
        if len(labels) > MAX_LABELS:
            raise ValueError(f'{paths[0]}: {len(labels)} label lines, at most {MAX_LABELS} are supported')
        proj = parse_calib(cal.decode(), paths[1])
        metas.append((labels, proj, camera_offset(proj)))
    files = [f for _, _, d in frames for f in d[2:]]
    names = [p for _, paths, _ in frames for p in paths[2:]]
    buf, desc = decode_png_raw(files, names, device)
    fr = np.zeros(len(frames), _FRAME)
    nbox = 0
    for k, (stem, paths, _) in enumerate(frames):
        im, sg = desc[2 * k], desc[2 * k + 1]
        if im['color_type'] != 2 or im['bit_depth'] != 8:
            raise ValueError(f'{paths[2]}: the frame must be an 8-bit RGB PNG')
        if sg['color_type'] != 0 or sg['bit_depth'] != 16:
            raise ValueError(f'{paths[3]}: the instance map must be a 16-bit grey PNG')
        if (im['h'], im['w']) != (sg['h'], sg['w']):
            raise ValueError(f'{paths[3]}: size {sg["w"]} x {sg["h"]} differs from the frame\'s {im["w"]} x {im["h"]}')
        fr[k] = (sg['out_offset'] // 2, sg['h'], sg['w'], nbox, len(metas[k][0]))
        nbox += len(metas[k][0])
    seg16 = buf.view(torch.int16) if buf.numel() % 2 == 0 else buf[:-1].view(torch.int16)
    boxes = torch.empty(max(nbox, 1) * 5, dtype=torch.int32, device=device)
    d_fr = torch.from_numpy(fr.view(np.uint8).copy()).to(device)
    N.check(N.lib().ssdnerf_kitti_boxes(N.ptr(seg16), N.ptr(d_fr), len(frames), N.ptr(boxes), nbox, N.stream_ptr(device)))
    bx = boxes.cpu().numpy().reshape(-1, 5)

    jobs, priors, outs = [], [], []
    crop_off = 0
    for k, (stem, paths, _) in enumerate(frames):
        labels, proj, cam_t = metas[k]
        whitening = []                                        # earlier instances of this frame that whitened it
        for i, lab in enumerate(labels):
            if not (lab[1] == 0 and lab[2] == 0):
                continue
            cnt, y0, y1, x0, x1 = (np.int64(v) for v in bx[int(fr[k]['box_offset']) + i])
            if cnt == 0:
                continue
            c2w, pad_tgt, scale, pad_x, pad_y, intr = instance_geometry(lab, cam_t, proj, y0, y1, x0, x1, out_size, out_border)
            first = len(priors)
            priors.extend(whitening)
            whitening.append((int(y0), int(y1), int(x0), int(x1), 1000 + i))
            if scale > 1:
                continue
            h, w = int(y1 - y0), int(x1 - x0)
            jobs.append((int(desc[2 * k]['out_offset']), int(fr[k]['seg_offset']), crop_off, 0, int(fr[k]['w']), int(y0), int(x0), h, w,
                         1000 + i, pad_tgt, pad_y, pad_x, first, len(priors) - first, 0))
            outs.append((stem + '_{:03d}'.format(i), c2w, intr, (h, w), crop_off))
            crop_off = _align(crop_off + 3 * h * w, 16)
    if not jobs:
        return 0
    nj = len(jobs)
    view_bytes = 3 * out_size * out_size
    job = np.array(jobs, dtype=_CROP)
    job['view_offset'] = crop_off + view_bytes * np.arange(nj, dtype=np.uint64)
    pr = np.array(priors if priors else [(0, 0, 0, 0, 0)], dtype=np.int32)
    d_job = torch.from_numpy(job.view(np.uint8).copy()).to(device)
    d_pr = torch.from_numpy(pr).to(device)
    pix = torch.empty(crop_off + view_bytes * nj, dtype=torch.uint8, device=device)
    N.check(N.lib().ssdnerf_kitti_crops(N.ptr(buf), N.ptr(seg16), N.ptr(d_job), nj, N.ptr(d_pr), out_size, out_border, N.ptr(pix),
                                        N.ptr(pix), N.stream_ptr(device)))
    shapes = [(out_size, out_size)] * nj + [o[3] for o in outs]
    offs = [int(v) for v in job['view_offset']] + [o[4] for o in outs]
    pngs = encode_bgr(pix, shapes, offs, device)

    def write(j):
        name, c2w, intr, _, _ = outs[j]
        inst = os.path.join(out_dir, name)
        os.makedirs(os.path.join(inst, 'rgb'), exist_ok=True)
        os.makedirs(os.path.join(inst, 'pose'), exist_ok=True)
        with open(os.path.join(inst, 'rgb', '000000.png'), 'wb') as f:
            f.write(pngs[j])
        with open(os.path.join(inst, '000000.png'), 'wb') as f:
            f.write(pngs[nj + j])
        with open(os.path.join(inst, 'pose', '000000.txt'), 'w') as f:
            f.write(pose_text(c2w))
        with open(os.path.join(inst, 'intrinsics.txt'), 'w') as f:
            f.write(intr)
    list(pool.map(write, range(nj))) if pool is not None else [write(j) for j in range(nj)]
    return nj


def preprocess(kitti_dir='data/kitti/training', out_dir='data/shapenet/cars_kitti', out_size=128, out_border=4, device=None,
               batch_frames=16, threads=8):
    """the reference's kitti_preproc main(): every label_2/*.txt in name order; returns the number of instances written"""
    if out_size <= 2 * out_border:
        raise ValueError(f'out_size {out_size} must exceed 2 * out_border {out_border}')
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    os.makedirs(out_dir, exist_ok=True)
    stems = [os.path.splitext(f)[0] for f in sorted(os.listdir(os.path.join(kitti_dir, 'label_2')))]
    total = 0
    with ThreadPoolExecutor(threads) as pool, torch.cuda.device(device):
        for b in range(0, len(stems), batch_frames):
            chunk = stems[b:b + batch_frames]
            got = list(pool.map(lambda s: _frame_inputs(kitti_dir, s), chunk))
            frames = [(s, paths, data) for s, (paths, data) in zip(chunk, got)]
            total += process_batch(frames, out_dir, out_size, out_border, device, pool)
    return total


def main(argv=None):
    p = argparse.ArgumentParser(description='Preprocess the KITTI dataset on the GPU (the reference\'s tools/kitti_preproc.py)')
    p.add_argument('--kitti-dir', default='data/kitti/training')
    p.add_argument('--out-dir', default='data/shapenet/cars_kitti')
    p.add_argument('--out-size', type=int, default=128)
    p.add_argument('--out-border', type=int, default=4)
    a = p.parse_args(argv)
    n = preprocess(a.kitti_dir, a.out_dir, a.out_size, a.out_border)
    print(f'{n} instances written to {a.out_dir}')
