"""ShapeNet SRN scenes without mmcv: the reference's `ShapeNetSRN` dataset (lib/datasets/shapenet_srn.py) and a collate that decodes
every view of a batch on the GPU.

`ShapeNetSRN.__getitem__` reads metadata and the views' file bytes only (no CUDA, so DataLoader workers may fork); `collate` stacks a
list of scenes like the runner's collate + scatter and decodes all their PNG files in one `decode_png` call.  `decode_png` checks the
chunk structure on the host and inflates, unfilters and converts on the device (csrc/png_decode.cu, header section 9); its values equal
`cv2.imread(path, cv2.IMREAD_COLOR)[..., ::-1].astype(np.float32) / 255` bit for bit.
"""
import ctypes
import os
import pickle
import random
import struct
import zlib

import numpy as np
import torch

from . import _lib as N
from .registry import DATASETS

PNG_SIGNATURE = b'\x89PNG\r\n\x1a\n'
_BPP = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# deflate emits at most 258 bytes per two code bits: no valid stream of s bytes inflates to more than this many bytes
_MAX_INFLATE_RATIO = 1032

STATUS_REASONS = {
    1: 'truncated zlib stream', 2: 'bad zlib header', 3: 'deflate block type 3', 4: 'stored block LEN != ~NLEN',
    5: 'bad Huffman code lengths', 6: 'invalid Huffman symbol', 7: 'match distance before the start of the data',
    8: 'more image data than IHDR allows', 9: 'less image data than IHDR requires', 10: 'row filter type above 4',
    11: 'Adler-32 mismatch', 12: 'bad descriptor',
}

_DESC = np.dtype([('stream_offset', '<u8'), ('palette_offset', '<u8'), ('work_offset', '<u8'), ('out_offset', '<u8'),
                  ('stream_bytes', '<u4'), ('h', '<u4'), ('w', '<u4'), ('color_type', '<i4')])


class PngInfo:
    """one file's IHDR fields, its PLTE (768 bytes, zero-padded) and its IDAT payloads"""
    __slots__ = ('name', 'w', 'h', 'color_type', 'palette', 'idat', 'stream_bytes')


def png_chunks(data, name):
    """Yields (type, body) for each chunk of a PNG file before IEND, with the checks every PNG reader here makes: the signature,
    chunks inside the file, every chunk's CRC, IHDR first, once and 13 bytes long, and an IEND chunk.  Raises ValueError naming the
    file."""
    mv = memoryview(data)
    if bytes(mv[:8]) != PNG_SIGNATURE:
        raise ValueError(f'{name}: not a PNG file (bad signature)')
    pos, seen_ihdr = 8, False
    while True:
        if pos + 12 > len(mv):
            raise ValueError(f'{name}: file ends before the IEND chunk')
        length, ctype = struct.unpack('>I4s', mv[pos:pos + 8])
        if length > len(mv) - pos - 12:
            raise ValueError(f'{name}: chunk {ctype!r} runs past the end of the file')
        body = mv[pos + 8:pos + 8 + length]
        crc, = struct.unpack('>I', mv[pos + 8 + length:pos + 12 + length])
        if zlib.crc32(body, zlib.crc32(ctype)) != crc:
            raise ValueError(f'{name}: bad CRC in chunk {ctype!r}')
        if not seen_ihdr and ctype != b'IHDR':
            raise ValueError(f'{name}: the first chunk is {ctype!r}, not IHDR')
        if ctype == b'IHDR':
            if seen_ihdr or length != 13:
                raise ValueError(f'{name}: bad IHDR chunk')
            seen_ihdr = True
        elif ctype == b'IEND':
            return
        yield ctype, body
        pos += 12 + length


def parse_png(data, name='<bytes>'):
    """Checks the file's chunks (png_chunks), parses IHDR / PLTE, gathers the IDAT payloads.  Raises ValueError naming the file
    for a malformed file and NotImplementedError for what the decoder does not cover: bit depths other than 8, Adam7 interlacing,
    and an eXIf chunk (cv2 would rotate the image by it)."""
    info = PngInfo()
    info.name, info.palette, info.idat = name, None, []
    for ctype, body in png_chunks(data, name):
        if ctype == b'IHDR':
            w, h, depth, ct, comp, filt, interlace = struct.unpack('>IIBBBBB', body)
            if w == 0 or h == 0 or w >= 2 ** 31 or h >= 2 ** 31:
                raise ValueError(f'{name}: IHDR size {w} x {h} is invalid')
            if ct not in _BPP:
                raise ValueError(f'{name}: IHDR colour type {ct} is invalid')
            if depth != 8:
                raise NotImplementedError(f'{name}: bit depth {depth} is not supported (8 bits only)')
            if interlace:
                raise NotImplementedError(f'{name}: Adam7 interlaced PNG files are not supported')
            if comp or filt:
                raise ValueError(f'{name}: unknown compression or filter method in IHDR')
            info.w, info.h, info.color_type = w, h, ct
        elif ctype == b'PLTE':
            if len(body) % 3 or not 3 <= len(body) <= 768:
                raise ValueError(f'{name}: bad PLTE chunk')
            info.palette = bytes(body) + bytes(768 - len(body))
        elif ctype == b'IDAT':
            info.idat.append(body)
        elif ctype == b'eXIf':
            raise NotImplementedError(f'{name}: eXIf chunk (cv2 would apply its orientation) is not supported')
    if not info.idat:
        raise ValueError(f'{name}: no IDAT chunk')
    if info.color_type == 3 and info.palette is None:
        raise ValueError(f'{name}: colour type 3 without a PLTE chunk')
    info.stream_bytes = sum(len(b) for b in info.idat)
    filtered = info.h * (1 + info.w * _BPP[info.color_type])
    if filtered >= 2 ** 31 or filtered > _MAX_INFLATE_RATIO * (info.stream_bytes + 1):
        raise ValueError(f'{name}: IHDR size {info.w} x {info.h} is more than its {info.stream_bytes}-byte zlib stream can hold')
    return info


def _status_error(name, code):
    return ValueError(f'{name}: corrupt PNG data ({STATUS_REASONS.get(code, f"status {code}")})')


def decode_png_host(data, name='<bytes>'):
    """One file decoded on the CPU by the same validation code as the device (ssdnerf_png_decode_host): returns (float32 [h, w, 3],
    status).  Status 0 is a good image; any other value is one of STATUS_REASONS and the array is undefined."""
    info = parse_png(data, name)
    stream = b''.join(bytes(b) for b in info.idat)
    out = np.empty((info.h, info.w, 3), np.float32)
    status = ctypes.c_int32(-1)
    N.check(N.lib().ssdnerf_png_decode_host(stream, len(stream), info.h, info.w, info.color_type, info.palette,
                                             out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(status)))
    return out, status.value


def _align(x, a):
    return (x + a - 1) // a * a


def _pack(infos):
    """parsed files -> (pinned uint8 host buffer: the streams, palettes and descriptors; descriptor offset; workspace bytes; float
    offsets of the images in the output)"""
    n = len(infos)
    ws = [N.lib().ssdnerf_png_decode_workspace_bytes(info.h, info.w, info.color_type) for info in infos]
    desc = np.zeros(n, _DESC)
    off = 0
    for i, info in enumerate(infos):
        desc[i]['stream_offset'], desc[i]['stream_bytes'] = off, info.stream_bytes
        off = _align(off + info.stream_bytes, 16)
        if info.color_type == 3:
            desc[i]['palette_offset'] = off
            off += 768
    desc_off = _align(off, 16)
    desc['h'] = [info.h for info in infos]
    desc['w'] = [info.w for info in infos]
    desc['color_type'] = [info.color_type for info in infos]
    desc['work_offset'] = np.concatenate([[0], np.cumsum(ws[:-1])]).astype(np.uint64)
    offsets = np.concatenate([[0], np.cumsum([info.h * info.w * 3 for info in infos])]).astype(np.int64)
    desc['out_offset'] = offsets[:-1].astype(np.uint64)

    host = torch.empty(desc_off + desc.nbytes, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for i, info in enumerate(infos):
        p = int(desc[i]['stream_offset'])
        for b in info.idat:
            hv[p:p + len(b)] = np.frombuffer(b, np.uint8)
            p += len(b)
        if info.color_type == 3:
            p = int(desc[i]['palette_offset'])
            hv[p:p + 768] = np.frombuffer(info.palette, np.uint8)
    hv[desc_off:] = desc.view(np.uint8)
    return host, desc_off, sum(ws), offsets


def _launch(dev, desc_off, work, out, status, device):
    N.require_cuda(dev, work, out, status)
    N.check(N.lib().ssdnerf_png_decode(N.ptr(dev), desc_off, ctypes.c_void_p(dev.data_ptr() + desc_off), status.numel(), N.ptr(work),
                                       work.numel(), N.ptr(out), out.numel(), N.ptr(status), N.stream_ptr(device)))


def _decode(infos, device):
    """parsed files (any sizes) -> (float32 buffer on `device` holding image i at floats [offsets[i], offsets[i + 1]), offsets,
    statuses); one pinned host buffer, one host-to-device copy, one launch, one read of the statuses"""
    n = len(infos)
    work_total = sum(N.lib().ssdnerf_png_decode_workspace_bytes(info.h, info.w, info.color_type) for info in infos)
    out_floats = sum(info.h * info.w * 3 for info in infos)
    need = work_total + 4 * out_floats
    with torch.cuda.device(device):
        free, _ = torch.cuda.mem_get_info()
    if need > free:
        raise ValueError(f'decode_png: {n} images need {need / 2 ** 30:.2f} GiB of device memory, {free / 2 ** 30:.2f} GiB are free')
    host, desc_off, work_total, offsets = _pack(infos)
    with torch.cuda.device(device):
        dev = host.to(device, non_blocking=True)
        work = torch.empty(work_total, dtype=torch.uint8, device=device)
        out = torch.empty(out_floats, dtype=torch.float32, device=device)
        status = torch.empty(n, dtype=torch.int32, device=device)
        _launch(dev, desc_off, work, out, status, device)
        st = status.cpu().numpy()
    return out, offsets, st


def _device(device):
    return torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)


def decode_png_images(files, device=None, names=None):
    """PNG files of any sizes -> a list of float32 [h, w, 3] tensors on `device`, decoded in one launch (see `decode_png`)"""
    names = [f'file {i}' for i in range(len(files))] if names is None else list(names)
    infos = [parse_png(f, nm) for f, nm in zip(files, names)]
    if not infos:
        return []
    out, offsets, st = _decode(infos, _device(device))
    bad = np.flatnonzero(st)
    if bad.size:
        raise _status_error(names[bad[0]], int(st[bad[0]]))
    return [out[offsets[i]:offsets[i + 1]].view(info.h, info.w, 3) for i, info in enumerate(infos)]


def decode_png(files, device=None, names=None):
    """PNG files (a list of bytes) -> float32 [n, h, w, 3] RGB in [0, 1] on `device`, equal to cv2.imread(IMREAD_COLOR) BGR -> RGB
    / 255.  All files must have one size.  Every file is parsed and checked on the host before anything is allocated or launched;
    a decode error raises ValueError naming the first bad file."""
    names = [f'file {i}' for i in range(len(files))] if names is None else list(names)
    if not files:
        raise ValueError('decode_png: no files')
    infos = [parse_png(f, nm) for f, nm in zip(files, names)]
    h, w = infos[0].h, infos[0].w
    for info in infos[1:]:
        if (info.h, info.w) != (h, w):
            raise ValueError(f'{info.name}: size {info.w} x {info.h} differs from {infos[0].name}\'s {w} x {h} '
                             '(images of one batch are stacked)')
    out, _, st = _decode(infos, _device(device))
    bad = np.flatnonzero(st)
    if bad.size:
        raise _status_error(names[bad[0]], int(st[bad[0]]))
    return out.view(len(infos), h, w, 3)


# ------------------------------------------------------------------------------------------------ ShapeNet SRN scenes
def load_intrinsics(path):
    """SRN intrinsics.txt: `f cx cy _`, the grid barycenter, the scale, `height width` -> (fx, fy, cx, cy, height, width)"""
    with open(path) as f:
        f0, cx, cy, _ = (float(x) for x in f.readline().split())
        f.readline()
        f.readline()
        height, width = (int(x) for x in f.readline().split())
    return f0, f0, cx, cy, height, width


def load_pose(path):
    return torch.from_numpy(np.loadtxt(path, dtype=np.float32, delimiter=' ').reshape(4, 4))


def _normalise_pose(c2w, center, radius):
    """camera-to-world [4, 4] -> rotation and (t - center) / radius, with the homogeneous row"""
    c2w = torch.as_tensor(c2w, dtype=torch.float32)
    top = torch.cat([c2w[:3, :3], (c2w[:3, 3:] - center[:, None]) / radius[:, None]], dim=-1)
    return torch.cat([top, top.new_tensor([[0.0, 0.0, 0.0, 1.0]])], dim=-2)


@DATASETS.register_module()
class ShapeNetSRN(torch.utils.data.Dataset):
    """The reference's ShapeNetSRN: same arguments and `parse_scene` keys.  `cond_imgs` / `test_imgs` are lists of the files' bytes
    (decoded by `collate`); the DataContainer values of the reference are plain values here."""

    def __init__(self, data_prefix, code_dir=None, code_only=False, load_imgs=True, specific_observation_idcs=None, num_test_imgs=0,
                 random_test_imgs=False, scene_id_as_name=False, cache_path=None, test_pose_override=None, num_train_imgs=-1,
                 load_cond_data=True, load_test_data=True, max_num_scenes=-1, radius=0.5, test_mode=False, step=1):
        super().__init__()
        self.data_prefix, self.code_dir, self.code_only, self.load_imgs = data_prefix, code_dir, code_only, load_imgs
        self.specific_observation_idcs, self.num_test_imgs, self.random_test_imgs = specific_observation_idcs, num_test_imgs, random_test_imgs
        self.scene_id_as_name, self.cache_path, self.test_pose_override = scene_id_as_name, cache_path, test_pose_override
        self.num_train_imgs, self.load_cond_data, self.load_test_data = num_train_imgs, load_cond_data, load_test_data
        self.max_num_scenes, self.step = max_num_scenes, step
        self.radius = torch.tensor([radius], dtype=torch.float32).expand(3)
        self.center = torch.zeros_like(self.radius)
        self.load_scenes()
        if test_pose_override is not None:
            pose_dir = os.path.join(test_pose_override, 'pose')
            self.test_poses = torch.stack([_normalise_pose(load_pose(os.path.join(pose_dir, p)), self.center, self.radius)
                                           for p in sorted(os.listdir(pose_dir))])
            fx, fy, cx, cy, _, _ = load_intrinsics(os.path.join(test_pose_override, 'intrinsics.txt'))
            self.test_intrinsics = torch.tensor([fx, fy, cx, cy], dtype=torch.float32)[None].expand(self.test_poses.size(0), -1)
        else:
            self.test_poses = self.test_intrinsics = None

    def _scan(self):
        prefixes = self.data_prefix if isinstance(self.data_prefix, list) else [self.data_prefix]
        scenes = []
        for prefix in prefixes:
            for name in os.listdir(prefix):
                scene_dir = os.path.join(prefix, name)
                if not os.path.isdir(scene_dir):
                    continue
                image_dir = os.path.join(scene_dir, 'rgb')
                image_names = sorted(os.listdir(image_dir))
                scenes.append(dict(
                    intrinsics=load_intrinsics(os.path.join(scene_dir, 'intrinsics.txt')),
                    image_paths=[os.path.join(image_dir, n) for n in image_names],
                    poses=[load_pose(os.path.join(scene_dir, 'pose', os.path.splitext(n)[0] + '.txt')) for n in image_names]))
        # by scene folder name (a stable sort, as the reference's)
        return sorted(scenes, key=lambda s: s['image_paths'][0].split('/')[-3])

    def load_scenes(self):
        if self.cache_path is not None and os.path.exists(self.cache_path):
            with open(self.cache_path, 'rb') as f:
                scenes = pickle.load(f)
        else:
            scenes = self._scan()
            if self.cache_path is not None:
                with open(self.cache_path, 'wb') as f:
                    pickle.dump(scenes, f, protocol=2)
        end = len(scenes)
        if self.max_num_scenes >= 0:
            end = min(end, self.max_num_scenes * self.step)
        self.scenes = scenes[:end:self.step]
        self.num_scenes = len(self.scenes)

    def _gather(self, scene, ids):
        poses = torch.stack([_normalise_pose(scene['poses'][i], self.center, self.radius) for i in ids])
        fx, fy, cx, cy, _, _ = scene['intrinsics']
        intrinsics = torch.tensor([fx, fy, cx, cy], dtype=torch.float32)[None].expand(len(ids), -1)
        paths = [scene['image_paths'][i] for i in ids]
        imgs = None
        if self.load_imgs:
            imgs = []
            for p in paths:
                with open(p, 'rb') as f:
                    imgs.append(f.read())
        return imgs, poses, intrinsics, paths

    def parse_scene(self, scene_id):
        scene = self.scenes[scene_id]
        paths = scene['image_paths']
        scene_name = paths[0].split('/')[-3]
        results = dict(scene_id=scene_id, scene_name='{:04d}'.format(scene_id) if self.scene_id_as_name else scene_name)
        if not self.code_only:
            num_imgs = len(paths)
            if self.specific_observation_idcs is None:
                num_train = self.num_train_imgs if self.num_train_imgs >= 0 else num_imgs - self.num_test_imgs
                if self.random_test_imgs:
                    cond_ids = random.sample(range(num_imgs), num_train)
                else:
                    cond_ids = np.round(np.linspace(0, num_imgs - 1, num_train)).astype(np.int64)
            else:
                cond_ids = self.specific_observation_idcs
            test_ids = list(range(num_imgs))
            for i in cond_ids:
                test_ids.remove(i)
            for prefix, ids, load in (('cond', cond_ids, self.load_cond_data), ('test', test_ids, self.load_test_data)):
                if load and len(ids) > 0:
                    imgs, poses, intrinsics, img_paths = self._gather(scene, ids)
                    results[f'{prefix}_poses'], results[f'{prefix}_intrinsics'] = poses, intrinsics
                    results[f'{prefix}_img_paths'] = img_paths
                    if imgs is not None:
                        results[f'{prefix}_imgs'] = imgs
        if self.code_dir is not None:
            code_file = os.path.join(self.code_dir, scene_name + '.pth')
            if os.path.exists(code_file):
                results['code'] = torch.load(code_file, map_location='cpu')
        if self.test_pose_override is not None:
            results.update(test_poses=self.test_poses, test_intrinsics=self.test_intrinsics)
        return results

    def __len__(self):
        return self.num_scenes

    def __getitem__(self, scene_id):
        return self.parse_scene(scene_id)


_LIST_KEYS = ('scene_id', 'scene_name', 'cond_img_paths', 'test_img_paths', 'code')
_IMG_KEYS = ('cond_imgs', 'test_imgs')


def collate(scenes, device=None):
    """A list of `ShapeNetSRN` items -> the batch `train_step` / `val_step` take: poses and intrinsics stacked on `device`; ids, names,
    paths and codes kept as lists; every view of every scene decoded in one `decode_png` call into float32 [B, n, h, w, 3]."""
    device = _device(device)
    batch = {}
    files, names, spans = [], [], []
    for key in scenes[0]:
        vals = [s[key] for s in scenes]
        if key in _LIST_KEYS:
            batch[key] = vals
        elif key in _IMG_KEYS:
            counts = {len(v) for v in vals}
            if len(counts) != 1:
                raise ValueError(f'collate: scenes have different numbers of {key} ({sorted(counts)}) and cannot be stacked')
            paths = [s.get(key[:-1] + '_paths') or [f'{s["scene_name"]} {key}[{j}]' for j in range(len(v))] for s, v in zip(scenes, vals)]
            spans.append((key, len(files), len(scenes), len(vals[0])))
            for v, p in zip(vals, paths):
                files.extend(v)
                names.extend(p)
        else:
            batch[key] = torch.stack([torch.as_tensor(v) for v in vals]).to(device)
    if files:
        imgs = decode_png(files, device, names)
        for key, start, b, n in spans:
            batch[key] = imgs[start:start + b * n].reshape(b, n, *imgs.shape[1:])
    return batch
