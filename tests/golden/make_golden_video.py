"""Pins for the orbit-video path (csrc/jpeg.cu, ssdnerf_b200/video.py):
  * a JPEG corpus: RGB u8 images and the files `cv2.imencode('.jpg', bgr, [IMWRITE_JPEG_QUALITY, q])` writes for them (libjpeg-turbo):
    sizes 1x1 .. 255x257, flat, noise, render-like gradients, blocks that force ZRL runs and DC differences of category 11, noise whose
    entropy-coded data holds 0xFF bytes; qualities 1, 25, 50, 75, 95, 100;
  * the camera path: the reference's own surround_views / look_at (lib/core/utils/camera_utils.py, executed from the checkout) from
    demo/camera_spiral_cars pose 64 after the GUI's cam_to_ndc, for (num_frames, angle_amp) = (120, 1.0), (7, 1.0), (60, 0.5); the
    pose file and intrinsics.txt are stored as text.

    python tests/golden/make_golden_video.py [REFERENCE_ROOT]          (needs cv2 and the reference checkout)
-> tests/golden/reference_video_v1.npz, replayed by tests/test_orbit_cpu.py and tests/test_orbit_gpu.py.
"""
import importlib.util
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(1, 1), (8, 8), (7, 9), (16, 15), (17, 33), (128, 128), (256, 256), (255, 257)]
QUALITIES = [1, 25, 50, 75, 95, 100]
CAMERA_ID = 64
PATHS = [(120, 1.0), (7, 1.0), (60, 0.5)]


def gradient(h, w, rng):
    """a render-like frame: a shaded ellipse over white, smooth edges"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    cy, cx = (h - 1) * rng.uniform(0.4, 0.6), (w - 1) * rng.uniform(0.4, 0.6)
    d = ((y - cy) / (0.35 * h + 0.5)) ** 2 + ((x - cx) / (0.3 * w + 0.5)) ** 2
    base = rng.uniform(40, 220, 3)
    shade = (1 - 0.5 * d)[..., None] * base + 12 * np.sin(x / 7 + y / 11)[..., None]
    a = np.clip(1.5 - d, 0, 1)[..., None]
    return np.clip(np.rint(a * shade + (1 - a) * 255), 0, 255).astype(np.uint8)


def zrl_dc11(h, w):
    """8 x 8 blocks alternating black and white (DC differences of 2040: category 11 at quality 100) with a (0, 1) and a (7, 7)
    cosine on mid-grey blocks (one low and one last zigzag coefficient: a run of zeros longer than 16 between them)"""
    r, c = np.mgrid[0:8, 0:8]
    wave = 128 + 40 * np.cos((2 * c + 1) * np.pi / 16) + 40 * np.cos((2 * r + 1) * 7 * np.pi / 16) * np.cos((2 * c + 1) * 7 * np.pi / 16)
    wave = np.clip(np.rint(wave), 0, 255)
    by, bx = np.mgrid[0:h, 0:w] // 8
    kind = (by * 3 + bx) % 3
    out = np.where(kind == 0, 0, np.where(kind == 1, 255, wave[np.arange(h)[:, None] % 8, np.arange(w)[None] % 8]))
    out = np.stack([out, out[:, ::-1], np.roll(out, 3, axis=0)], -1)
    return out.astype(np.uint8)


def corpus():
    rng = np.random.default_rng(7)
    items = []
    for h, w in SIZES:
        big = h * w > 40 * 40
        kinds = ['flat', 'gradient', 'zrl_dc11'] + (['noise'] if not big or (h, w) == (128, 128) else [])
        for kind in kinds:
            if kind == 'flat':
                img = np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()
            elif kind == 'noise':
                img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            elif kind == 'gradient':
                img = gradient(h, w, rng)
            else:
                img = zrl_dc11(h, w)
            qs = QUALITIES if not (big and kind == 'noise') else [50, 100]
            for q in qs:
                items.append((f'{kind}_{h}x{w}_q{q}', img, q))
    return items


def load_reference_camera_utils(ref):
    spec = importlib.util.spec_from_file_location('ref_camera_utils', os.path.join(ref, 'lib', 'core', 'utils', 'camera_utils.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    out = {}
    items = corpus()
    names, images, files, qualities, shapes = [], [], [], [], []
    ff_files = 0
    for name, img, q in items:
        ok, enc = cv2.imencode('.jpg', np.ascontiguousarray(img[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, q])
        assert ok
        data = enc.tobytes()
        ff_files += b'\xff\x00' in data
        names.append(name)
        images.append(img.reshape(-1))
        files.append(np.frombuffer(data, np.uint8))
        qualities.append(q)
        shapes.append(img.shape[:2])
    assert ff_files > 0, 'the corpus must hold stuffed 0xFF bytes'
    pix_off = np.cumsum([0] + [len(i) for i in images])
    file_off = np.cumsum([0] + [len(f) for f in files])
    out.update(jpeg_names=np.array(names), jpeg_shapes=np.array(shapes, np.int64), jpeg_quality=np.array(qualities, np.int64),
               jpeg_pixels=np.concatenate(images), jpeg_pixel_offsets=pix_off.astype(np.int64),
               jpeg_files=np.concatenate(files), jpeg_file_offsets=file_off.astype(np.int64))
    # camera path, executed from the reference
    cu = load_reference_camera_utils(ref)
    cam_dir = os.path.join(ref, 'demo', 'camera_spiral_cars')
    pose_name = sorted(os.listdir(os.path.join(cam_dir, 'pose')))[CAMERA_ID]
    with open(os.path.join(cam_dir, 'pose', pose_name)) as f:
        pose_text = f.read()
    with open(os.path.join(cam_dir, 'intrinsics.txt')) as f:
        intr_text = f.read()
    c2w = torch.from_numpy(np.loadtxt(os.path.join(cam_dir, 'pose', pose_name), dtype=np.float32, delimiter=' ').reshape(4, 4))
    cam_to_ndc = torch.cat([c2w[:3, :3], c2w[:3, 3:] * 2], dim=-1)
    pose = torch.cat([cam_to_ndc, cam_to_ndc.new_tensor([[0.0, 0.0, 0.0, 1.0]])], dim=-2)
    out.update(camera_pose_name=np.array(pose_name), camera_pose_text=np.array(pose_text), camera_intrinsics_text=np.array(intr_text),
               camera_id=np.int64(CAMERA_ID), gui_pose=pose.numpy())
    for num_frames, amp in PATHS:
        out[f'surround_{num_frames}_{amp}'] = cu.surround_views(pose, angle_amp=amp, num_frames=num_frames).numpy()
    path = os.path.join(HERE, 'reference_video_v1.npz')
    np.savez_compressed(path, **out)
    print(f'{path}: {len(items)} JPEG files ({ff_files} with stuffed 0xFF), {len(PATHS)} camera paths, {os.path.getsize(path)} bytes')


if __name__ == '__main__':
    main()
