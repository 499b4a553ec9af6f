"""KITTI preprocessing on synthetic 1242 x 375 frames: the native tool (ssdnerf_b200.kitti) against a 4-thread cv2 proxy of the
reference loop (cv2.imread unchanged, mask / whiten / pad / cv2.resize, cv2.imwrite), split into host reads and the rest (device work, copies and writes) for the native tool, and into reads, pixel work and
writes (thread-seconds) for the proxy.

    python tests/perf/kitti_preproc_timing.py [--frames 64] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from ssdnerf_b200 import kitti as K  # noqa: E402
from tests.golden.make_golden_kitti import _calib, _label  # noqa: E402


def make_frames(root, n, cv2):
    rng = np.random.default_rng(0)
    for d in ('image_2', 'instance_2', 'label_2', 'calib'):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for f in range(n):
        stem = f'{f:06d}'
        yy, xx = np.mgrid[:375, :1242]
        img = (np.stack([xx % 256, yy % 256, (xx + yy) % 256], -1) + rng.integers(0, 16, (375, 1242, 3))).clip(0, 255).astype(np.uint8)
        seg = np.zeros((375, 1242), np.uint16)
        lines = []
        for i in range(6):
            x0, y0 = int(rng.integers(0, 1000)), int(rng.integers(100, 250))
            w, h = int(rng.integers(40, 240)), int(rng.integers(30, 120))
            m = np.zeros_like(seg, np.uint8)
            cv2.ellipse(m, (x0 + w // 2, y0 + h // 2), (w // 2, h // 2), 0, 0, 360, 1, -1)
            seg[m.astype(bool)] = 1000 + i
            lines.append(_label('Car', 0.0, int(i == 5), (x0, y0, x0 + w, y0 + h), (1.5, 1.6, 3.9), (float(rng.uniform(-8, 8)), 1.7,
                                float(rng.uniform(8, 40))), float(rng.uniform(-3, 3))))
        cv2.imwrite(os.path.join(root, 'image_2', stem + '.png'), img)
        cv2.imwrite(os.path.join(root, 'instance_2', stem + '.png'), seg)
        open(os.path.join(root, 'label_2', stem + '.txt'), 'w').write('\n'.join(lines) + '\n')
        open(os.path.join(root, 'calib', stem + '.txt'), 'w').write(_calib())


def cv2_proxy(root, out, cv2, threads=4):
    """the reference loop per frame on a 4-thread pool: returns (read s, pixel s, write s) summed over frames / threads"""
    stems = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(root, 'label_2')))
    t = np.zeros(3)

    def one(stem):
        a = time.perf_counter()
        labels = K.parse_labels(open(os.path.join(root, 'label_2', stem + '.txt')).read(), stem)
        proj = K.parse_calib(open(os.path.join(root, 'calib', stem + '.txt')).read(), stem)
        cam_t = K.camera_offset(proj)
        img = cv2.imread(os.path.join(root, 'image_2', stem + '.png'), cv2.IMREAD_UNCHANGED)
        seg = cv2.imread(os.path.join(root, 'instance_2', stem + '.png'), cv2.IMREAD_UNCHANGED)
        b = time.perf_counter()
        res, wt = [], 0.0
        for i, lab in enumerate(labels):
            if lab[1] != 0 or lab[2] != 0:
                continue
            ys, xs = (seg == 1000 + i).nonzero()
            if not len(ys):
                continue
            y0, y1, x0, x1 = ys.min(), ys.max() + 1, xs.min(), xs.max() + 1
            crop = img[y0:y1, x0:x1]
            crop[~(seg[y0:y1, x0:x1] == 1000 + i)] = 255
            c2w, pad, scale, px, py, text = K.instance_geometry(lab, cam_t, proj, y0, y1, x0, x1)
            if scale > 1:
                continue
            sq = np.pad(crop, ((py, pad - crop.shape[0] - py), (px, pad - crop.shape[1] - px), (0, 0)), constant_values=255)
            view = np.pad(cv2.resize(sq, (120, 120), interpolation=cv2.INTER_LINEAR), ((4, 4), (4, 4), (0, 0)), constant_values=255)
            c = time.perf_counter()
            d = os.path.join(out, f'{stem}_{i:03d}')
            os.makedirs(os.path.join(d, 'rgb'), exist_ok=True)
            os.makedirs(os.path.join(d, 'pose'), exist_ok=True)
            cv2.imwrite(os.path.join(d, 'rgb', '000000.png'), view)
            cv2.imwrite(os.path.join(d, '000000.png'), crop)
            np.savetxt(os.path.join(d, 'pose', '000000.txt'), c2w.reshape(1, -1))
            open(os.path.join(d, 'intrinsics.txt'), 'w').write(text)
            wt += time.perf_counter() - c
        e = time.perf_counter()
        return b - a, e - b - wt, wt

    w0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as pool:
        for r in pool.map(one, stems):
            t += r
    return time.perf_counter() - w0, t


def native(root, out, dev, batch=16):
    stems = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(root, 'label_2')))
    t = {'read_s': 0.0, 'device_and_write_s': 0.0}
    n = 0
    w0 = time.perf_counter()
    with ThreadPoolExecutor(8) as pool:
        for b in range(0, len(stems), batch):
            a = time.perf_counter()
            chunk = stems[b:b + batch]
            got = list(pool.map(lambda s: K._frame_inputs(root, s), chunk))
            frames = [(s, p, d) for s, (p, d) in zip(chunk, got)]
            c = time.perf_counter()
            t['read_s'] += c - a
            n += K.process_batch(frames, out, 128, 4, dev, pool)
            torch.cuda.synchronize()
            t['device_and_write_s'] += time.perf_counter() - c         # decode, boxes, crops, encode, copies and the writes
    return time.perf_counter() - w0, t, n


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, 'kitti')
        make_frames(root, a.frames, cv2)
        native(root, os.path.join(tmp, 'warm'), dev, batch=4)                # warm-up: module load, first launches
        res = {'gpu': gpu, 'frames': a.frames}
        for rep in range(2):
            wall, parts, n = native(root, os.path.join(tmp, f'native{rep}'), dev)
            res[f'native_{rep}'] = dict(wall_s=wall, instances=n, **parts)
            pwall, pt = cv2_proxy(root, os.path.join(tmp, f'proxy{rep}'), cv2)
            res[f'cv2_proxy_{rep}'] = dict(wall_s=pwall, read_thread_s=pt[0], pixel_thread_s=pt[1], write_thread_s=pt[2])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        open(a.out, 'w').write(line + '\n')


if __name__ == '__main__':
    main()
