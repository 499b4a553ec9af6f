"""Time the dataset PNG path at the bench's val_cond batch: 16 scenes x 251 views = 4016 views of 128 x 128 RGBA, written from seeded
render-like images at the writer's default compression (OpenCV when importable, else PIL) into a temporary directory.

Reports, in one call:
  * the card's name and power limit;
  * the device decode (CUDA events around the decode launch alone, median of --reps);
  * the host-to-device copy of the packed compressed streams against that of the equivalent float32 images (pinned, CUDA events);
  * the host side of the native path: file reads, and chunk parsing + packing;
  * the native path end to end (reads, parsing, copy, decode, status read; synchronised) and the reference's proxy,
    `cv2.imread(IMREAD_COLOR)` -> RGB -> `astype(float32) / 255` per file and `torch.stack`, on 1 and on 4 threads, the three
    alternating per repetition, as medians.
Prints one JSON line.

    python tests/perf/png_decode_timing.py [--views 4016] [--reps 5]
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
from ssdnerf_b200 import datasets as D  # noqa: E402

try:
    import cv2
except ImportError:       # the proxy then reads with PIL
    cv2 = None


def render_like(rng, h, w):
    """an RGBA object render: a shaded ellipse on a white, transparent background"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    cy, cx = h * rng.uniform(0.4, 0.6), w * rng.uniform(0.4, 0.6)
    ry, rx = h * rng.uniform(0.2, 0.35), w * rng.uniform(0.2, 0.35)
    d = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2
    inside = d < 1
    shade = (1 - 0.6 * d)[..., None] * rng.uniform(0, 255, 3) + 20 * np.sin(x / 3 + y / 5)[..., None]
    rgb = np.clip(np.where(inside[..., None], shade + rng.normal(0, 1.5, shade.shape), 255.0), 0, 255).astype(np.uint8)
    return np.concatenate([rgb, np.where(inside, 255, 0).astype(np.uint8)[..., None]], -1)


def write_file(path, rgba):
    if cv2 is not None:
        cv2.imwrite(path, rgba[..., [2, 1, 0, 3]])
    else:
        from PIL import Image
        Image.fromarray(rgba).save(path)


def read_proxy(path):
    if cv2 is not None:
        img = cv2.imread(path, cv2.IMREAD_COLOR)[..., ::-1]
    else:
        from PIL import Image
        img = np.asarray(Image.open(path).convert('RGB'))
    return torch.from_numpy(img.astype(np.float32) / 255)


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip()
    except Exception as e:      # noqa: BLE001
        power = f'unavailable ({e})'
    return name, power


def events_ms(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=4016)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dev = torch.device('cuda', torch.cuda.current_device())
    name, power = card()
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i in range(a.views):
            p = os.path.join(tmp, f'{i:06d}.png')
            write_file(p, render_like(rng, 128, 128))
            paths.append(p)
        file_bytes = sum(os.path.getsize(p) for p in paths)

        def native():
            files = []
            for p in paths:
                with open(p, 'rb') as f:
                    files.append(f.read())
            out = D.decode_png(files, dev, paths)
            torch.cuda.synchronize()
            return out

        def proxy(threads):
            if threads == 1:
                imgs = [read_proxy(p) for p in paths]
            else:
                with ThreadPoolExecutor(threads) as ex:
                    imgs = list(ex.map(read_proxy, paths))
            return torch.stack(imgs)

        # results agree (the native path is bit-exact with cv2; PIL's decode gives the same bytes for these files)
        ref = proxy(4)
        got = native()
        assert torch.equal(got.cpu(), ref), 'native decode differs from the proxy'

        # host side of the native path
        t0 = time.perf_counter()
        files = []
        for p in paths:
            with open(p, 'rb') as f:
                files.append(f.read())
        t_read = time.perf_counter() - t0
        t0 = time.perf_counter()
        infos = [D.parse_png(f, p) for f, p in zip(files, paths)]
        host, desc_off, work_bytes, offsets = D._pack(infos)
        t_parse = time.perf_counter() - t0

        # device pieces
        dbuf = host.to(dev)
        work = torch.empty(work_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty(int(offsets[-1]), dtype=torch.float32, device=dev)
        status = torch.empty(len(infos), dtype=torch.int32, device=dev)
        D._launch(dbuf, desc_off, work, out, status, dev)
        torch.cuda.synchronize()
        assert not status.any().item()
        t_decode = events_ms(lambda: D._launch(dbuf, desc_off, work, out, status, dev), a.reps * 4)
        h2d_streams = events_ms(lambda: dbuf.copy_(host, non_blocking=True), a.reps * 4)
        pinned_f32 = torch.empty(out.numel(), dtype=torch.float32, pin_memory=True)
        h2d_f32 = events_ms(lambda: out.copy_(pinned_f32, non_blocking=True), a.reps * 4)

        # end to end, alternating
        tn, t1, t4 = [], [], []
        for _ in range(a.reps):
            for fn, acc in ((native, tn), (lambda: proxy(1), t1), (lambda: proxy(4), t4)):
                t0 = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t0)
    res = dict(
        card=name, power_limit=power, views=a.views, size='128x128 RGBA', writer_and_proxy='cv2' if cv2 is not None else 'PIL',
        file_bytes=file_bytes, packed_bytes=int(host.numel()), float32_bytes=int(out.numel() * 4),
        device_decode_ms=round(t_decode, 3), h2d_streams_ms=round(h2d_streams, 3), h2d_float32_ms=round(h2d_f32, 3),
        host_read_ms=round(t_read * 1e3, 1), host_parse_pack_ms=round(t_parse * 1e3, 1),
        native_end_to_end_ms=round(float(np.median(tn)) * 1e3, 1),
        proxy_1_thread_ms=round(float(np.median(t1)) * 1e3, 1), proxy_4_threads_ms=round(float(np.median(t4)) * 1e3, 1),
        decode_speedup_vs_4_threads=round(float(np.median(t4)) * 1e3 / t_decode, 1),
        end_to_end_speedup_vs_4_threads=round(float(np.median(t4)) / float(np.median(tn)), 2))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
