"""Time the viz_dir PNG path at the bench's val_cond batch: 4016 views of 128 x 256 (real | prediction), as eval_and_viz writes them.

Reports the device encode time (CUDA events around the four kernels), the device-to-host copy of the compressed bytes, the host file
writes, the bytes written with their ratio to zlib level 6 on the same filtered streams, and the reference's proxy: PIL's
`Image.fromarray(rgba).save(png)` per image (what plt.imsave calls), single thread, in this process.  The images are synthetic
render-like views (tests/test_viz_gpu.py:_render_like).  Prints one JSON line.

    python tests/perf/viz_png_timing.py [--views 4016] [--proxy-views 256] [--bench-dump DIR]

With --bench-dump DIR (from `bench.py --dump-outputs DIR`) the size ratio to zlib level 6 is also taken on the bench's own renders (views
as real | prediction pairs of two views) and on its sampled triplanes as visualize maps.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from ssdnerf_b200 import _lib as N  # noqa: E402
from ssdnerf_b200 import viz  # noqa: E402
from tests import png_check  # noqa: E402
from tests.test_viz_gpu import _render_like  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=4016)
    ap.add_argument('--proxy-views', type=int, default=256)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--bench-dump', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dev = torch.device('cuda:0')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,temperature.gpu,utilization.gpu', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    base_p, base_r = _render_like(64, 128, 128, 0, dev), _render_like(64, 128, 128, 1, dev)
    reps = -(-a.views // 64)
    pred = base_p.repeat(reps, 1, 1, 1)[:a.views].contiguous()
    real = base_r.flip(0).repeat(reps, 1, 1, 1)[:a.views].contiguous()
    pred = (pred + 0.02 * torch.rand(pred.shape, device=dev, generator=torch.Generator(dev).manual_seed(0))).contiguous()
    n, h, wv = a.views, 128, 128
    L, stream = N.lib(), N.stream_ptr()
    ws_b, out_b = L.ssdnerf_png_workspace_bytes(n, h, 2 * wv), L.ssdnerf_png_output_bound(n, h, 2 * wv)
    work = torch.empty(ws_b, dtype=torch.uint8, device=dev)
    out = torch.empty(out_b, dtype=torch.uint8, device=dev)
    off = torch.empty(n + 1, dtype=torch.int64, device=dev)

    def encode():
        N.check(L.ssdnerf_png_encode_views(N.ptr(pred), N.ptr(real), n, h, wv, N.ptr(work), ws_b, N.ptr(out), out_b, N.ptr(off), stream))
    encode()
    torch.cuda.synchronize()
    t_dev = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        encode()
        e1.record()
        torch.cuda.synchronize()
        t_dev.append(e0.elapsed_time(e1) / 1e3)
    t0 = time.perf_counter()
    offs = off.cpu().tolist()
    data = out[:offs[-1]].cpu().numpy().tobytes()
    t_d2h = time.perf_counter() - t0
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        for i in range(n):
            with open(os.path.join(d, f'{i:05d}.png'), 'wb') as f:
                f.write(data[offs[i]:offs[i + 1]])
        t_write = time.perf_counter() - t0
    t0 = time.perf_counter()
    files = viz.encode_png(pred=pred, real=real)
    torch.cuda.synchronize()
    t_api = time.perf_counter() - t0
    assert files == [data[offs[i]:offs[i + 1]] for i in range(n)]
    # size against zlib level 6 on the same filtered streams (a sample of 256 files), decoded pixels checked on the same sample
    exp = torch.round(torch.round(pred.clamp(0, 1) * 255) / 255 * 255).to(torch.uint8)
    exp = torch.cat([(real * 255).to(torch.uint8), exp], dim=2)
    exp = torch.cat([exp, torch.full_like(exp[..., :1], 255)], dim=-1)
    idx = np.linspace(0, n - 1, min(n, 256)).astype(int)
    native = z6 = 0
    for i in idx:
        px, raw, payload = png_check.decode(files[i])
        assert np.array_equal(px, exp[i].cpu().numpy())
        native += payload
        z6 += len(zlib.compress(raw, 6)) - 6
    # reference proxy: PIL per image
    from PIL import Image
    rgba = exp[:a.proxy_views].cpu().numpy()
    t0 = time.perf_counter()
    for i in range(len(rgba)):
        buf = io.BytesIO()
        Image.fromarray(rgba[i]).save(buf, format='png')
    t_pil = (time.perf_counter() - t0) / len(rgba)
    res = dict(gpu=gpu, views=n, shape=[h, 2 * wv], device_encode_s=min(t_dev), device_encode_all_s=t_dev, d2h_s=t_d2h, host_write_s=t_write,
               encode_png_call_s=t_api, bytes_total=offs[-1], bytes_per_view=offs[-1] / n, ratio_vs_zlib6=native / z6,
               pil_proxy_s_per_image=t_pil, pil_proxy_batch_s=t_pil * n,
               speedup_end_to_end=(t_pil * n) / (min(t_dev) + t_d2h + t_write), workspace_bytes=ws_b, output_bound_bytes=out_b)
    if a.bench_dump:
        img = torch.from_numpy(np.load(os.path.join(a.bench_dump, 'image.npy'))).to(dev)
        img = img.reshape(-1, *img.shape[2:]).contiguous()
        code = torch.from_numpy(np.load(os.path.join(a.bench_dump, 'code.npy'))).to(dev)
        for kind, files in (('views', viz.encode_png(pred=img, real=img.roll(1, 0).contiguous())),
                            ('maps', viz.encode_png(maps=viz.code_maps(code).contiguous(), vmin=-1, vmax=1))):
            res[f'bench_{kind}_ratio_vs_zlib6'] = _ratio(files)
            res[f'bench_{kind}_zlib1_ratio_vs_zlib6'] = _ratio(files, level=1)
        res['bench_dump_views'] = len(img)
    print(json.dumps(res))


def _ratio(files, level=None):
    """total native deflate bytes (or zlib at `level` on the same filtered streams) over zlib level 6's"""
    num = z6 = 0
    for data in files:
        _, raw, payload = png_check.decode(data)
        num += payload if level is None else len(zlib.compress(raw, level)) - 6
        z6 += len(zlib.compress(raw, 6)) - 6
    return num / z6


if __name__ == '__main__':
    main()
