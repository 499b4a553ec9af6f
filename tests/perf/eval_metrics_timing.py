"""Time the val_step metrics over a bench-size val_cond batch: 16 scenes x 251 views = 4016 (pred, target) pairs of 128 x 128 images.
SSIM (one launch) and LPIPS(VGG16, random Kaiming weights: the time does not depend on their values) with CUDA events after a warm-up.
Prints one JSON line: ms per metric, LPIPS TFLOP/s from shape-computed flops, and the card's name, power limit and max SM clock read in
the same run.  Run from the repository root: python tests/perf/eval_metrics_timing.py"""
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from oracle import metrics_port as mp
from ssdnerf_b200 import lpips as LP
from ssdnerf_b200 import metrics as M


def vgg_flops(h, w):
    """2 x MACs of the 13 convolutions (3 x 3, the real 3 input channels of the first) for one image"""
    f, hl, wl, cin = 0, h, w, 3
    for li, cout in enumerate(mp.VGG_CHANNELS):
        if li in (2, 4, 7, 10):
            hl, wl = hl // 2, wl // 2
        f += 2 * hl * wl * cout * cin * 9
        cin = cout
    return f


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    dev = torch.device('cuda:0')
    n, h, w = 4016, 128, 128
    p, t = mp.synthetic_pairs(64, h, w, seed=0)
    idx = torch.arange(n) % 64
    pred, target = torch.from_numpy(p)[idx].to(dev), torch.from_numpy(t)[idx].to(dev)
    with tempfile.TemporaryDirectory() as d:
        vgg, lin = mp.random_weights(0)
        torch.save(vgg, os.path.join(d, 'vgg16.pth'))
        torch.save(lin, os.path.join(d, 'vgg.pth'))
        lp = LP.LPIPS(os.path.join(d, 'vgg16.pth'), os.path.join(d, 'vgg.pth'))
    ssim_ms = timed(lambda: M.ssim(pred, target), 20)
    lpips_ms = timed(lambda: lp(pred, target), 3)
    flops = 2 * n * vgg_flops(h, w)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    res = dict(pairs=n, size=[h, w], ssim_ms=round(ssim_ms, 3), lpips_ms=round(lpips_ms, 2), lpips_chunk=lp.chunk(h, w),
               lpips_tflops=round(flops / (lpips_ms * 1e-3) / 1e12, 1), lpips_tflop_per_batch=round(flops / 1e12, 2), gpu=smi)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
