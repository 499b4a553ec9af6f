"""Time Inception-v3 feature extraction for FID / KID over one bench val_cond batch: 16 scenes x 251 views = 4016 images at 128 x 128
(resized to 299 x 299 inside, as the StyleGAN TorchScript does).  Weights are the seeded, calibrated ones of the test fixture (the time
does not depend on their values).

Native: ssdnerf_b200.inception.InceptionV3.  Proxy for the reference: the oracle network (oracle/inception_port.py) in float32 under
torch defaults with cuDNN, TF32 allowed and `cudnn.benchmark = True` as the configs set, fed the same preprocessed input in chunks of
251 images.  The two alternate in the same process, `--rounds` times after a warm-up; CUDA events around each.  Prints one JSON line:
median ms of each, TFLOP/s from the shape-computed 11.42 GFLOP per image, the share of the 989 TFLOP/s dense fp16 data-sheet figure,
and the card's name, power limit and max SM clock read in the same run.  Run from the repository root:
python tests/perf/inception_timing.py"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch
import torch.nn.functional as F

from oracle import inception_port as ip
from ssdnerf_b200.inception import InceptionV3

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'golden', 'reference_inception_v1.npz')


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    sd = ip.fixture_state_dict(np.load(GOLDEN))
    net = InceptionV3.from_state_dict(sd)
    P = {k: (w.float().to(dev), b.float().to(dev)) for k, (w, b) in ip.folded_params(sd).items()}
    n, h, w = 4016, 128, 128
    g = torch.Generator().manual_seed(0)
    x = (F.interpolate(torch.rand(n, 3, 8, 8, generator=g) * 2 - 1, size=(h, w), mode='bicubic', align_corners=False)
         + 0.15 * torch.randn(n, 3, h, w, generator=g)).clamp(-1, 1).to(dev)
    x299 = [ip.preprocess(x[j:j + 251].cpu(), torch.float32).to(dev) for j in range(0, n, 251)]   # the proxy's input, prepared once

    def native():
        net(x)

    def proxy():
        with torch.no_grad():
            for t in x299:
                ip.forward(P, t)

    native(); proxy()
    nat, prx = [], []
    for _ in range(args.rounds):
        nat.append(timed(native))
        prx.append(timed(proxy))
    nat_ms, prx_ms = float(np.median(nat)), float(np.median(prx))
    flops = n * ip.shape_gflop() * 1e9
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    res = dict(images=n, size=[h, w], chunk=net.chunk(), native_ms=round(nat_ms, 1), native_ms_all=[round(v, 1) for v in nat],
               proxy_fp32_cudnn_tf32_ms=round(prx_ms, 1), proxy_ms_all=[round(v, 1) for v in prx],
               proxy_excludes_preprocessing=True, speedup=round(prx_ms / nat_ms, 2),
               native_tflops=round(flops / (nat_ms * 1e-3) / 1e12, 1), share_of_989=round(flops / (nat_ms * 1e-3) / 989e12, 3),
               tflop_per_batch=round(flops / 1e12, 1), gpu=smi)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
