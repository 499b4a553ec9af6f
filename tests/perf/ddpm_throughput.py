"""Sampling throughput of the captured DDPM loop next to the captured DDIM loop, same process, same cars denoiser (18 x 128 x 128 latents,
widths 128 / 256 / 512, random weights), batch 16: per-evaluation time of whole calls (1000-step DDPM, 50-step DDIM, run alternately,
medians), and the fused update kernels alone (k_ddpm_update with its in-kernel noise, k_ddim_update) on the same buffers, CUDA events
over many launches.  Card name, power limit and max SM clock are read in the same run.  Prints one JSON line.

    python tests/perf/ddpm_throughput.py [--batch 16] [--ddpm-steps 1000] [--ddim-steps 50] [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import unet_port as up  # noqa: E402
from ssdnerf_b200 import _lib as N  # noqa: E402
from ssdnerf_b200.diffusion import GaussianDiffusion  # noqa: E402
from ssdnerf_b200.unet import DenoisingUnetMod  # noqa: E402

CARS = dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2, num_heads=4,
            attention_res=[32, 16, 8], use_scale_shift_norm=True)


def _timed(fn, n=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1000.0 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--ddpm-steps', type=int, default=1000)
    ap.add_argument('--ddim-steps', type=int, default=50)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    m = DenoisingUnetMod(**CARS)
    m.load_state_dict(up.random_state_dict(up.unet_spec(), seed=0), strict=True)
    m = m.to(dev).eval()
    B = args.batch
    diffs = dict(ddpm=GaussianDiffusion(m, betas_cfg=dict(type='linear'), sample_method='ddpm',
                                        test_cfg=dict(num_timesteps=args.ddpm_steps, clip_range=[-2, 2])),
                 ddim=GaussianDiffusion(m, betas_cfg=dict(type='linear'), test_cfg=dict(num_timesteps=args.ddim_steps, clip_range=[-2, 2])))
    steps = dict(ddpm=args.ddpm_steps, ddim=args.ddim_steps)
    noise = torch.randn(B, 18, 128, 128, device=dev)
    for d in diffs.values():
        d(noise, return_loss=False)                       # capture + warm-up
    per_eval = {k: [] for k in diffs}
    for _ in range(args.reps):
        for k, d in diffs.items():
            per_eval[k].append(1000 * _timed(lambda: d(noise, return_loss=False)) / steps[k])
    # the update kernels alone, on the engine's own buffers (v = one UNet output, next input = the engine's input buffer)
    eng = m.engine(B, dev, (128, 128))
    x = noise.clone()
    eng.load_input_nchw(x)
    v = eng.forward_nhwc().clone()
    L, s = N.lib(), N.stream_ptr()
    C, H, W = 18, 128, 128
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    seed = torch.full((1,), 1234, dtype=torch.int64, device=dev)
    coef_p = diffs['ddpm'].ddpm_coefficients(diffs['ddpm'].ddim_timesteps(args.ddpm_steps)).to(dev)
    coef_i = diffs['ddim'].ddim_coefficients(diffs['ddim'].ddim_timesteps(args.ddim_steps)).to(dev)
    args_common = (N.ptr(x), N.ptr(v), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W), N.c_u32(v.shape[-1]))
    launch = dict(
        k_ddpm_update=lambda: N.check(L.ssdnerf_ddpm_update(*args_common, N.ptr(coef_p), N.ptr(step), N.ptr(seed), N.c_int(1), N.c_f32(-2), N.c_f32(2),
                                                            N.ptr(eng.x_in), N.c_u32(eng.CPAD_IN), s)),
        k_ddim_update=lambda: N.check(L.ssdnerf_ddim_update(*args_common, N.ptr(coef_i), N.ptr(step), N.c_int(1), N.c_f32(-2), N.c_f32(2), None,
                                                            N.ptr(eng.x_in), N.c_u32(eng.CPAD_IN), s)))
    kernel_us = {}
    for k, fn in launch.items():
        fn()
        torch.cuda.synchronize()
        kernel_us[k] = round(1e6 * statistics.median(_timed(fn, 200) for _ in range(5)), 2)
    px = B * H * W
    bytes_moved = px * (2 * C * 4 + C * 4 + eng.CPAD_IN * 2)           # x_t read + write, the C used channels of v, the fp16 next input
    line = dict(gpu=gpu, batch=B, ddpm_steps=args.ddpm_steps, ddim_steps=args.ddim_steps,
                ddpm_ms_per_eval=round(statistics.median(per_eval['ddpm']), 3), ddim_ms_per_eval=round(statistics.median(per_eval['ddim']), 3),
                ddpm_ms_per_eval_all=[round(t, 3) for t in per_eval['ddpm']], ddim_ms_per_eval_all=[round(t, 3) for t in per_eval['ddim']],
                ddpm_call_s=round(statistics.median(per_eval['ddpm']) * args.ddpm_steps / 1000, 3),
                update_kernel_us=kernel_us, update_bytes=bytes_moved,
                ddpm_update_GBps=round(bytes_moved / kernel_us['k_ddpm_update'] / 1e3, 1))
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
