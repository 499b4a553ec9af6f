"""DDIM-stage throughput of the tiled-triplane denoiser (6 x 128 x 384 latents, widths 80 / 160 / 320, GroupNorm(16)) next to the
standard cars denoiser (18 x 128 x 128, widths 128 / 256 / 512) in the same process: captured-graph unguided DDIM at batch 8
(samples_per_gpu), random weights, CUDA-event timing.  Prints one JSON line per model (and writes them to --out as a JSON list).

    python tests/perf/ddim_tiled_throughput.py [--steps 75] [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import unet_port as up  # noqa: E402
from ssdnerf_b200.diffusion import GaussianDiffusion  # noqa: E402
from ssdnerf_b200.unet import DenoisingUnetMod  # noqa: E402

MODELS = {
    'tiled': (dict(image_size=128, in_channels=6, base_channels=80, channels_cfg=[1, 1, 2, 2, 4, 4], resblocks_per_downsample=2, num_heads=4,
                   attention_res=[16, 8, 4], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True),
              dict(image_size=128, in_channels=6, base_channels=80, channels_cfg=(1, 1, 2, 2, 4, 4), attention_res=(16, 8, 4)), (6, 128, 384)),
    'standard': (dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2, num_heads=4,
                      attention_res=[32, 16, 8], use_scale_shift_norm=True), dict(), (18, 128, 128)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=75)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda')
    props = torch.cuda.get_device_properties(dev)
    lines = []
    for name, (cfg, spec_kw, shape) in MODELS.items():
        m = DenoisingUnetMod(**cfg)
        m.load_state_dict(up.random_state_dict(up.unet_spec(**spec_kw), seed=0), strict=True)
        m = m.to(dev).eval()
        diff = GaussianDiffusion(m, betas_cfg=dict(type='linear'), num_timesteps=1000,
                                 test_cfg=dict(num_timesteps=args.steps, clip_range=[-2, 2])).to(dev)
        noise = torch.randn(args.batch, *shape, device=dev)
        diff(noise, return_loss=False)                    # capture + warm-up
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            diff(noise, return_loss=False)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b) / 1000.0)
        t = min(times)
        lines.append(dict(model=name, latent=list(shape), batch=args.batch, ddim_steps=args.steps, seconds=round(t, 4),
                          triplanes_per_s=round(args.batch / t, 3), ms_per_eval=round(1000 * t / args.steps, 3),
                          spread_s=[round(x, 4) for x in times], gpu=props.name))
        print(json.dumps(lines[-1]), flush=True)
        del diff, m
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
