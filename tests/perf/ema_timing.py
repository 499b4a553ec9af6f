"""EMA update of the cars denoiser's state (plus the decoder): the fused kernel against the bit-identical
`torch._foreach_sub / _foreach_mul / _foreach_add` composition and against mmgen's per-tensor loop (`a + (b - a) * m`, then
`load_state_dict`).  The kernel is timed twice: `fused_launch` calls the C entry point on a table built once (the launch alone),
`fused` calls `ema.ema_lerp_`, which rebuilds the ctypes table in Python on every call.  CUDA events around each, the four
alternated over several rounds; prints one JSON line with the median milliseconds, the bytes the kernel moves by the shapes and
the card's name and power limit.

    python tests/perf/ema_timing.py [--rounds 7] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import ssdnerf_b200 as S
    from ssdnerf_b200.ema import ema_lerp_, rampup_momentum
    c = json.load(open(os.path.join(os.path.dirname(os.path.dirname(__file__)), 'golden', 'reference_configs.json')))
    c = c['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg']).cuda()
    pairs = [(model.diffusion_ema, model.diffusion), (model.decoder_ema, model.decoder)]
    ema, src, tr = [], [], []
    for e_net, s_net in pairs:
        es = e_net.state_dict(keep_vars=True)
        for k, v in s_net.state_dict(keep_vars=True).items():
            ema.append(es[k])
            src.append(v)
            tr.append(v.requires_grad)
    ema_d, src_d = [t.detach() for t in ema], [t.detach() for t in src]
    m = rampup_momentum(100, ema_kimg=4, ema_rampup=0.05, batch_size=16, eps=1e-8)
    n = sum(t.numel() for t in ema)

    def fused():
        ema_lerp_(ema, src, tr, m, 0.0)

    # the launch alone: the ctypes table built once, the C entry point called directly
    from ssdnerf_b200 import _lib as N
    table = (N.EmaTensor * len(ema))()
    for i, (e, s_, t) in enumerate(zip(ema, src, tr)):
        table[i].ema, table[i].src, table[i].n, table[i].trainable = e.data_ptr(), s_.data_ptr(), e.numel(), int(t)
    L, stream = N.lib(), N.stream_ptr()

    def fused_launch():
        N.check(L.ssdnerf_ema_lerp_f32(table, len(ema), m, 0.0, stream))

    def foreach():
        d = torch._foreach_sub(ema_d, src_d)
        torch._foreach_mul_(d, m)
        res = torch._foreach_add(src_d, d)
        torch._foreach_copy_(ema_d, res)

    def mmgen():
        for e_net, s_net in pairs:
            states_ema = e_net.state_dict()
            for k, v in s_net.state_dict(keep_vars=True).items():
                states_ema[k] = (v + (states_ema[k] - v) * (m if v.requires_grad else 0.0)).detach()
            e_net.load_state_dict(states_ema, strict=True)

    fns = dict(fused_launch=fused_launch, fused=fused, foreach=foreach, mmgen=mmgen)
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / args.reps)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out = dict(card=card(), tensors=len(ema), elements=n, momentum=m, ms_median=med, ms_all=times,
               fused_bytes=3 * 4 * n, fused_launch_GBps=3 * 4 * n / med['fused_launch'] / 1e6,
               speedup_vs_foreach=med['foreach'] / med['fused'], speedup_vs_mmgen=med['mmgen'] / med['fused'])
    print(json.dumps(out))


if __name__ == '__main__':
    main()
