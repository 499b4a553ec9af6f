"""Time `python -m ssdnerf_b200.test`'s loop (`SceneBatches` + `evaluate_3d`) on the cars unconditional config
(configs/paper_cfgs/ssdnerf_cars_uncond.py: 50-step DDIM, 128 x 128 renders) at samples_per_gpu = 8, with a seeded random denoiser,
over a synthetic SRN tree of --scenes scenes x 251 views in a temporary directory (8 distinct scenes; the others are symbolic links
to them, so the files are read again under other scene names).

Two workloads:
  * val_uncond as the config has it: no image files are read (`load_imgs=False`), 251 test poses per scene;
  * val_uncond with its test images (`load_imgs=True, num_train_imgs=0`): 251 PNG reads and decodes per scene, PSNR / SSIM logged.
For each, scenes/s through the driver with and without the prefetch thread, alternated --reps times in this one call (medians and
all runs reported), then one torch.profiler trace of two batches of the second workload with the prefetch thread: device time by
kernel, the share of PyTorch's own (at::native) kernels, and the idle time of the device between and within the batches.
The card's name and power limit are read in the same call.  Prints one JSON line.

    python tests/perf/eval_driver_timing.py [--scenes 96] [--reps 2] [--trace-dir DIR]
"""
import argparse
import itertools
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import ssdnerf_b200 as S  # noqa: E402
from ssdnerf_b200.evaluation import SceneBatches, evaluate_3d  # noqa: E402
from tests.test_eval_driver_gpu import _ref_cfg, write_srn_tree  # noqa: E402

VIEWS, RES, SPG = 251, 128, 8


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()[0]
        return [x.strip() for x in q.split(',')]
    except Exception as e:          # the numbers still print; the card is then unknown
        return [f'nvidia-smi failed: {e}']


def build_model():
    from oracle import unet_port as up
    c = _ref_cfg('ssdnerf_cars_uncond')
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg'])
    sd = up.random_state_dict(up.unet_spec(), seed=7, std=0.02)
    for diff in (model.diffusion, model.diffusion_ema):
        diff.denoising.load_state_dict(sd, strict=True)
    return model.cuda().eval()


def run(model, ds, prefetch, max_batches=None):
    batches = SceneBatches(ds, SPG, 'cuda', prefetch=prefetch)
    if max_batches is not None:
        batches = itertools.islice(batches, max_batches)
    torch.manual_seed(0)          # the same noise in every run: the two loops' log_vars are comparable
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    log_vars = evaluate_3d(model, batches, metrics=None)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, log_vars


def kernel_summary(trace_path, num_batches):
    with open(trace_path) as f:
        events = [e for e in json.load(f)['traceEvents'] if e.get('cat') == 'kernel' and 'dur' in e]
    events.sort(key=lambda e: e['ts'])
    by_name = {}
    for e in events:
        by_name[e['name']] = by_name.get(e['name'], 0.0) + e['dur']
    total = sum(by_name.values())
    aten = sum(v for k, v in by_name.items() if 'at::native' in k)
    span = events[-1]['ts'] + events[-1]['dur'] - events[0]['ts']
    gaps, end = [], events[0]['ts']
    for e in events:
        if e['ts'] > end:
            gaps.append(e['ts'] - end)
        end = max(end, e['ts'] + e['dur'])
    top = sorted(by_name.items(), key=lambda kv: -kv[1])[:12]
    return dict(batches=num_batches, kernels=len(events), kernel_us=round(total), span_us=round(span), idle_us=round(sum(gaps)),
                largest_gaps_us=[round(g) for g in sorted(gaps, reverse=True)[:5]], aten_share=round(aten / total, 4),
                aten_us=round(aten), top=[(k[:90], round(v), round(v / total, 4)) for k, v in top])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=96)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--trace-dir', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs a GPU'
    info = card()
    c = _ref_cfg('ssdnerf_cars_uncond')
    with tempfile.TemporaryDirectory() as tmp:
        tree = os.path.join(tmp, 'cars_test')
        write_srn_tree(tree, args.scenes, VIEWS, RES, distinct=8)
        model = build_model()
        workloads = dict(
            config=S.build_dataset(dict(type='ShapeNetSRN', data_prefix=tree, load_imgs=False, num_test_imgs=VIEWS, scene_id_as_name=True)),
            test_imgs=S.build_dataset(dict(type='ShapeNetSRN', data_prefix=tree, num_train_imgs=0, scene_id_as_name=True)))
        result = dict(card=info, scenes=args.scenes, views=VIEWS, res=RES, samples_per_gpu=SPG,
                      num_timesteps=c['test_cfg']['num_timesteps'])
        for name, ds in workloads.items():
            run(model, ds, True, max_batches=2)                      # warm-up: graph capture, modules, allocator
            times = {True: [], False: []}
            logs = {}
            for _ in range(args.reps):
                for prefetch in (True, False):
                    t, logs[prefetch] = run(model, ds, prefetch)
                    times[prefetch].append(t)
            result[name] = dict(
                prefetch_scenes_per_s=round(args.scenes / float(np.median(times[True])), 3),
                no_prefetch_scenes_per_s=round(args.scenes / float(np.median(times[False])), 3),
                prefetch_s=[round(t, 3) for t in times[True]], no_prefetch_s=[round(t, 3) for t in times[False]],
                log_vars={str(k): {n: float(v) for n, v in lv.items()} for k, lv in logs.items()})
        # one trace of two batches with test images
        from torch.profiler import ProfilerActivity, profile
        trace_dir = args.trace_dir or tmp
        os.makedirs(trace_dir, exist_ok=True)
        trace = os.path.join(trace_dir, 'eval_driver_trace.json')
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            run(model, workloads['test_imgs'], True, max_batches=2)
        prof.export_chrome_trace(trace)
        result['profile'] = kernel_summary(trace, 2)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
