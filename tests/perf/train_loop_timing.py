"""The training driver's overhead on stage 2 (`configs/paper_cfgs/stage2_cars_uncond.py`: the denoiser trained on stored triplanes):
iterations/s of `runner.train_model` (loader with prefetch, LR / EMA / logger hooks, as the config registers them; no checkpoints,
no evaluation) against a bare loop of `collate` + `train_step` over the same synthetic scenes, the two alternated over several rounds.
Prints one JSON line with both rates, the EMA hook's share measured by CUDA events, and the card's name and power limit.

    python tests/perf/train_loop_timing.py [--scenes 64] [--iters 40] [--rounds 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=64)
    ap.add_argument('--iters', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import ssdnerf_b200 as S
    from ssdnerf_b200 import ema as E
    from ssdnerf_b200.config import _wrap
    from ssdnerf_b200.runner import build_optimizers, train_model
    from tests.perf.ema_timing import card
    from tests.test_eval_driver_gpu import write_srn_tree
    golden = os.path.join(ROOT, 'tests', 'golden')
    ref = json.load(open(os.path.join(golden, 'reference_configs.json')))['configs/paper_cfgs/stage2_cars_uncond.py']
    rc = json.load(open(os.path.join(golden, 'reference_runner_configs.json')))['configs/paper_cfgs/stage2_cars_uncond.py']
    tmp = tempfile.mkdtemp()
    tree, code = os.path.join(tmp, 'srn'), os.path.join(tmp, 'code')
    os.makedirs(code)
    names = write_srn_tree(tree, args.scenes, 2, 32, distinct=2)
    g = torch.Generator().manual_seed(0)
    for n in names:
        torch.save(dict(scene_name=n, param=dict(code=torch.randn(3, 6, 128, 128, generator=g) * 0.5,
                                                   density_grid=torch.zeros(64 ** 3, dtype=torch.float16),
                                                   density_bitfield=torch.zeros(64 ** 3 // 8, dtype=torch.uint8))),
                   os.path.join(code, n + '.pth'))
    spg = ref['samples_per_gpu']
    train = dict(rc['data.train'], data_prefix=tree, code_dir=code)
    train.pop('cache_path', None)
    device = torch.device('cuda')

    def build():
        torch.manual_seed(0)
        return S.build_model(ref['model'], train_cfg=ref['train_cfg'], test_cfg=ref['test_cfg']).to(device)

    def driver(work):
        model = build()
        cfg = _wrap(dict(data=dict(samples_per_gpu=spg, train=train), optimizer=rc['optimizer'], lr_config=rc['lr_config'],
                         checkpoint_config=None, log_config=dict(rc['log_config'], hooks=[dict(type='TextLoggerHook')]),
                         custom_hooks=rc['custom_hooks'], total_iters=args.iters, workflow=rc['workflow'], work_dir=work, seed=0))
        ds = S.build_dataset(train)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        train_model(model, ds, cfg, device=device)
        torch.cuda.synchronize()
        return args.iters / (time.perf_counter() - t0)

    def bare():
        model = build().train()
        opts = build_optimizers(model, rc['optimizer'])
        ds = S.build_dataset(train)
        order = torch.randperm(len(ds)).tolist()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(args.iters):
            ids = [order[(i * spg + k) % len(order)] for k in range(spg)]
            model.train_step(S.collate([ds[j] for j in ids], device), opts, running_status=dict(iteration=i, epoch=0))
        torch.cuda.synchronize()
        return args.iters / (time.perf_counter() - t0)

    # the EMA hook alone on the same model, by CUDA events
    model = build()
    hook = E.ExponentialMovingAverageHook(**{k: v for k, v in rc['custom_hooks'][0].items() if k not in ('type', 'priority')})
    for i in range(3):
        hook.update(model, i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    for i in range(20):
        hook.update(model, i)
    b.record()
    b.synchronize()
    ema_ms, ema_host_ms = a.elapsed_time(b) / 20, (time.perf_counter() - t0) * 1e3 / 20
    del model

    driver(os.path.join(tmp, 'warm'))
    bare()
    rates = dict(driver=[], bare=[])
    for r in range(args.rounds):
        rates['driver'].append(driver(os.path.join(tmp, f'w{r}')))
        rates['bare'].append(bare())
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    print(json.dumps(dict(card=card(), scenes=args.scenes, samples_per_gpu=spg, iters=args.iters, its_per_s=rates, median=med,
                          driver_over_bare=med['driver'] / med['bare'], ema_hook_ms_device=ema_ms, ema_hook_ms_host=ema_host_ms)))


if __name__ == '__main__':
    main()
