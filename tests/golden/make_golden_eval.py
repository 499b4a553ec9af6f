"""Pins for ssdnerf_b200.evaluation: the reference's OWN `evaluate_3d` (lib/apis/test.py) and `DistributedSampler`
(lib/datasets/samplers/distributed_sampler.py), executed from /root/reference with mmcv / mmgen stubbed.  The stubs are what those two
files import: `mmcv.print_log` / `ProgressBar` (silent), `mmcv.runner.get_dist_info` (the torch.distributed state, or the sampler's
rank under test), mmgen's `FID` / `IS` classes (for the isinstance check), `get_module_device`, and mmgen's `DistributedSampler` base,
whose padding arithmetic is restated from memory [mmgen-memory] (`ceil(N / W / samples_per_gpu) * samples_per_gpu` per rank).

A deterministic stub model replays stored per-batch `log_vars`, `num_samples` and `pred_imgs` and records the `val_step` kwargs; two
recording metrics (one an `FID`, one not) record every feed's mode, shape and SHA-256.  Recorded:
    single/...  one process: 4 batches, the third without `test_imgs`, feed_batch_size 4, viz_step 2, sample_kwargs
    dist/...    world size 2 over gloo: each rank's batches and the all-reduced `log_vars` the reference returns on each rank
    sampler/N_W_spg/r   the indices rank r iterates, for (N, W, spg) in (10, 1, 4), (10, 2, 4), (10, 3, 2), (704, 8, 8)
-> tests/golden/reference_eval_v1.npz, replayed by tests/test_eval_driver_cpu.py.

    python tests/golden/make_golden_eval.py          (needs /root/reference)
"""
import hashlib
import importlib.util
import json
import math
import os
import socket
import sys
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
FEED_BATCH_SIZE, VIZ_DIR, VIZ_STEP = 4, 'work_dirs/viz', 2
SAMPLE_KWARGS = dict(num_timesteps=3, clip_range=[-1, 1])
SAMPLER_CASES = ((10, 1, 4), (10, 2, 4), (10, 3, 2), (704, 8, 8))
_SAMPLER_RANK = {}


def stub_mm():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class ProgressBar:
        def __init__(self, *a, **k):
            pass

        def update(self, *a, **k):
            pass

    def get_dist_info():
        if 'rank' in _SAMPLER_RANK:
            return _SAMPLER_RANK['rank'], _SAMPLER_RANK['world']
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
        return 0, 1

    class FID:
        name = 'FID'

    class IS:
        name = 'IS'

    def get_module_device(module):
        p = next(module.parameters())
        return p.get_device() if p.is_cuda else torch.device('cpu')

    class MMGenDistributedSampler(torch.utils.data.DistributedSampler):
        """mmgen.datasets.samplers.DistributedSampler [mmgen-memory]"""

        def __init__(self, dataset, num_replicas=None, rank=None, shuffle=True, samples_per_gpu=1, seed=0):
            super().__init__(dataset, num_replicas=num_replicas, rank=rank)
            self.shuffle, self.samples_per_gpu = shuffle, samples_per_gpu
            self.num_samples_per_replica = int(math.ceil(len(self.dataset) * 1.0 / self.num_replicas / samples_per_gpu))
            self.num_samples = self.num_samples_per_replica * self.samples_per_gpu
            self.total_size = self.num_samples * self.num_replicas
            self.seed = seed if seed is not None else 0

    mod('mmcv', print_log=lambda *a, **k: None, ProgressBar=ProgressBar).__path__ = []
    mod('mmcv.runner', get_dist_info=get_dist_info)
    for name in ('mmgen', 'mmgen.core', 'mmgen.core.evaluation', 'mmgen.models', 'mmgen.models.architectures'):
        mod(name).__path__ = []
    mod('mmgen.core.evaluation.metrics', FID=FID, IS=IS)
    mod('mmgen.models.architectures.common', get_module_device=get_module_device)
    mod('mmgen.datasets', DistributedSampler=MMGenDistributedSampler).__path__ = []


def load_ref(rel, name):
    stub_mm()
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def make_batches(seed, sizes, views, res, no_test_imgs=()):
    """per-batch stored inputs: pred_imgs [n, v, 3, res, res], test_imgs [n, v, res, res, 3] (not for batches in no_test_imgs),
    log_vars and num_samples"""
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(sizes):
        b = dict(n=n, pred=rng.random((n, views, 3, res, res), dtype=np.float32),
                 log_vars=dict(test_psnr=float(rng.uniform(10, 30)), test_ssim=float(rng.uniform(0.5, 1))))
        if i not in no_test_imgs:
            b['test_imgs'] = rng.random((n, views, res, res, 3), dtype=np.float32)
        out.append(b)
    return out


class StubModel(torch.nn.Module):
    """val_step replays the stored outputs of batch data['batch'] and records its keyword arguments"""

    def __init__(self, stored):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.stored, self.calls = stored, []

    def val_step(self, data, **kwargs):
        self.calls.append(json.dumps(kwargs, sort_keys=True))
        b = self.stored[data['batch']]
        return dict(log_vars=dict(b['log_vars']), num_samples=b['n'], pred_imgs=torch.from_numpy(b['pred']))


def batch_dicts(stored):
    out = []
    for i, b in enumerate(stored):
        d = dict(batch=i)
        if 'test_imgs' in b:
            d['test_imgs'] = torch.from_numpy(b['test_imgs'])
        out.append(d)
    return out


def feed_record(metric, imgs, mode):
    x = imgs.contiguous().numpy()
    return [metric, mode, list(x.shape), hashlib.sha256(x.tobytes()).hexdigest()]


def make_metrics(fid_base, feeds):
    class FakesOnly(fid_base):
        def feed(self, imgs, mode):
            feeds.append(feed_record('fakes_only', imgs, mode))

    class Both:
        name = 'Both'

        def feed(self, imgs, mode):
            feeds.append(feed_record('both', imgs, mode))
    return [FakesOnly(), Both()]


class Loader(list):
    def __init__(self, items, batch_size, num_scenes):
        super().__init__(items)
        self.batch_size, self.dataset = batch_size, list(range(num_scenes))


def save_stored(out, prefix, stored):
    out[f'{prefix}/num_batches'] = np.array(len(stored))
    for i, b in enumerate(stored):
        out[f'{prefix}/{i}/pred'] = b['pred']
        out[f'{prefix}/{i}/n'] = np.array(b['n'])
        out[f'{prefix}/{i}/log_vars'] = np.array(json.dumps(b['log_vars']))
        if 'test_imgs' in b:
            out[f'{prefix}/{i}/test_imgs'] = b['test_imgs']


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def dist_sizes(rank):
    return [3, 3, 2] if rank == 0 else [3, 1, 3]


def _dist_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    test = load_ref('lib/apis/test.py', 'ref_apis_test')
    stored = make_batches(100 + rank, dist_sizes(rank), 2, 4)
    model = StubModel(stored)
    log_vars = test.evaluate_3d(model, Loader(batch_dicts(stored), 3, 12), metrics=None, feed_batch_size=FEED_BATCH_SIZE,
                                viz_dir=VIZ_DIR, viz_step=VIZ_STEP, sample_kwargs=SAMPLE_KWARGS)
    q.put((rank, json.dumps(log_vars), model.calls))
    dist.destroy_process_group()


def main():
    out = {}
    test = load_ref('lib/apis/test.py', 'ref_apis_test')
    fid_base = sys.modules['mmgen.core.evaluation.metrics'].FID
    # --- one process
    stored = make_batches(0, [3, 3, 3, 1], 2, 4, no_test_imgs=(2,))
    model, feeds = StubModel(stored), []
    log_vars = test.evaluate_3d(model, Loader(batch_dicts(stored), 3, 10), metrics=make_metrics(fid_base, feeds),
                                feed_batch_size=FEED_BATCH_SIZE, viz_dir=VIZ_DIR, viz_step=VIZ_STEP, sample_kwargs=SAMPLE_KWARGS)
    save_stored(out, 'single', stored)
    out['single/kwargs'] = np.array(json.dumps(model.calls))
    out['single/feeds'] = np.array(json.dumps(feeds))
    out['single/log_vars'] = np.array(json.dumps({k: float(v) for k, v in log_vars.items()}))
    out['params'] = np.array(json.dumps(dict(feed_batch_size=FEED_BATCH_SIZE, viz_dir=VIZ_DIR, viz_step=VIZ_STEP,
                                             sample_kwargs=SAMPLE_KWARGS)))
    # --- world size 2 over gloo
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r, (lv, calls)) for r, lv, calls in (q.get(timeout=300) for _ in procs))
    for p in procs:
        p.join()
        assert p.exitcode == 0
    for r in range(2):
        save_stored(out, f'dist/{r}', make_batches(100 + r, dist_sizes(r), 2, 4))
        out[f'dist/{r}/log_vars_out'] = np.array(res[r][0])
        out[f'dist/{r}/kwargs'] = np.array(json.dumps(res[r][1]))
    # --- the sampler's per-rank indices
    sampler = load_ref('lib/datasets/samplers/distributed_sampler.py', 'ref_sampler')
    for n, w, spg in SAMPLER_CASES:
        for r in range(w):
            _SAMPLER_RANK.update(rank=r, world=w)
            s = sampler.DistributedSampler(list(range(n)), w, r, shuffle=False, samples_per_gpu=spg, seed=None)
            out[f'sampler/{n}_{w}_{spg}/{r}'] = np.array(list(iter(s)), np.int64)
        _SAMPLER_RANK.clear()
    path = os.path.join(HERE, 'reference_eval_v1.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes')


if __name__ == '__main__':
    main()
