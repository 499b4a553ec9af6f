"""Pins for ssdnerf_b200.runner / sharding.train_indices: the reference's OWN training-loop pieces, executed from /root/reference with
mmcv / mmgen stubbed (the stubs of make_golden_eval.py, plus mmcv's `Hook` / `HOOKS`, `build_optimizer`, `track_iter_progress` and
`MMDistributedDataParallel`, each the plain behaviour those files rely on).  Recorded:
    sampler/N_W_spg_split/e/r[_skip]   DistributedSampler(shuffle=True, seed=2021) indices of rank r in epoch e, with split_data
                                        on / off, and with skip_iter = 3 in epoch 1
    disjoint/N_W_spg_split/e/r          the same with check_batch_disjoint=True over epochs 0-3 (python's `random` seeded 7 + r)
    updater/<iter>                      the settings ModelUpdaterHook (lib/runner/hooks/model_updater.py, rsetattr) leaves on a stub
                                        model before each iteration, for the cars-uncond schedule scaled to steps [2, 4, 6]
    optim/<key>                         the parameter names build_optimizers (lib/core/optimizer/builder.py) gives each key
    mean/codes, mean/out                MeanCacheHook's input codes (TanhCode scale 2 applied to code_) and its mean code
-> tests/golden/reference_train_loop_v1.npz.  Also writes tests/golden/reference_runner_configs.json: each shipped config's runner
sections (optimizer, lr_config, checkpoint_config, log_config, custom_hooks, evaluation, total_iters, workflow, data.train,
train_dataloader), resolved by ssdnerf_b200.Config.

    python tests/golden/make_golden_train_loop.py          (needs /root/reference)
"""
import glob
import importlib.util
import json
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden_eval as MGE  # noqa: E402

REF = MGE.REF
SAMPLER_CASES = ((10, 1, 4, False), (10, 2, 4, False), (10, 3, 2, False), (10, 2, 4, True), (11, 3, 2, True), (704, 8, 8, True))
DISJOINT_CASES = ((24, 1, 4, False), (40, 2, 4, True), (60, 3, 4, False), (614, 2, 16, True))
SEED = 2021
UPDATER = dict(step=[2, 4, 6], cfgs=[{'train_cfg.extra_scene_step': 3},
                                     {'train_cfg.extra_scene_step': 1, 'diffusion.ddpm_loss.freeze_norm': True},
                                     {'train_cfg.extra_scene_step': 1, 'train_cfg.optimizer.lr': 2.5e-3,
                                      'diffusion.ddpm_loss.freeze_norm': True, 'pixel_loss.loss_weight': 10.0,
                                      'reg_loss.loss_weight': 1.5e-3}])
RUNNER_KEYS = ('optimizer', 'lr_config', 'checkpoint_config', 'log_config', 'custom_hooks', 'evaluation', 'total_iters', 'workflow')


def stub_more():
    MGE.stub_mm()

    class Registry(dict):
        def register_module(self, *a, **k):
            return lambda cls: cls

    class Hook:
        pass

    def build_optimizer(module, cfg):
        cfg = dict(cfg)
        return getattr(torch.optim, cfg.pop('type'))(module.parameters(), **cfg)

    class MMDistributedDataParallel:
        pass

    sys.modules['mmcv'].track_iter_progress = lambda x: x
    sys.modules['mmcv.runner'].build_optimizer = build_optimizer
    sys.modules['mmcv.runner'].Hook = Hook
    sys.modules['mmcv.runner'].HOOKS = Registry()
    for name in ('mmcv.runner.hooks', 'mmcv.runner.hooks.hook'):
        m = types.ModuleType(name)
        m.__path__ = []
        m.Hook, m.HOOKS = Hook, sys.modules['mmcv.runner'].HOOKS
        sys.modules[name] = m
    par = types.ModuleType('mmcv.parallel')
    par.MMDistributedDataParallel = MMDistributedDataParallel
    sys.modules['mmcv.parallel'] = par


def load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def ref_lib():
    """lib.core.utils (misc.py's rgetattr / rsetattr), lib.core.optimizer.builder and the hooks, as packages under `lib`"""
    stub_more()
    for name in ('lib', 'lib.core', 'lib.core.optimizer', 'lib.runner', 'lib.runner.hooks', 'lib.datasets'):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    misc = load('lib/core/utils/misc.py', 'lib.core.utils')
    sys.modules['lib.core'].rsetattr, sys.modules['lib.core'].rgetattr = misc.rsetattr, misc.rgetattr
    sys.modules['lib.datasets'].build_dataloader = None
    builder = load('lib/core/optimizer/builder.py', 'lib.core.optimizer.builder')
    updater = load('lib/runner/hooks/model_updater.py', 'lib.runner.hooks.model_updater')
    cache = load('lib/runner/hooks/cache.py', 'lib.runner.hooks.cache')
    sampler = load('lib/datasets/samplers/distributed_sampler.py', 'lib.datasets.samplers.distributed_sampler')
    return builder, updater, cache, sampler


class StubNeRF(torch.nn.Module):
    """the attribute paths the schedules and optimizer keys name: train_cfg (a live dict), decoder, diffusion.denoising,
    diffusion.ddpm_loss, pixel_loss, reg_loss; TanhCode(scale=2) as code_activation"""

    def __init__(self):
        from ssdnerf_b200.config import ConfigDict
        super().__init__()
        self.train_cfg = ConfigDict(extra_scene_step=15, optimizer=ConfigDict(type='Adam', lr=5e-3))
        self.decoder = torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.Linear(4, 2))
        self.diffusion = torch.nn.Module()
        self.diffusion.denoising = torch.nn.Linear(2, 2)
        self.diffusion.ddpm_loss = torch.nn.Module()
        self.diffusion.ddpm_loss.freeze_norm = False
        self.pixel_loss = torch.nn.Module()
        self.pixel_loss.loss_weight = 20.0
        self.reg_loss = torch.nn.Module()
        self.reg_loss.loss_weight = 3e-3

    @staticmethod
    def code_activation(code_):
        return torch.tanh(code_ / 2) * 2

    def get_init_density_grid(self, num_scenes, device=None):
        return torch.zeros(8 ** 3, dtype=torch.float16)

    def get_init_density_bitfield(self, num_scenes, device=None):
        return torch.zeros(8 ** 3 // 8, dtype=torch.uint8)


def updater_state(model):
    return [model.train_cfg['extra_scene_step'], model.train_cfg['optimizer']['lr'], float(model.diffusion.ddpm_loss.freeze_norm),
            model.pixel_loss.loss_weight, model.reg_loss.loss_weight]


def runner_configs():
    from ssdnerf_b200 import Config
    from make_config_fixtures import plain
    out = {}
    for path in sorted(glob.glob(os.path.join(REF, 'configs', '**', '*.py'), recursive=True)):
        cfg = Config.fromfile(path)
        if 'model' not in cfg:
            continue
        rec = {k: plain(cfg.get(k)) for k in RUNNER_KEYS}
        rec['data.train'] = plain(cfg['data']['train'])
        rec['train_dataloader'] = plain(cfg['data'].get('train_dataloader', {}))
        out[os.path.relpath(path, REF)] = rec
    return out


def main():
    builder, updater, cache, sampler = ref_lib()
    out = {}
    # --- sampler orders
    for n, w, spg, split in SAMPLER_CASES:
        for r in range(w):
            MGE._SAMPLER_RANK.update(rank=r, world=w)
            s = sampler.DistributedSampler(list(range(n)), w, r, shuffle=True, samples_per_gpu=spg, split_data=split, seed=SEED)
            for e in range(3):
                s.set_epoch(e)
                out[f'sampler/{n}_{w}_{spg}_{int(split)}/{e}/{r}'] = np.array(list(iter(s)), np.int64)
            s.set_epoch(1)
            s.skip_iter = 3
            out[f'sampler/{n}_{w}_{spg}_{int(split)}/1/{r}_skip'] = np.array(list(iter(s)), np.int64)
    # --- check_batch_disjoint: each rank's sampler over epochs 0-3, python's generator seeded 7 + rank first
    for n, w, spg, split in DISJOINT_CASES:
        for r in range(w):
            MGE._SAMPLER_RANK.update(rank=r, world=w)
            random.seed(7 + r)
            s = sampler.DistributedSampler(list(range(n)), w, r, shuffle=True, samples_per_gpu=spg, split_data=split, seed=SEED,
                                           check_batch_disjoint=True)
            for e in range(4):
                s.set_epoch(e)
                out[f'disjoint/{n}_{w}_{spg}_{int(split)}/{e}/{r}'] = np.array(list(iter(s)), np.int64)
    MGE._SAMPLER_RANK.clear()
    # --- ModelUpdaterHook
    model = StubNeRF()
    runner = types.SimpleNamespace(model=types.SimpleNamespace(module=model), iter=0, epoch=0)
    hook = updater.ModelUpdaterHook(by_epoch=False, **UPDATER)
    for it in range(8):
        runner.iter = it
        hook.before_train_iter(runner)
        out[f'updater/{it}'] = np.array(updater_state(model), np.float64)
    # --- build_optimizers key resolution
    model = StubNeRF()
    names = {id(p): n for n, p in model.named_parameters()}
    opts = builder.build_optimizers(model, dict(decoder=dict(type='Adam', lr=1e-3), diffusion=dict(type='Adam', lr=1e-4),
                                                **{'diffusion.denoising': dict(type='SGD', lr=0.1)}))
    for key, o in opts.items():
        out[f'optim/{key}'] = np.array([names[id(p)] for g in o.param_groups for p in g['params']])
    # --- MeanCacheHook's mean code
    g = torch.Generator().manual_seed(5)
    codes = [torch.randn(3, 4, 4, 4, generator=g) * 2 for _ in range(3)]
    with tempfile.TemporaryDirectory() as src, tempfile.TemporaryDirectory() as dst:
        for i, c in enumerate(codes):
            par = dict(code_=c) if i != 1 else dict(code=torch.tanh(c / 2) * 2)     # one file holds the activated code only
            torch.save(dict(param=par), os.path.join(src, f'scene{i}.pth'))
        model = StubNeRF()
        model.train_cfg['cache_load_from'] = dst
        runner = types.SimpleNamespace(model=types.SimpleNamespace(module=model, cache_loaded=True), iter=0, epoch=0, rank=0,
                                       logger=types.SimpleNamespace(info=lambda *a: None))
        dist.init_process_group('gloo', init_method=f'file://{os.path.join(dst, ".pg")}', rank=0, world_size=1)
        try:
            cache.MeanCacheHook(step=[0], load_from=src, by_epoch=False).before_train_iter(runner)
        finally:
            dist.destroy_process_group()
        files = sorted(f for f in os.listdir(dst) if f != '.pg')
        assert files == sorted(os.listdir(src))
        outs = [torch.load(os.path.join(dst, f)) for f in files]
        out['mean/order'] = np.array(os.listdir(src))
        out['mean/codes'] = np.stack([c.numpy() for c in codes])
        out['mean/out'] = outs[0]['param']['code'].numpy()
        for o in outs:
            assert torch.equal(o['param']['code'], outs[0]['param']['code'])
    np.savez_compressed(os.path.join(HERE, 'reference_train_loop_v1.npz'), **out)
    with open(os.path.join(HERE, 'reference_runner_configs.json'), 'w') as f:
        json.dump(runner_configs(), f, indent=1, sort_keys=True)


if __name__ == '__main__':
    main()
