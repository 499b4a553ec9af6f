"""The training runner without a GPU: sampler orders, ModelUpdaterHook settings, optimizer keys and MeanCacheHook's mean equal the
reference's own code (tests/golden/reference_train_loop_v1.npz, make_golden_train_loop.py); LR schedules of every shipped
`lr_config`; the EMA momentum schedule; checkpoint layout, `max_keep_ckpts`, `weights_only` loading and resume bookkeeping with a
pure-torch stub model; CLI parsing and refusals; `Config.dump`; and the sampler on a world-size-2 gloo group."""
import json
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FIX = np.load(os.path.join(GOLDEN, 'reference_train_loop_v1.npz'))
RUNNER_CFGS = json.load(open(os.path.join(GOLDEN, 'reference_runner_configs.json')))
SAMPLER_CASES = ((10, 1, 4, False), (10, 2, 4, False), (10, 3, 2, False), (10, 2, 4, True), (11, 3, 2, True), (704, 8, 8, True))
DISJOINT_CASES = ((24, 1, 4, False), (40, 2, 4, True), (60, 3, 4, False), (614, 2, 16, True))


class StubNeRF(torch.nn.Module):
    """the attribute paths of make_golden_train_loop.StubNeRF"""

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


# --------------------------------------------------------------------------------------------------------------------- fixture
@pytest.mark.parametrize('case', SAMPLER_CASES)
def test_sampler_orders_equal_the_reference(case):
    from ssdnerf_b200.sharding import train_indices
    n, w, spg, split = case
    for r in range(w):
        for e in range(3):
            got = train_indices(n, e, 2021, r, w, spg, split)
            assert got == FIX[f'sampler/{n}_{w}_{spg}_{int(split)}/{e}/{r}'].tolist(), (case, r, e)
        got = train_indices(n, 1, 2021, r, w, spg, split, skip_iter=3)
        assert got == FIX[f'sampler/{n}_{w}_{spg}_{int(split)}/1/{r}_skip'].tolist()


@pytest.mark.parametrize('case', DISJOINT_CASES)
def test_check_batch_disjoint_orders_equal_the_reference(case):
    """each rank's epochs 0-3 with check_batch_disjoint, python's generator seeded as the fixture seeded it"""
    import random
    from ssdnerf_b200.sharding import disjoint_first_batch, train_indices
    n, w, spg, split = case
    for r in range(w):
        random.seed(7 + r)
        last = set()
        for e in range(4):
            got, last = disjoint_first_batch(train_indices(n, e, 2021, r, w, spg, split), spg, last)
            assert got == FIX[f'disjoint/{n}_{w}_{spg}_{int(split)}/{e}/{r}'].tolist(), (case, r, e)


def test_check_batch_disjoint_redraws_and_refuses():
    import random
    from ssdnerf_b200.runner import TrainLoader
    from ssdnerf_b200.sharding import disjoint_first_batch, train_indices
    redrawn = 0
    for k in FIX.files:
        if k.startswith('disjoint/'):
            _, case, e, r = k.split('/')
            n, w, spg, split = (int(x) for x in case.split('_'))
            redrawn += FIX[k].tolist() != train_indices(n, int(e), 2021, int(r), w, spg, bool(split))
    assert redrawn >= 4                             # the fixture exercises the redraw, not only the check
    with pytest.raises(RuntimeError, match='too small'):
        disjoint_first_batch([0, 1, 2, 3, 4, 5], 2, {0, 1, 2, 3, 4, 5})
    with pytest.raises(RuntimeError, match='too small'):
        disjoint_first_batch([0, 1, 2, 3, 3, 4], 2, set())
    # one process: every epoch's first batch is disjoint from the previous epoch's last
    random.seed(0)
    torch.manual_seed(0)
    loader = TrainLoader(list(range(24)), 4, check_batch_disjoint=True)
    prev = None
    for e in range(8):
        loader.epoch = e
        order = loader.epoch_order()
        if prev is not None:
            assert set(order[:4]).isdisjoint(prev[-4:]), e
        prev = order


def test_unknown_train_dataloader_options_raise(tmp_path):
    from ssdnerf_b200.runner import train_model
    cfg = dict(data=dict(samples_per_gpu=2, train_dataloader=dict(split_data=True, drop_last=True)), work_dir=str(tmp_path))
    with pytest.raises(NotImplementedError, match='drop_last'):
        train_model(torch.nn.Linear(1, 1), list(range(4)), cfg)


def test_model_updater_settings_equal_the_reference():
    import types
    from ssdnerf_b200.runner import ModelUpdaterHook
    model = StubNeRF()
    hook = ModelUpdaterHook(step=[2, 4, 6], by_epoch=False, cfgs=[
        {'train_cfg.extra_scene_step': 3}, {'train_cfg.extra_scene_step': 1, 'diffusion.ddpm_loss.freeze_norm': True},
        {'train_cfg.extra_scene_step': 1, 'train_cfg.optimizer.lr': 2.5e-3, 'diffusion.ddpm_loss.freeze_norm': True,
         'pixel_loss.loss_weight': 10.0, 'reg_loss.loss_weight': 1.5e-3}])
    runner = types.SimpleNamespace(model=model, iter=0)
    for it in range(8):
        runner.iter = it
        hook.before_train_iter(runner)
        got = [model.train_cfg['extra_scene_step'], model.train_cfg['optimizer']['lr'], float(model.diffusion.ddpm_loss.freeze_norm),
               model.pixel_loss.loss_weight, model.reg_loss.loss_weight]
        assert got == FIX[f'updater/{it}'].tolist(), it


def test_rsetattr_sets_items_of_plain_dicts():
    from ssdnerf_b200.runner import rsetattr
    m = torch.nn.Module()
    m.train_cfg = dict(optimizer=dict(lr=1.0))
    rsetattr(m, 'train_cfg.optimizer.lr', 2.0)
    rsetattr(m, 'train_cfg.extra_scene_step', 3)
    assert m.train_cfg == dict(optimizer=dict(lr=2.0), extra_scene_step=3)


def test_optimizer_keys_equal_the_reference():
    from ssdnerf_b200.runner import build_optimizers
    model = StubNeRF()
    names = {id(p): n for n, p in model.named_parameters()}
    opts = build_optimizers(model, dict(decoder=dict(type='Adam', lr=1e-3), diffusion=dict(type='Adam', lr=1e-4),
                                        **{'diffusion.denoising': dict(type='SGD', lr=0.1)}))
    assert sorted(opts) == ['decoder', 'diffusion', 'diffusion.denoising']
    for key, o in opts.items():
        assert [names[id(p)] for g in o.param_groups for p in g['params']] == FIX[f'optim/{key}'].tolist()
    assert isinstance(opts['diffusion.denoising'], torch.optim.SGD)
    with pytest.raises(ValueError, match='torch.optim'):
        build_optimizers(model, dict(decoder=dict(type='NoSuchOptimizer', lr=1.0)))


def test_mean_cache_equals_the_reference(tmp_path):
    from ssdnerf_b200.runner import mean_cache
    codes = torch.from_numpy(FIX['mean/codes'])
    for i, c in enumerate(codes):
        par = dict(code_=c) if i != 1 else dict(code=torch.tanh(c / 2) * 2)
        torch.save(dict(param=par), tmp_path / f'scene{i}.pth')
    files, mean = mean_cache(str(tmp_path), StubNeRF.code_activation)
    assert sorted(files) == ['scene0.pth', 'scene1.pth', 'scene2.pth']
    torch.testing.assert_close(mean, torch.from_numpy(FIX['mean/out']), rtol=0, atol=1e-6)   # summation order follows listdir


# --------------------------------------------------------------------------------------------------------------------- schedules
def _mmcv_lr(cfg, it, base):
    """mmcv LrUpdaterHook by iteration, restated"""
    if cfg['policy'] == 'Fixed':
        lr = base
    else:
        step = cfg['step']
        exp = it // step if isinstance(step, int) else next((i for i, s in enumerate(step) if it < s), len(step))
        lr = base * cfg.get('gamma', 0.1) ** exp
    if cfg.get('warmup') == 'linear' and it < cfg['warmup_iters']:
        lr = lr * (1 - (1 - it / cfg['warmup_iters']) * (1 - cfg['warmup_ratio']))
    return lr


@pytest.mark.parametrize('name', sorted(RUNNER_CFGS))
def test_lr_schedule_of_every_shipped_config(name):
    import types
    from ssdnerf_b200.runner import LrUpdaterHook, build_optimizers
    rc = RUNNER_CFGS[name]
    model = StubNeRF()
    optim_cfg = {k: v for k, v in rc['optimizer'].items() if k in ('decoder', 'diffusion')}
    assert optim_cfg, name
    opts = build_optimizers(model, optim_cfg)
    hook = LrUpdaterHook(**rc['lr_config'])
    runner = types.SimpleNamespace(optimizer=opts, iter=0)
    hook.before_run(runner)
    cfg = dict(rc['lr_config'])
    cfg['policy'] = cfg['policy'].title() if cfg['policy'] == cfg['policy'].lower() else cfg['policy']
    its = sorted({0, 1, cfg.get('warmup_iters', 0) - 1, cfg.get('warmup_iters', 0), 1000, rc['total_iters'] - 1}
                 | {s + d for s in (cfg.get('step') or []) for d in (-1, 0)})
    for it in its:
        runner.iter = it
        hook.before_train_iter(runner)
        for k, o in opts.items():
            assert o.param_groups[0]['lr'] == pytest.approx(_mmcv_lr(cfg, it, optim_cfg[k]['lr']), rel=1e-12), (name, k, it)


def test_lr_hook_refusals():
    from ssdnerf_b200.runner import LrUpdaterHook
    with pytest.raises(NotImplementedError, match='policy'):
        LrUpdaterHook(policy='cosine')
    with pytest.raises(NotImplementedError, match='warmup'):
        LrUpdaterHook(policy='Fixed', warmup='exp')


def test_ema_momentum_schedule():
    from ssdnerf_b200.ema import rampup_momentum
    cfg = dict(ema_kimg=4, ema_rampup=0.05, batch_size=16, eps=1e-8)
    assert rampup_momentum(0, **cfg) == 0.5 ** (16 / 0.8)
    assert rampup_momentum(99, **cfg) == 0.5 ** (16 / (1600 * 0.05))
    assert rampup_momentum(4999, **cfg) == 0.5 ** (16 / 4000)       # 80000 images * 0.05 = 4000: the cap is reached
    assert rampup_momentum(10 ** 6, **cfg) == 0.5 ** (16 / 4000)
    ms = [rampup_momentum(i, **cfg) for i in range(0, 6000, 50)]
    assert all(a <= b for a, b in zip(ms, ms[1:]))
    assert np.float32(rampup_momentum(7, **cfg)) == np.float32(0.5 ** (16.0 / (8 * 16 * 0.05)))


def test_ema_hook_refusals():
    from ssdnerf_b200.ema import ExponentialMovingAverageHook as H
    ok = dict(module_keys=('diffusion_ema',), interval=1, momentum_policy='rampup')
    H(**ok)
    with pytest.raises(NotImplementedError, match='interp_mode'):
        H(**dict(ok, interp_mode='slerp'))
    with pytest.raises(NotImplementedError, match='momentum_policy'):
        H(**dict(ok, momentum_policy='fixed'))
    with pytest.raises(NotImplementedError, match='start_iter'):
        H(**dict(ok, start_iter=5))
    with pytest.raises(ValueError, match='_ema'):
        H(**dict(ok, module_keys=('diffusion',)))


def test_ema_hook_names_non_fp32_state(monkeypatch):
    from ssdnerf_b200 import ema as E
    model = torch.nn.Module()
    model.net = torch.nn.Linear(2, 2)
    model.net.register_buffer('count', torch.zeros(1, dtype=torch.int64))
    model.net_ema = torch.nn.Linear(2, 2)
    model.net_ema.register_buffer('count', torch.zeros(1, dtype=torch.int64))
    monkeypatch.setattr(E, 'ema_lerp_', lambda *a, **k: None)
    hook = E.ExponentialMovingAverageHook(('net_ema',), interval=1, momentum_policy='rampup')
    with pytest.raises(ValueError, match='net.count'):
        hook.update(model, 0)


# --------------------------------------------------------------------------------------------------------------------- runner
class PureTorchModel(torch.nn.Module):
    """a stub whose train_step is one SGD-able torch step on a quadratic; records the running_status it is given"""

    def __init__(self):
        super().__init__()
        self.decoder = torch.nn.Linear(3, 1)
        self.register_buffer('seen', torch.zeros(1))
        self.status = []

    def train_step(self, data, optimizer, running_status=None):
        self.status.append(dict(running_status))
        optimizer['decoder'].zero_grad()
        loss = (self.decoder(data['x']) - 1).square().mean()
        loss.backward()
        optimizer['decoder'].step()
        self.seen += 1
        return dict(log_vars=dict(loss=float(loss.detach())), num_samples=data['x'].shape[0])


class ListLoader:
    """endless batches of a fixed list, the epoch advancing per pass (mmcv's IterLoader)"""

    def __init__(self, n=4):
        g = torch.Generator().manual_seed(0)
        self.batches = [dict(x=torch.randn(2, 3, generator=g)) for _ in range(n)]
        self.epoch, self.pos = 0, 0

    def __len__(self):
        return len(self.batches)

    def __next__(self):
        if self.pos == len(self.batches):
            self.epoch, self.pos = self.epoch + 1, 0
        self.pos += 1
        return self.batches[self.pos - 1]


def _runner(work_dir, max_keep=2):
    from ssdnerf_b200.runner import CheckpointHook, LoggerHook, LrUpdaterHook, Runner, build_optimizers
    torch.manual_seed(0)
    model = PureTorchModel()
    opts = build_optimizers(model, dict(decoder=dict(type='Adam', lr=1e-2)))
    r = Runner(model, opts, work_dir, meta=dict(seed=2021, exp_name='stub.py', config='x = 1\n'), timestamp='t0')
    r.register_hook(LoggerHook(interval=2), 'VERY_LOW')
    r.register_hook(CheckpointHook(interval=2, max_keep_ckpts=max_keep, out_dir=os.path.join(work_dir, 'ckpt')), 'NORMAL')
    r.register_hook(LrUpdaterHook(policy='Fixed', warmup='linear', warmup_iters=3, warmup_ratio=0.1), 'VERY_HIGH')
    return r


def test_checkpoint_layout_max_keep_and_weights_only(tmp_path):
    from ssdnerf_b200.test import load_checkpoint
    work = str(tmp_path / 'exp')
    r = _runner(work)
    r.run(ListLoader(), [('train', 2)], 7)
    ck = os.path.join(work, 'ckpt', 'exp')
    assert sorted(os.listdir(ck)) == ['iter_4.pth', 'iter_6.pth', 'iter_7.pth', 'latest.pth']      # iter_2 deleted; save_last
    assert os.path.realpath(os.path.join(ck, 'latest.pth')) == os.path.realpath(os.path.join(ck, 'iter_7.pth'))
    ckpt = torch.load(os.path.join(ck, 'iter_6.pth'), weights_only=True)
    assert set(ckpt) == {'meta', 'state_dict', 'optimizer'}
    assert ckpt['meta']['iter'] == 6 and ckpt['meta']['epoch'] == 2 and ckpt['meta']['seed'] == 2021 and ckpt['meta']['exp_name'] == 'stub.py'
    assert set(ckpt['meta']) >= {'iter', 'epoch', 'seed', 'exp_name', 'config', 'time'}
    assert set(ckpt['state_dict']) == {'decoder.weight', 'decoder.bias', 'seen'} and float(ckpt['state_dict']['seen']) == 6
    assert all(not v.is_cuda for v in ckpt['state_dict'].values())
    assert set(ckpt['optimizer']) == {'decoder'}
    fresh = PureTorchModel()
    assert load_checkpoint(fresh, os.path.join(ck, 'iter_6.pth')) == ([], [])
    recs = [json.loads(line) for line in open(os.path.join(work, 't0.log.json'))]
    assert [x['iter'] for x in recs] == [2, 4, 6, 7]
    assert recs[0]['lr']['decoder'] == pytest.approx(1e-2 * (1 - (1 - 1 / 3) * 0.9))
    assert recs[1]['lr']['decoder'] == 1e-2


def test_resume_restores_model_optimizer_and_iteration(tmp_path):
    work = str(tmp_path / 'exp')
    full = _runner(work, max_keep=-1)
    full.run(ListLoader(), [('train', 2)], 6)
    r = _runner(str(tmp_path / 'exp2'), max_keep=-1)
    r.resume(os.path.join(work, 'ckpt', 'exp', 'iter_4.pth'))
    assert r.iter == 4 and r.epoch == 0 and float(r.model.seen) == 4
    assert int(r.optimizer['decoder'].state_dict()['state'][0]['step']) == 4
    loader = ListLoader()
    for _ in range(4):                      # the data position the first run had reached
        next(loader)
    r.run(loader, [('train', 2)], 6)
    assert [s['iteration'] for s in r.model.status] == [4, 5]
    for k, v in full.model.state_dict().items():
        assert torch.equal(v, r.model.state_dict()[k]), k


def test_eval_hook_keeps_the_best_checkpoint(tmp_path):
    """mmgen's save_best_ckpt default: best_fid_iter_<n>.pth follows the lowest fid; the file it replaces is removed"""
    from ssdnerf_b200.runner import GenerativeEvalHook3D
    work = str(tmp_path / 'exp')
    r = _runner(work)
    hook = GenerativeEvalHook3D(dataloader=[], interval=1, data='val_cond')
    assert hook.save_best_ckpt and hook.best_metric == ['fid']
    for it, fid in ((0, 10.0), (1, 12.0), (2, 5.0), (3, 5.0)):
        r.iter = it
        hook.save_best(r, 'fid', fid)
        hook.save_best(r, 'test_psnr', 30.0)               # not a best_metric: no file
    assert sorted(f for f in os.listdir(work) if f.startswith('best_')) == ['best_fid_iter_3.pth']
    ckpt = torch.load(os.path.join(work, 'best_fid_iter_3.pth'), weights_only=True)
    assert ckpt['meta']['iter'] == 3
    psnr = GenerativeEvalHook3D(dataloader=[], best_metric='test_psnr')
    for it, v in ((0, 20.0), (1, 25.0)):
        r.iter = it
        psnr.save_best(r, 'test_psnr', v)
    assert os.path.exists(os.path.join(work, 'best_test_psnr_iter_2.pth'))
    assert not os.path.exists(os.path.join(work, 'best_test_psnr_iter_1.pth'))
    with pytest.raises(ValueError, match='best_metric'):
        GenerativeEvalHook3D(dataloader=[], best_metric='accuracy')
    GenerativeEvalHook3D(dataloader=[], save_best_ckpt=False, best_metric='accuracy')


def test_hook_priority_order(tmp_path):
    from ssdnerf_b200.runner import Runner
    r = Runner(torch.nn.Linear(1, 1), {}, str(tmp_path / 'unused'))
    names = []
    for name, prio in (('lr', 'VERY_HIGH'), ('ckpt', 'NORMAL'), ('logger', 'VERY_LOW'), ('eval', 'LOW'), ('ema', 'VERY_HIGH'),
                       ('savecache', 'NORMAL'), ('updater', 'NORMAL')):
        h = type(name, (), {})()
        h.name = name
        r.register_hook(h, prio)
    names = [h.name for h in r.hooks]
    assert names == ['lr', 'ema', 'ckpt', 'savecache', 'updater', 'eval', 'logger']


def test_workflow_refusal(tmp_path):
    r = _runner(str(tmp_path / 'w'))
    with pytest.raises(NotImplementedError, match='workflow'):
        r.run(ListLoader(), [('train', 1), ('val', 1)], 2)


# --------------------------------------------------------------------------------------------------------------------- CLI / config
def test_cli_parsing_and_refusals(tmp_path):
    from ssdnerf_b200 import train as T
    a = T.parse_args(['c.py', '--work-dir', 'w', '--resume-from', 'r.pth', '--no-validate', '--gpu-id', '1', '--seed', '3', '--diff_seed',
                      '--deterministic', '--cfg-options', 'a.b=1', 'c=[1,2]', '--launcher', 'none'])
    assert (a.work_dir, a.resume_from, a.no_validate, a.gpu_id, a.seed, a.diff_seed, a.deterministic) == ('w', 'r.pth', True, 1, 3, True, True)
    assert a.cfg_options == {'a.b': 1, 'c': [1, 2]}
    assert T.parse_args(['c.py']).seed == 2021
    for launcher in ('slurm', 'mpi', 'other'):
        with pytest.raises(SystemExit):
            T.parse_args(['c.py', '--launcher', launcher])
    cfg = tmp_path / 'c.py'
    for extra in ('fp16 = dict(loss_scale=512.)', "apex_amp = dict(mode='gradient')"):
        cfg.write_text(f'model = dict(type="DiffusionNeRF")\n{extra}\n')
        with pytest.raises(NotImplementedError):
            T.main([str(cfg)])
    a = T.parse_args([str(cfg)])
    assert T.resolve_work_dir(a, {}) == os.path.join('./work_dirs', 'c')
    assert T.resolve_work_dir(a, {'work_dir': 'cfgdir'}) == 'cfgdir'
    assert T.resolve_work_dir(T.parse_args([str(cfg), '--work-dir', 'cli']), {'work_dir': 'cfgdir'}) == 'cli'


def test_config_dump_round_trip(tmp_path):
    from ssdnerf_b200.config import Config
    ref = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    src = tmp_path / 'src.py'
    rc = RUNNER_CFGS['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    src.write_text(f'model = {ref["model"]!r}\ntrain_cfg = {ref["train_cfg"]!r}\ncustom_hooks = {rc["custom_hooks"]!r}\n'
                   f'workflow = [("train", 5000)]\nmomentum = (0.9, 0.99)\nload_from = None\ngpu_ids = range(1)\n')
    cfg = Config.fromfile(str(src))
    Config.merge_options(cfg, {'train_cfg.extra_scene_step': 3})
    Config.dump(cfg, str(tmp_path / 'out.py'))
    back = Config.fromfile(str(tmp_path / 'out.py'))
    expect = dict(cfg, gpu_ids=[0])
    assert back == expect
    assert back['workflow'] == [('train', 5000)] and back['momentum'] == (0.9, 0.99)


# --------------------------------------------------------------------------------------------------------------------- gloo
def _gloo_worker(rank, world, init, out_dir):
    import torch.distributed as dist
    from ssdnerf_b200.runner import TrainLoader
    dist.init_process_group('gloo', init_method=init, rank=rank, world_size=world)
    try:
        rec = {}
        for n, spg, split in ((10, 4, False), (10, 4, True)):
            loader = TrainLoader(list(range(n)), spg, seed=2021, split_data=split)
            rec[f'{n}_{spg}_{int(split)}'] = dict(len=len(loader), orders=[loader.indices(e) for e in range(3)])
        import random
        random.seed(7 + rank)
        loader = TrainLoader(list(range(40)), 4, seed=2021, split_data=True, check_batch_disjoint=True)
        rec['disjoint'] = []
        for e in range(4):
            loader.epoch = e
            rec['disjoint'].append(loader.epoch_order())
        json.dump(rec, open(os.path.join(out_dir, f'{rank}.json'), 'w'))
    finally:
        dist.destroy_process_group()


def test_world_size_two_sampler(tmp_path):
    import torch.multiprocessing as mp
    init = f'file://{tmp_path / "pg"}'
    mp.spawn(_gloo_worker, args=(2, init, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        rec = json.load(open(tmp_path / f'{r}.json'))
        assert rec.pop('disjoint') == [FIX[f'disjoint/40_2_4_1/{e}/{r}'].tolist() for e in range(4)]
        for key, got in rec.items():
            n, spg, split = (int(x) for x in key.split('_'))
            assert got['orders'] == [FIX[f'sampler/{n}_2_{spg}_{split}/{e}/{r}'].tolist() for e in range(3)]
            assert got['len'] == -(-len(got['orders'][0]) // spg)


# --------------------------------------------------------------------------------------------------------------------- C ABI
def test_ema_tensor_struct_matches_header(tmp_path):
    """the ctypes mirror of `ssdnerf_ema_tensor` has the host compiler's sizeof and offsetof for the header"""
    import ctypes
    import subprocess
    from ssdnerf_b200 import _lib as N
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ssdnerf_b200.h"', 'int main(void) {',
             '    printf("%zu\\n", sizeof(ssdnerf_ema_tensor));']
    expect = [ctypes.sizeof(N.EmaTensor)]
    for name, _ in N.EmaTensor._fields_:
        lines.append(f'    printf("%zu\\n", offsetof(ssdnerf_ema_tensor, {name}));')
        expect.append(getattr(N.EmaTensor, name).offset)
    lines += ['    return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines) + '\n')
    subprocess.run(['cc', '-I', os.path.join(root, 'include'), '-o', str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == expect


def test_ema_entry_point_validates_on_the_host():
    """NULL tables and pointers and non-finite momenta are refused before anything is enqueued; count 0 is a no-op"""
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    t = (N.EmaTensor * 2)()
    t[0].ema, t[0].src, t[0].n, t[0].trainable = 1 << 20, 1 << 21, 16, 1
    t[1].ema, t[1].src, t[1].n = None, 1 << 22, 8
    assert L.ssdnerf_ema_lerp_f32(None, 0, 0.5, 0.0, None) == 0
    assert L.ssdnerf_ema_lerp_f32(None, 1, 0.5, 0.0, None) == -2 and b'NULL' in L.ssdnerf_last_error()
    assert L.ssdnerf_ema_lerp_f32(t, 2, 0.5, 0.0, None) == -2 and b'tensor 1' in L.ssdnerf_last_error()
    for m, mn in ((float('nan'), 0.0), (0.5, float('inf'))):
        assert L.ssdnerf_ema_lerp_f32(t, 1, m, mn, None) == -2 and b'not finite' in L.ssdnerf_last_error()
    t[0].ema = (1 << 20) + 2
    assert L.ssdnerf_ema_lerp_f32(t, 1, 0.5, 0.0, None) == -2 and b'aligned' in L.ssdnerf_last_error()
