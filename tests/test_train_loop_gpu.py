"""Training from a config on the GPU: the fused EMA kernel against torch's own arithmetic, the EMA hook against the modules that
render and sample through it, and `python -m ssdnerf_b200.train` end to end on synthetic SRN scenes (tests.test_eval_driver_gpu's
tree writer) with configs built from the shipped cars configs."""
import glob
import json
import os

import pytest
import torch

from tests.test_eval_driver_gpu import write_srn_tree

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _ref_cfg(name):
    return json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))[f'configs/paper_cfgs/{name}.py']


def _runner_cfg(name):
    return json.load(open(os.path.join(GOLDEN, 'reference_runner_configs.json')))[f'configs/paper_cfgs/{name}.py']


def _torch_lerp(ema, src, m):
    """mmgen's lerp as torch evaluates it: three element-wise kernels, m a Python float"""
    return src + (ema - src) * m


def _bits(t):
    return t.contiguous().view(torch.int32)


def _cars_model(test_over=None):
    import ssdnerf_b200 as S
    c = _ref_cfg('ssdnerf_cars_uncond')
    return S.build_model(c['model'], train_cfg=dict(c['train_cfg']), test_cfg=dict(c['test_cfg'], **(test_over or {}))).cuda()


def _perturb(module, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.no_grad():
        for t in module.state_dict().values():
            if t.dtype == torch.float32:
                t.add_(torch.randn(t.shape, generator=g, device='cuda') * 0.01)


def test_kernel_equals_torch_over_the_cars_denoiser_state():
    from ssdnerf_b200.ema import ema_lerp_, rampup_momentum
    model = _cars_model()
    _perturb(model.diffusion, 1)
    src = model.diffusion.state_dict(keep_vars=True)
    ema = model.diffusion_ema.state_dict(keep_vars=True)
    keys = list(src)
    assert len(keys) > 400
    for it in (0, 7, 5000):
        m = rampup_momentum(it, ema_kimg=4, ema_rampup=0.05, batch_size=16, eps=1e-8)
        expect = [_torch_lerp(ema[k].detach(), src[k].detach(), m if src[k].requires_grad else 0.0) for k in keys]
        before = torch.cuda.memory_allocated()
        ema_lerp_([ema[k] for k in keys], [src[k] for k in keys], [src[k].requires_grad for k in keys], m, 0.0)
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == before
        for k, e in zip(keys, expect):
            assert torch.equal(_bits(ema[k].detach()), _bits(e)), (it, k)


@pytest.mark.parametrize('offset', [0, 1, 2, 3])
def test_kernel_odd_lengths_offsets_and_special_values(offset):
    from ssdnerf_b200.ema import ema_lerp_
    g = torch.Generator(device='cuda').manual_seed(offset)
    sizes = [1, 3, 5, 7, 4095, 4096, 4097, 12345, 1 << 20]
    base_e = [torch.randn(n + 8, generator=g, device='cuda') for n in sizes]
    base_s = [torch.randn(n + 8, generator=g, device='cuda') for n in sizes]
    # special values at the head, middle and tail of every tensor
    specials = torch.tensor([float('nan'), float('inf'), -float('inf'), 0.0, -0.0, 1e-45, 3e38], device='cuda')
    for e, s in zip(base_e, base_s):
        idx = torch.randint(0, e.numel(), (14,), generator=g, device='cuda')
        e[idx[:7]] = specials
        s[idx[7:]] = specials
    # src at the same offset as ema (float4 path after a scalar head of (4 - offset) % 4 elements) and at another one (scalar path)
    for so, m, mn in [(so, m, mn) for so in (offset, (offset + 1) % 4) for m, mn in ((0.999, 0.0), (0.0, 0.5), (0.5, 0.0))]:
        ema = [b[offset:offset + n] for b, n in zip(base_e, sizes)]
        src = [b[so:so + n] for b, n in zip(base_s, sizes)]
        trainable = [i % 2 == 0 for i in range(len(sizes))]
        expect = [_torch_lerp(e.clone(), s, m if tr else mn) for e, s, tr in zip(ema, src, trainable)]
        untouched = [torch.cat([b[:offset], b[offset + n:]]).clone() for b, n in zip(base_e, sizes)]
        ema_lerp_(ema, src, trainable, m, mn)
        for i, (e, x) in enumerate(zip(ema, expect)):
            assert torch.equal(_bits(e), _bits(x)), (offset, so, m, sizes[i])
        for b, n, u in zip(base_e, sizes, untouched):
            assert torch.equal(_bits(torch.cat([b[:offset], b[offset + n:]])), _bits(u))
    # m = 0 with an infinite EMA gives NaN, as torch's (inf - s) * 0 does
    e, s = torch.full((5,), float('inf'), device='cuda'), torch.ones(5, device='cuda')
    x = _torch_lerp(e.clone(), s, 0.0)
    ema_lerp_([e], [s], [True], 0.0)
    assert torch.isnan(x).all() and torch.equal(_bits(e), _bits(x))


def test_kernel_argument_errors():
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200.ema import ema_lerp_
    t = torch.zeros(4, device='cuda')
    with pytest.raises(N.SSDNeRFNativeError, match='not finite'):
        ema_lerp_([t], [t.clone()], [True], float('nan'))
    with pytest.raises(ValueError, match='fp32'):
        ema_lerp_([t.half()], [t.half()], [True], 0.5)
    ema_lerp_([], [], [], 0.5)                                  # no-op


def test_ema_hook_refreshes_the_modules_that_sample_and_render():
    """after one hook call a DDIM chain of diffusion_ema agrees with that of a fresh module loaded with the same state (to the
    sampler's run-to-run round-off) and no longer with the chain on the old weights, and the decoder's packed blob equals the fresh
    module's (the kernel's writes do not bump Parameter._version)"""
    from ssdnerf_b200.ema import ExponentialMovingAverageHook
    model = _cars_model(dict(num_timesteps=3))
    noise = torch.randn(2, 18, 128, 128, generator=torch.Generator(device='cuda').manual_seed(3), device='cuda')
    with torch.no_grad():
        stale = model.diffusion_ema.ddim_sample(noise.clone())  # captures a graph on the old weights
        blob_old = model.decoder_ema.packed_blob().clone()
    _perturb(model.diffusion, 2)
    _perturb(model.decoder, 4)
    hook = ExponentialMovingAverageHook(('diffusion_ema', 'decoder_ema'), interval=1, momentum_policy='rampup',
                                        momentum_cfg=dict(ema_kimg=4, ema_rampup=0.05, batch_size=16, eps=1e-8))
    hook.update(model, 0)
    with torch.no_grad():
        got = model.diffusion_ema.ddim_sample(noise.clone())
        fresh = _cars_model(dict(num_timesteps=3))
        fresh.load_state_dict(model.state_dict())
        want = fresh.diffusion_ema.ddim_sample(noise.clone())
        err, moved = float((got - want).abs().max()), float((stale - want).abs().max())
        assert err < 5e-3 and moved > 20 * err, (err, moved)
        assert not torch.equal(model.decoder_ema.packed_blob(), blob_old)
        assert torch.equal(model.decoder_ema.packed_blob(), fresh.decoder_ema.packed_blob())


# --------------------------------------------------------------------------------------------------------------------- main()
RES, VIEWS, SCENES = 32, 6, 4


def _write_train_config(path, name, tree, work_dir, code_dir, total_iters, over=None):
    c, r = _ref_cfg(name), _runner_cfg(name)
    model = dict(c['model'], cache_size=SCENES if c['model'].get('cache_size', 0) else 0)
    train_cfg = dict(c['train_cfg'], n_inverse_rays=1024, n_decoder_rays=1024)
    if 'cache_load_from' in train_cfg:
        train_cfg['cache_load_from'] = code_dir
    test_cfg = dict(c['test_cfg'], img_size=(RES, RES), num_timesteps=2)
    train = dict(r['data.train'], data_prefix=tree)
    train.pop('cache_path', None)
    if 'code_dir' in train:
        train['code_dir'] = code_dir
    cfg = dict(model=model, train_cfg=train_cfg, test_cfg=test_cfg, optimizer=r['optimizer'],
               data=dict(samples_per_gpu=2, workers_per_gpu=1, train=train, train_dataloader=r['train_dataloader']),
               lr_config=dict(r['lr_config'], warmup_iters=4), checkpoint_config=dict(r['checkpoint_config'], interval=3),
               log_config=dict(r['log_config'], interval=1), total_iters=total_iters, workflow=[('train', 3)],
               custom_hooks=[dict(h, out_dir=code_dir, viz_dir=None) if h['type'] == 'SaveCacheHook' else h
                             for h in r['custom_hooks'] if h['type'] != 'ModelUpdaterHook'],
               work_dir=work_dir, resume_from=None, load_from=None, dist_params=dict(backend='nccl'))
    cfg.update(over or {})
    with open(path, 'w') as f:
        for k, v in cfg.items():
            f.write(f'{k} = {v!r}\n')


def _json_log(work_dir):
    recs = []
    for p in sorted(glob.glob(os.path.join(work_dir, '*.log.json'))):
        recs += [json.loads(line) for line in open(p)]
    return recs


def test_main_single_stage_checkpoints_resume_and_ema(tmp_path, monkeypatch):
    import ssdnerf_b200 as S
    from ssdnerf_b200 import ema as E
    from ssdnerf_b200 import train as T
    from ssdnerf_b200.test import load_checkpoint
    from ssdnerf_b200.evaluation import SceneBatches, evaluate_3d
    tree, work, code = str(tmp_path / 'srn'), str(tmp_path / 'work'), str(tmp_path / 'code')
    os.makedirs(code)
    write_srn_tree(tree, SCENES, VIEWS, RES)
    cfg_path = str(tmp_path / 'ssdnerf_cars_uncond.py')
    _write_train_config(cfg_path, 'ssdnerf_cars_uncond', tree, work, code, total_iters=6)

    # record every EMA step's inputs to check the weights against the formula
    snaps = []
    orig_update = E.ExponentialMovingAverageHook.update

    def update(self, model, iteration):
        before = {k: v.detach().clone() for k, v in model.decoder_ema.state_dict().items()}
        src = {k: (v.detach().clone(), v.requires_grad) for k, v in model.decoder.state_dict(keep_vars=True).items()}
        m = orig_update(self, model, iteration)
        snaps.append((before, src, m))
        return m
    monkeypatch.setattr(E.ExponentialMovingAverageHook, 'update', update)

    runner = T.main([cfg_path, '--no-validate'])
    assert runner.iter == 6
    ck = os.path.join(work, 'ckpt', 'work')
    assert sorted(os.listdir(ck)) == ['iter_3.pth', 'iter_6.pth', 'latest.pth']
    assert os.path.exists(os.path.join(work, 'ssdnerf_cars_uncond.py'))
    assert len(os.listdir(code)) == SCENES
    recs = _json_log(work)
    assert [r['iter'] for r in recs] == [1, 2, 3, 4, 5, 6]
    for r in recs:
        it = r['iter'] - 1
        for name, base in (('diffusion', 1e-4), ('decoder', 1e-3)):
            want = base * (1 - (1 - it / 4) * (1 - 0.001)) if it < 4 else base
            assert r['lr'][name] == pytest.approx(want, rel=1e-12)
        assert all(torch.isfinite(torch.tensor(v)) for k, v in r.items() if k.startswith('loss'))
    assert len(snaps) == 6
    for before, src, m in snaps:
        assert 0 < m < 1
    last_before, last_src, last_m = snaps[-1]
    for k, (v, tr) in last_src.items():
        want = last_src[k][0] + (last_before[k] - v) * (last_m if tr else 0.0)
        assert torch.equal(runner.model.decoder_ema.state_dict()[k], want), k

    # the checkpoint loads into a fresh model with nothing missing or unexpected, and evaluates
    c = S.Config.fromfile(cfg_path)
    fresh = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg'])
    missing, unexpected = load_checkpoint(fresh, os.path.join(ck, 'iter_6.pth'))
    assert missing == [] and unexpected == []
    fresh = fresh.cuda().eval()
    ds = S.build_dataset(dict(type='ShapeNetSRN', data_prefix=tree, load_imgs=False, num_test_imgs=2, scene_id_as_name=True))
    log_vars = evaluate_3d(fresh, SceneBatches(ds, 2, torch.device('cuda')), metrics=[])
    assert isinstance(log_vars, dict)

    # resuming from iter_3 continues with iteration 4 on the saved optimizer state
    saved = torch.load(os.path.join(ck, 'iter_3.pth'), weights_only=True)
    assert saved['meta']['iter'] == 3 and saved['meta']['seed'] == 2021
    work2 = str(tmp_path / 'work2')
    runner2 = T.main([cfg_path, '--no-validate', '--resume-from', os.path.join(ck, 'iter_3.pth'), '--work-dir', work2])
    assert runner2.iter == 6
    assert [r['iter'] for r in _json_log(work2)] == [4, 5, 6]
    st = runner2.optimizer['diffusion'].state_dict()['state']
    assert int(st[0]['step']) == 6


def test_main_stage1_cache_round_trip_and_stage2(tmp_path):
    from ssdnerf_b200 import train as T
    tree, code = str(tmp_path / 'srn'), str(tmp_path / 'code')
    os.makedirs(code)
    write_srn_tree(tree, SCENES, VIEWS, RES)
    cfg1 = str(tmp_path / 'stage1_cars_recons16v.py')
    _write_train_config(cfg1, 'stage1_cars_recons16v', tree, str(tmp_path / 'w1'), code, total_iters=3)
    r1 = T.main([cfg1, '--no-validate'])
    files = sorted(os.listdir(code))
    assert len(files) == SCENES
    saved = {f: torch.load(os.path.join(code, f), weights_only=True) for f in files}
    # a new model reads the cache files back through cache_load_from
    model = r1.model
    model.scene_cache.loaded = False
    model.scene_cache.entries = {i: None for i in range(SCENES)}
    model.load_cache(dict(scene_id=[0]))
    for i, f in enumerate(files):
        assert torch.equal(model.scene_cache.entries[i]['param']['code_'], saved[f]['param']['code_'])

    cfg2 = str(tmp_path / 'stage2_cars_uncond.py')
    _write_train_config(cfg2, 'stage2_cars_uncond', tree, str(tmp_path / 'w2'), code, total_iters=3)
    r2 = T.main([cfg2, '--no-validate'])
    assert r2.iter == 3
    for k, v in r2.model.decoder.state_dict().items():
        assert torch.equal(v, r2.model.decoder_ema.state_dict()[k]), k
    recs = _json_log(str(tmp_path / 'w2'))
    assert len(recs) == 3 and all(set(r['lr']) == {'diffusion'} for r in recs)
