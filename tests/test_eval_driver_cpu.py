"""The evaluation driver without a GPU: `ssdnerf_b200.evaluate_3d` replays the reference's own `evaluate_3d` (val_step kwargs, every
metric feed, the averaged log_vars; tests/golden/reference_eval_v1.npz) on one process and on a world-size-2 gloo group, the test
loader's per-rank order equals the reference's `DistributedSampler`, `--cfg-options` values parse as mmcv's `DictAction`, checkpoints
load as mmcv's `load_checkpoint`, and the evaluation plan of every shipped config equals its `evaluation` section."""
import glob
import hashlib
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from ssdnerf_b200 import evaluate_3d, test as T
from ssdnerf_b200.evaluation import SceneBatches
from ssdnerf_b200.metrics import FIDKID
from ssdnerf_b200.sharding import scene_indices

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REF = '/root/reference'


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_eval_v1.npz'))


def _stored(ref, prefix):
    out = []
    for i in range(int(ref[f'{prefix}/num_batches'])):
        b = dict(n=int(ref[f'{prefix}/{i}/n']), pred=ref[f'{prefix}/{i}/pred'], log_vars=json.loads(str(ref[f'{prefix}/{i}/log_vars'])))
        if f'{prefix}/{i}/test_imgs' in ref:
            b['test_imgs'] = ref[f'{prefix}/{i}/test_imgs']
        out.append(b)
    return out


class StubModel(torch.nn.Module):
    def __init__(self, stored):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.stored, self.calls = stored, []

    def val_step(self, data, **kwargs):
        self.calls.append(json.dumps(kwargs, sort_keys=True))
        b = self.stored[data['batch']]
        return dict(log_vars=dict(b['log_vars']), num_samples=b['n'], pred_imgs=torch.from_numpy(b['pred']))


def _batches(stored):
    return [dict(batch=i, **({'test_imgs': torch.from_numpy(b['test_imgs'])} if 'test_imgs' in b else {})) for i, b in enumerate(stored)]


def _record(feeds, name, imgs, mode):
    x = imgs.contiguous().numpy()
    feeds.append([name, mode, list(x.shape), hashlib.sha256(x.tobytes()).hexdigest()])


class FakesOnly(FIDKID):
    def __init__(self, feeds):
        super().__init__(num_images=1)
        self.feeds = feeds

    def feed(self, imgs, mode):
        _record(self.feeds, 'fakes_only', imgs, mode)


class Both:
    def __init__(self, feeds):
        self.feeds = feeds

    def feed(self, imgs, mode):
        _record(self.feeds, 'both', imgs, mode)


def test_one_process_replays_reference_evaluate_3d(ref):
    params = json.loads(str(ref['params']))
    stored = _stored(ref, 'single')
    model, feeds = StubModel(stored), []
    log_vars = evaluate_3d(model, _batches(stored), metrics=[FakesOnly(feeds), Both(feeds)], **params)
    assert model.calls == json.loads(str(ref['single/kwargs']))
    assert feeds == json.loads(str(ref['single/feeds']))
    want = json.loads(str(ref['single/log_vars']))
    assert set(log_vars) == set(want)
    for k, v in want.items():
        assert abs(float(log_vars[k]) - v) <= 1e-14 * abs(v), (k, log_vars[k], v)


def test_no_metrics_and_no_viz_dir(ref):
    stored = _stored(ref, 'single')
    model = StubModel(stored)
    evaluate_3d(model, _batches(stored), metrics=[], viz_step=2)
    assert all('viz_dir' not in json.loads(c) for c in model.calls)


def test_scene_indices_match_reference_sampler(ref):
    for key in ref.files:
        if key.startswith('sampler/'):
            case, r = key.split('/')[1:]
            n, w, spg = (int(x) for x in case.split('_'))
            assert scene_indices(n, int(r), w, spg) == ref[key].tolist(), key
    with pytest.raises(ValueError):
        scene_indices(3, 0, 4, 2)          # padding repeats the head once only: the sampler asserts here too


class _Scenes(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n, self.reads = n, []

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        self.reads.append(i)
        return dict(scene_id=i, scene_name=f'{i:04d}', test_poses=torch.full((2, 4, 4), float(i)))


@pytest.mark.parametrize('prefetch', [True, False])
def test_scene_batches_one_process(prefetch):
    ds = _Scenes(10)
    got = [b['scene_id'] for b in SceneBatches(ds, 4, 'cpu', prefetch=prefetch)]
    assert got == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
    assert ds.reads == list(range(10))
    b = next(iter(SceneBatches(ds, 3, 'cpu', prefetch=prefetch)))
    assert torch.equal(b['test_poses'][:, 0, 0, 0], torch.tensor([0.0, 1.0, 2.0]))


def test_scene_batches_prefetch_raises_reader_error():
    class Broken(_Scenes):
        def __getitem__(self, i):
            if i == 5:
                raise FileNotFoundError('scene 5')
            return super().__getitem__(i)
    it = iter(SceneBatches(Broken(8), 4, 'cpu'))
    assert next(it)['scene_id'] == [0, 1, 2, 3]
    with pytest.raises(FileNotFoundError, match='scene 5'):
        next(it)


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def _dist_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    ref = np.load(os.path.join(GOLDEN, 'reference_eval_v1.npz'))
    params = json.loads(str(ref['params']))
    stored = _stored(ref, f'dist/{rank}')
    model = StubModel(stored)
    log_vars = evaluate_3d(model, _batches(stored), metrics=None, **params)
    order = {f'{n}_{world}_{spg}': SceneBatches(_Scenes(n), spg, 'cpu').indices for n, spg in ((10, 4), (704, 8))}
    order['10_2_4_ids'] = [b['scene_id'] for b in SceneBatches(_Scenes(10), 4, 'cpu')]
    q.put((rank, log_vars, model.calls, order))
    dist.destroy_process_group()


def test_world_size_2_gloo_matches_reference(ref):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {r: rest for r, *rest in (q.get(timeout=300) for _ in procs)}
    for p in procs:
        p.join()
        assert p.exitcode == 0
    for r in range(2):
        log_vars, calls, order = res[r]
        assert log_vars == json.loads(str(ref[f'dist/{r}/log_vars_out'])), r
        assert calls == json.loads(str(ref[f'dist/{r}/kwargs']))
        assert order['10_2_4'] == ref[f'sampler/10_2_4/{r}'].tolist()
        assert order['10_2_4_ids'] == [ref[f'sampler/10_2_4/{r}'].tolist()[:4], ref[f'sampler/10_2_4/{r}'].tolist()[4:]]
        assert order['704_2_8'] == scene_indices(704, r, 2, 8)


# ------------------------------------------------------------------------------------------------------------------------ CLI
def test_cfg_options_parse_like_dictaction():
    # values as mmcv's DictAction._parse_iterable returns them
    cases = {'1': 1, '-3': -3, '0.5': 0.5, '1e-3': 1e-3, 'True': True, 'false': False, 'None': None, 'none': 'none',
             'work_dirs/x': 'work_dirs/x', '1,2': [1, 2], '[1,2,3]': [1, 2, 3], '(1,2)': (1, 2), '[(1,2),[3,4]]': [(1, 2), [3, 4]],
             "'[a, b]'": ['a', 'b'], '"(1.5,x,True)"': (1.5, 'x', True), '[]': [], '[[1],(2,)]': [[1], (2,)]}
    for text, want in cases.items():
        got = T.parse_cfg_value(text)
        assert got == want and type(got) is type(want), (text, got)
    args = T.parse_args(['c.py', 'k.pth', '--cfg-options', 'test_cfg.n_inverse_steps=3', 'data.samples_per_gpu=2',
                         'evaluation.viz_step=[1,2]', 'model.x=a=b'])
    assert args.cfg_options == {'test_cfg.n_inverse_steps': 3, 'data.samples_per_gpu': 2, 'evaluation.viz_step': [1, 2],
                                'model.x': 'a=b'}
    with pytest.raises(ValueError, match='imbalanced'):
        T.parse_cfg_value('[1,(2]')


def test_launcher_and_defaults():
    args = T.parse_args(['c.py', 'k.pth'])
    assert (args.launcher, args.seed, args.diff_seed, args.deterministic, args.data, args.cfg_options, args.gpu_id) == \
        ('none', 2021, False, False, None, None, 0)
    assert T.parse_args(['c.py', 'k.pth', '--launcher', 'pytorch', '--data', 'val_cond', 'val_uncond']).data == ['val_cond', 'val_uncond']
    for bad in ('slurm', 'mpi', 'ssh'):
        with pytest.raises(SystemExit):
            T.parse_args(['c.py', 'k.pth', '--launcher', bad])


def test_set_random_seed_seeds_python_numpy_torch():
    import random
    draws = []
    for _ in range(2):
        T.set_random_seed(7)
        draws.append((random.random(), float(np.random.rand()), float(torch.rand(1))))
    assert draws[0] == draws[1] and os.environ['PYTHONHASHSEED'] == '7'


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(2, 3)
        self.b = torch.nn.Linear(3, 1)


@pytest.mark.parametrize('layout', ['mmcv', 'ddp', 'bare'])
def test_load_checkpoint_layouts(tmp_path, layout):
    src = _Net()
    sd = src.state_dict()
    if layout == 'ddp':
        sd = {'module.' + k: v for k, v in sd.items()}
    path = tmp_path / 'iter_10.pth'
    torch.save(dict(state_dict=sd, meta=dict(iter=10, mmcv_version='1.6.0')) if layout != 'bare' else sd, path)
    dst = _Net()
    missing, unexpected = T.load_checkpoint(dst, str(path))
    assert missing == [] and unexpected == []
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v)


def test_load_checkpoint_lists_missing_and_unexpected(tmp_path, caplog):
    import logging
    sd = {k: v for k, v in _Net().state_dict().items() if not k.startswith('b.')}
    sd['ema.weight'] = torch.zeros(2)
    sd['a.bias'] = torch.zeros(5)          # wrong shape: skipped and reported
    torch.save(dict(state_dict=sd), tmp_path / 'c.pth')
    dst = _Net()
    before = dst.a.bias.detach().clone()
    logger = logging.getLogger('test_eval_driver_cpu')
    with caplog.at_level(logging.WARNING, logger='test_eval_driver_cpu'):
        missing, unexpected = T.load_checkpoint(dst, str(tmp_path / 'c.pth'), logger)
    assert sorted(missing) == ['a.bias', 'b.bias', 'b.weight'] and unexpected == ['ema.weight']
    assert torch.equal(dst.a.bias, before)
    text = caplog.text
    assert 'unexpected key in source state_dict: ema.weight' in text and 'missing keys in source state_dict' in text
    assert 'size mismatch for a.bias' in text


def test_load_checkpoint_refuses_pickled_objects(tmp_path):
    import collections
    torch.save(dict(state_dict=_Net().state_dict(), meta=collections.Counter(a=1), hook=_Net), tmp_path / 'full.pth')
    with pytest.raises(RuntimeError, match='weights_only=True'):
        T.load_checkpoint(_Net(), str(tmp_path / 'full.pth'))


def _check_plan(cfg, name):
    evals = cfg['evaluation']
    evals = [evals] if isinstance(evals, dict) else evals
    plan = T.eval_plan(cfg)
    assert len(plan) == len(evals), name
    for p, ev in zip(plan, evals):
        metrics = ev['metrics'] if isinstance(ev['metrics'], list) else [ev['metrics']]
        assert p['dataset'] == cfg['data'][ev['data']] and p['metrics'] == metrics, name
        assert (p['feed_batch_size'], p['viz_dir'], p['viz_step']) == (ev['feed_batch_size'], ev['viz_dir'], ev['viz_step']), name
        assert p['sample_kwargs'] == ev.get('sample_kwargs', {}) and p['samples_per_gpu'] == cfg['data']['samples_per_gpu'], name
        for m in metrics:
            metric = T.build_metric(m)
            assert metric.name == m['type'] and metric.num_images == m['num_images'] and metric.bgr2rgb == m['bgr2rgb']
    assert T.eval_plan(cfg, data=['nothing']) == []


def test_eval_plan_of_every_shipped_config():
    cfgs = json.loads(str(np.load(os.path.join(GOLDEN, 'reference_dataset_v1.npz'))['configs']))
    assert len(cfgs) == 24
    for name, cfg in cfgs.items():
        _check_plan(cfg, name)
    with pytest.raises(NotImplementedError, match="'IS'"):
        T.build_metric(dict(type='IS', num_images=10))


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'configs')), reason='needs the reference checkout')
def test_eval_plan_of_the_reference_config_files():
    from ssdnerf_b200.config import Config
    files = sorted(glob.glob(os.path.join(REF, 'configs', '*_cfgs', '**', '*.py'), recursive=True))
    assert len(files) == 24
    for f in files:
        _check_plan(Config.fromfile(f), f)
