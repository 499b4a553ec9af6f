"""Evaluate a checkpoint on a config's evaluation sets: the reference's tools/test.py on the package's own pieces, without mmcv / mmgen.

    python -m ssdnerf_b200.test CONFIG CHECKPOINT [--data val_cond ...] [--seed 2021] [--diff_seed] [--deterministic]
                                [--cfg-options k=v ...] [--gpu-id 0] [--launcher {none,pytorch}]

For every entry of `cfg.evaluation` (those whose `data` is listed in `--data`, when given) it builds the entry's FID / FIDKID metrics
and `cfg.data[entry.data]`, runs `evaluation.evaluate_3d` over the test loader's batches with the entry's `feed_batch_size`, `viz_dir`,
`viz_step` and `sample_kwargs`, then prints `name = value` for the metric results and the averaged `log_vars` and appends the same
lines to `<checkpoint dir>/<checkpoint stem>_eval_log.txt`.  `--launcher pytorch` reads torchrun's environment and evaluates on every
rank over NCCL.  The Inception TorchScript and the LPIPS weights are external assets and are never downloaded.
"""
import argparse
import logging
import os
import random
import re
import sys

import numpy as np
import torch
import torch.distributed as dist

from .config import Config
from .evaluation import SceneBatches, evaluate_3d
from .metrics import METRICS
from .registry import build_dataset, build_model

_LOG_FORMAT = '%(asctime)s - %(name)s - %(levelname)s - %(message)s'


# --------------------------------------------------------------------------------------------------------------------- arguments
def parse_cfg_value(val):
    """mmcv `DictAction._parse_iterable` [mmcv-memory]: `a,b`, `[a,b]` and `(a,b)` (nested, quotes and spaces stripped) become lists /
    tuples; a single value becomes an int, a float, a bool (`true` / `false`, any case), None (`None`) or stays a string."""
    val = val.strip('\'"').replace(' ', '')
    is_tuple = False
    if val.startswith('(') and val.endswith(')'):
        is_tuple, val = True, val[1:-1]
    elif val.startswith('[') and val.endswith(']'):
        val = val[1:-1]
    elif ',' not in val:
        return _parse_scalar(val)
    values = []
    while len(val) > 0:
        end = _next_comma(val)
        values.append(parse_cfg_value(val[:end]))
        val = val[end + 1:]
    return tuple(values) if is_tuple else values


def _parse_scalar(val):
    for cast in (int, float):
        try:
            return cast(val)
        except ValueError:
            pass
    if val.lower() in ('true', 'false'):
        return val.lower() == 'true'
    if val == 'None':
        return None
    return val


def _next_comma(s):
    """index of the first comma outside brackets (len(s) if none)"""
    if s.count('(') != s.count(')') or s.count('[') != s.count(']'):
        raise ValueError(f'--cfg-options: imbalanced brackets in {s!r}')
    for i, ch in enumerate(s):
        pre = s[:i]
        if ch == ',' and pre.count('(') == pre.count(')') and pre.count('[') == pre.count(']'):
            return i
    return len(s)


class DictAction(argparse.Action):
    """`key=value` pairs -> dict, values parsed by `parse_cfg_value`"""

    def __call__(self, parser, namespace, values, option_string=None):
        options = {}
        for kv in values:
            if '=' not in kv:
                parser.error(f'{option_string}: {kv!r} is not of the form key=value')
            key, val = kv.split('=', maxsplit=1)
            options[key] = parse_cfg_value(val)
        setattr(namespace, self.dest, options)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description='Test and eval a model')
    parser.add_argument('config', help='test config file path')
    parser.add_argument('checkpoint', help='checkpoint file')
    parser.add_argument('--launcher', default='none', help='job launcher: none or pytorch (torchrun); slurm and mpi are not supported')
    parser.add_argument('--gpu-id', type=int, default=0, help='id of the GPU to use (non-distributed testing only)')
    parser.add_argument('--seed', type=int, default=2021, help='random seed')
    parser.add_argument('--diff_seed', action='store_true', help='set different seeds for different ranks')
    parser.add_argument('--deterministic', action='store_true', help='set deterministic options for the cuDNN backend')
    parser.add_argument('--data', type=str, nargs='+', help='evaluate only the entries whose `data` is one of these')
    parser.add_argument('--cfg-options', nargs='+', action=DictAction,
                        help='override settings of the config: key-value pairs in xxx=yyy format, merged into the config')
    parser.add_argument('--local_rank', type=int, default=0)
    args = parser.parse_args(argv)
    if args.launcher in ('slurm', 'mpi'):
        parser.error(f'--launcher {args.launcher} is not supported (none or pytorch)')
    if args.launcher not in ('none', 'pytorch'):
        parser.error(f'--launcher: unknown launcher {args.launcher!r} (none or pytorch)')
    return args


# --------------------------------------------------------------------------------------------------------------------- set-up
def set_random_seed(seed, deterministic=False, use_rank_shift=False):
    """mmgen `set_random_seed` [mmgen-memory]: python, numpy and torch (every device), `PYTHONHASHSEED`; `use_rank_shift` adds the rank"""
    if use_rank_shift and dist.is_available() and dist.is_initialized():
        seed += dist.get_rank()
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    os.environ['PYTHONHASHSEED'] = str(seed)
    if deterministic:
        torch.backends.cudnn.deterministic = True
        torch.backends.cudnn.benchmark = False


def load_checkpoint(model, filename, logger=None):
    """mmcv `load_checkpoint(model, filename, map_location='cpu', strict=False)` [mmcv-memory]: the file's `state_dict` (or the file itself
    when it has none), a leading `module.` stripped from every key, loaded non-strictly.  Keys the model lacks, model keys the file lacks
    and shape mismatches are logged and skipped, so EMA-only files load.  The file is read with `torch.load(weights_only=True)`; a file
    that needs the full unpickler raises.  Returns (missing keys, unexpected keys)."""
    try:
        ckpt = torch.load(filename, map_location='cpu', weights_only=True)
    except Exception as e:
        raise RuntimeError(f'{filename}: cannot be loaded with torch.load(weights_only=True): {e}') from e
    state_dict = ckpt['state_dict'] if isinstance(ckpt, dict) and 'state_dict' in ckpt else ckpt
    if not isinstance(state_dict, dict):
        raise RuntimeError(f'{filename}: no state dict in the file (found {type(state_dict).__name__})')
    state_dict = {re.sub(r'^module\.', '', k): v for k, v in state_dict.items()}
    own = model.state_dict()
    mismatched = [k for k, v in state_dict.items() if k in own and tuple(own[k].shape) != tuple(v.shape)]
    msgs = [f'size mismatch for {k}: copying a param with shape {tuple(state_dict[k].shape)} from checkpoint, '
            f'the shape in current model is {tuple(own[k].shape)}.' for k in mismatched]
    for k in mismatched:
        del state_dict[k]
    missing, unexpected = model.load_state_dict(state_dict, strict=False)
    if unexpected:
        msgs.insert(0, f'unexpected key in source state_dict: {", ".join(unexpected)}')
    if missing:
        msgs.insert(1 if unexpected else 0, f'missing keys in source state_dict: {", ".join(missing)}')
    if msgs and logger is not None:
        logger.warning('The model and loaded state dict do not match exactly\n\n' + '\n'.join(msgs) + '\n')
    return list(missing), list(unexpected)


def eval_plan(cfg, data=None):
    """the evaluations tools/test.py runs for `cfg` (only those whose `data` is in `data`, when given): one dict per entry with the
    dataset dict `cfg.data[entry.data]`, the metric dicts, `feed_batch_size`, `viz_dir`, `viz_step`, `sample_kwargs` and the test
    loader's `samples_per_gpu` (`cfg.data.samples_per_gpu`, overridden by `cfg.data.test_dataloader`)"""
    evals = cfg.get('evaluation', [])
    evals = [evals] if isinstance(evals, dict) else list(evals)
    spg = dict(samples_per_gpu=cfg['data']['samples_per_gpu'], **cfg['data'].get('test_dataloader', {}))['samples_per_gpu']
    plan = []
    for ev in evals:
        if data is not None and ev['data'] not in data:
            continue
        metrics = ev['metrics']
        metrics = [metrics] if isinstance(metrics, dict) else list(metrics)
        plan.append(dict(data=ev['data'], dataset=cfg['data'][ev['data']], metrics=metrics,
                         feed_batch_size=ev.get('feed_batch_size', 32), viz_dir=ev.get('viz_dir', None), viz_step=ev.get('viz_step', 1),
                         sample_kwargs=ev.get('sample_kwargs', dict()), samples_per_gpu=spg))
    return plan


def build_metric(cfg):
    """an FID / FIDKID metric from its config dict (the metrics tools/test.py allows in distributed runs); other types raise"""
    if cfg.get('type') not in ('FID', 'FIDKID'):
        raise NotImplementedError(f'metric type {cfg.get("type")!r} is not supported (FID and FIDKID are)')
    return METRICS.build(cfg)


def _logger(log_path):
    logger = logging.getLogger('ssdnerf_b200')
    logger.setLevel(logging.INFO)
    logger.propagate = False
    handlers = [logging.StreamHandler(sys.stdout)]
    if log_path is not None:
        handlers.append(logging.FileHandler(log_path, mode='a'))
    for h in handlers:
        h.setFormatter(logging.Formatter(_LOG_FORMAT))
        logger.addHandler(h)
    return logger, handlers


def _init_dist(cfg):
    """torchrun's environment (RANK, LOCAL_RANK, WORLD_SIZE, MASTER_ADDR / PORT) -> NCCL process group, one device per local rank"""
    local_rank = int(os.environ.get('LOCAL_RANK', os.environ['RANK']))
    torch.cuda.set_device(local_rank % torch.cuda.device_count())
    dist.init_process_group(backend=cfg.get('dist_params', {}).get('backend', 'nccl'))


# --------------------------------------------------------------------------------------------------------------------- driver
def main(argv=None):
    """Runs the evaluations; returns [(data name, [each metric's results {name: value}], log_vars)] per evaluated entry (every rank
    gets the same values; only rank 0 prints and writes the log)."""
    args = parse_args(argv)
    cfg = Config.fromfile(args.config)
    if args.cfg_options is not None:
        Config.merge_options(cfg, args.cfg_options)
    distributed = args.launcher == 'pytorch'
    if distributed:
        _init_dist(cfg)
        rank = dist.get_rank()
    else:
        torch.cuda.set_device(args.gpu_id)
        rank = 0
    device = torch.device('cuda', torch.cuda.current_device())
    dirname, ckpt = os.path.split(args.checkpoint)
    log_path = os.path.join(dirname, ckpt.split('.')[0] + '_eval_log.txt') if rank == 0 else None
    logger, handlers = _logger(log_path)
    try:
        if rank == 0:
            logger.info('evaluation')
        if args.seed is not None:
            if rank == 0:
                logger.info(f'Set random seed to {args.seed}, deterministic: {args.deterministic}, use_rank_shift: {args.diff_seed}')
            set_random_seed(args.seed, deterministic=args.deterministic, use_rank_shift=args.diff_seed)
        model = build_model(cfg['model'], train_cfg=cfg.get('train_cfg'), test_cfg=cfg.get('test_cfg'))
        load_checkpoint(model, args.checkpoint, logger if rank == 0 else None)
        model = model.to(device).eval()
        out = []
        for entry in eval_plan(cfg, args.data):
            metrics = [build_metric(m) for m in entry['metrics']]
            for metric in metrics:
                metric.prepare()
            batches = SceneBatches(build_dataset(entry['dataset']), entry['samples_per_gpu'], device)
            log_vars = evaluate_3d(model, batches, metrics=metrics, feed_batch_size=entry['feed_batch_size'],
                                   viz_dir=entry['viz_dir'], viz_step=entry['viz_step'], sample_kwargs=entry['sample_kwargs'])
            results = []
            for metric in metrics:
                metric.summary()
                results.append(dict(metric._result_dict))
            if rank == 0:
                for name, val in [kv for r in results for kv in r.items()] + list(log_vars.items()):
                    logger.info(f'{name} = {val}')
            out.append((entry['data'], results, log_vars))
        return out
    finally:
        for h in handlers:
            logger.removeHandler(h)
            h.close()


if __name__ == '__main__':
    main()
