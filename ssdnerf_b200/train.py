"""Train a model from a config: the reference's tools/train.py on the package's own runner (`runner.train_model`), without mmcv / mmgen.

    python -m ssdnerf_b200.train CONFIG [--work-dir DIR] [--resume-from CKPT] [--no-validate] [--gpu-id 0] [--seed 2021]
                                 [--diff_seed] [--deterministic] [--cfg-options k=v ...] [--launcher {none,pytorch}]

The work directory is `--work-dir`, else the config's `work_dir`, else `./work_dirs/<config name>`.  It receives the merged config
(`<config file name>`, readable by `Config.fromfile`), the text log `<timestamp>.log` and its `.log.json` twin, the checkpoints
under `ckpt/<work dir name>/` and, when tensorboard imports, `tf_logs/`.  `--launcher pytorch` reads torchrun's environment and
trains on every rank over NCCL; `slurm` and `mpi` are not supported.
"""
import argparse
import os
import time

import torch

from .config import Config
from .registry import build_dataset, build_model
from .runner import train_model
from .test import DictAction, _init_dist, _logger, set_random_seed


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description='Train a model')
    parser.add_argument('config', help='train config file path')
    parser.add_argument('--work-dir', help='the dir to save logs and models')
    parser.add_argument('--resume-from', help='the checkpoint file to resume from')
    parser.add_argument('--no-validate', action='store_true', help='do not evaluate during training')
    parser.add_argument('--gpu-id', type=int, default=0, help='id of the GPU to use (non-distributed training only)')
    parser.add_argument('--seed', type=int, default=2021, help='random seed')
    parser.add_argument('--diff_seed', action='store_true', help='set different seeds for different ranks')
    parser.add_argument('--deterministic', action='store_true', help='set deterministic options for the cuDNN backend')
    parser.add_argument('--cfg-options', nargs='+', action=DictAction,
                        help='override settings of the config: key-value pairs in xxx=yyy format, merged into the config')
    parser.add_argument('--launcher', default='none', help='job launcher: none or pytorch (torchrun); slurm and mpi are not supported')
    parser.add_argument('--local_rank', type=int, default=0)
    args = parser.parse_args(argv)
    if args.launcher in ('slurm', 'mpi'):
        parser.error(f'--launcher {args.launcher} is not supported (none or pytorch)')
    if args.launcher not in ('none', 'pytorch'):
        parser.error(f'--launcher: unknown launcher {args.launcher!r} (none or pytorch)')
    return args


def resolve_work_dir(args, cfg):
    """tools/train.py: the command line, then the config, then `./work_dirs/<config file stem>`"""
    if args.work_dir is not None:
        return args.work_dir
    if cfg.get('work_dir', None) is not None:
        return cfg['work_dir']
    return os.path.join('./work_dirs', os.path.splitext(os.path.basename(args.config))[0])


def main(argv=None):
    """Trains as the config says; returns the runner (its `iter`, `epoch`, `log_buffer` and `work_dir`)."""
    args = parse_args(argv)
    cfg = Config.fromfile(args.config)
    if args.cfg_options is not None:
        Config.merge_options(cfg, args.cfg_options)
    for key in ('apex_amp', 'fp16'):
        if cfg.get(key, None):
            raise NotImplementedError(f'{key} is not supported')
    if cfg.get('cudnn_benchmark', False):
        torch.backends.cudnn.benchmark = True
    cfg['work_dir'] = resolve_work_dir(args, cfg)
    if args.resume_from is not None:
        cfg['resume_from'] = args.resume_from
    distributed = args.launcher == 'pytorch'
    if distributed:
        _init_dist(cfg)
        rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
        cfg['gpu_ids'] = list(range(world))
    else:
        torch.cuda.set_device(args.gpu_id)
        rank, cfg['gpu_ids'] = 0, [args.gpu_id]
    device = torch.device('cuda', torch.cuda.current_device())

    os.makedirs(os.path.abspath(cfg['work_dir']), exist_ok=True)
    if rank == 0:
        Config.dump(cfg, os.path.join(cfg['work_dir'], os.path.basename(args.config)))
    timestamp = time.strftime('%Y%m%d_%H%M%S', time.localtime())
    logger, handlers = _logger(os.path.join(cfg['work_dir'], f'{timestamp}.log') if rank == 0 else None)
    try:
        config_text = open(os.path.join(cfg['work_dir'], os.path.basename(args.config))).read() if rank == 0 else ''
        meta = dict(config=config_text)
        if rank == 0:
            logger.info(f'Distributed training: {distributed}')
            logger.info(f'Config:\n{config_text}')
        if args.seed is not None:
            if rank == 0:
                logger.info(f'Set random seed to {args.seed}, deterministic: {args.deterministic}, use_rank_shift: {args.diff_seed}')
            set_random_seed(args.seed, deterministic=args.deterministic, use_rank_shift=args.diff_seed)
        cfg['seed'] = args.seed
        meta.update(seed=args.seed, exp_name=os.path.basename(args.config))
        model = build_model(cfg['model'], train_cfg=cfg.get('train_cfg'), test_cfg=cfg.get('test_cfg')).to(device)
        dataset = build_dataset(cfg['data']['train'])
        return train_model(model, dataset, cfg, distributed=distributed, validate=not args.no_validate, timestamp=timestamp, meta=meta,
                           logger=logger, device=device)
    finally:
        for h in handlers:
            logger.removeHandler(h)
            h.close()


if __name__ == '__main__':
    main()
