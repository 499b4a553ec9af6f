"""Real-image Inception statistics for FID / KID: the reference's tools/inception_stat.py on the package's own pieces.

    python -m ssdnerf_b200.inception_stat CONFIG [--batch-size 32]

For every evaluation of CONFIG with an `FID` / `FIDKID` metric, builds `cfg.data[eval.data]` with `num_train_imgs=0` and
`load_imgs=True` (dropping `specific_observation_idcs` and `max_num_scenes`), feeds every scene's `test_imgs * 2 - 1` through the
feature path `FIDKID.feed(..., 'reals')` uses, and writes the metric's `inception_pkl` as the reference does: `feats_np` float32,
`mean` (np.mean), `cov` (np.cov, rowvar=False), `size`, and `name`, which is the file's extension as the reference stores it.  The
Inception weights are the metric's `inception_args['inception_path']`; nothing is downloaded.
"""
import argparse
import os
import pickle

import numpy as np
import torch

from .config import Config
from .datasets import collate
from .metrics import FIDKID
from .registry import build_dataset


def fid_metrics(cfg):
    """(evaluation dict, FID / FIDKID metric dict) pairs of a config"""
    evals = cfg.get('evaluation', [])
    evals = [evals] if isinstance(evals, dict) else list(evals)
    out = []
    for ev in evals:
        metrics = ev['metrics']
        metrics = [metrics] if isinstance(metrics, dict) else metrics
        fid = None
        for m in metrics:
            if m['type'] in ('FID', 'FIDKID'):
                fid = m
        if fid is not None:
            out.append((ev, fid))
    return out


def real_features(dataset, inception_args, batch_size=32, device=None):
    """float32 [N, 2048] Inception features of every test image of `dataset`, scene by scene in order"""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    metric = FIDKID(num_images=2 ** 62, inception_args=inception_args)
    for i in range(len(dataset)):
        batch = collate([dataset[i]], device)
        imgs = batch['test_imgs'][0].permute(0, 3, 1, 2) * 2 - 1
        for chunk in imgs.split(batch_size, dim=0):
            metric.feed(chunk.contiguous(), 'reals')
    return torch.cat(metric.real_feats, 0).cpu().numpy()


def write_stats(features, pkl_path):
    d = os.path.dirname(pkl_path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(pkl_path, 'wb') as f:
        pickle.dump({'feats_np': features, 'mean': np.mean(features, axis=0), 'cov': np.cov(features, rowvar=False),
                     'size': features.shape[0], 'name': os.path.splitext(os.path.basename(pkl_path))[1]}, f)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Pre-calculate the real-image Inception statistics of a config\'s FID metrics')
    parser.add_argument('config', help='config file path')
    parser.add_argument('--batch-size', type=int, default=32, help='images per Inception call')
    args = parser.parse_args(argv)
    cfg = Config.fromfile(args.config)
    pairs = fid_metrics(cfg)
    if not pairs:
        print(f'{args.config}: no evaluation with an FID / FIDKID metric')
    for ev, metric in pairs:
        data_cfg = dict(cfg['data'][ev['data']], num_train_imgs=0, load_imgs=True)
        data_cfg.pop('specific_observation_idcs', None)
        data_cfg.pop('max_num_scenes', None)
        dataset = build_dataset(data_cfg)
        features = real_features(dataset, metric['inception_args'], args.batch_size)
        write_stats(features, metric['inception_pkl'])
        print(f'{metric["inception_pkl"]}: {features.shape[0]} features')


if __name__ == '__main__':
    main()
