"""The evaluation loop of the reference's tools/test.py and GenerativeEvalHook3D: `evaluate_3d` (lib/apis/test.py:12-73) over the test
loader's batches, and `SceneBatches`, that loader without mmcv.

`evaluate_3d` runs `val_step` per batch, passes `viz_dir` on every `viz_step`-th batch, feeds the rendered test views to the metrics
(`pred_imgs * 2 - 1` in `feed_batch_size` chunks; the real test views only to metrics other than FID / FIDKID) and averages each
`log_vars` entry over the batches with their `num_samples` as weights.  `SceneBatches` yields this rank's scenes in the loader's order,
each batch `collate`d on the device; the file reads of batch i + 1 run on a background thread while the caller works on batch i.
"""
from concurrent.futures import ThreadPoolExecutor
from copy import deepcopy

import numpy as np
import torch
import torch.distributed as dist

from .datasets import collate
from .metrics import FIDKID
from .sharding import scene_indices


def _dist_info():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class SceneBatches:
    """The test loader of tools/test.py (`shuffle=False`) over `dataset`: batches of `samples_per_gpu` scenes, collated on `device`.

    One process takes every scene in order, the last batch partial.  In a distributed run (the default process group is initialised)
    each rank takes `sharding.scene_indices(len(dataset), rank, world, samples_per_gpu)`: the sampler's padded strided share, in full
    batches.  An explicit `indices` list (the training loader's order) replaces both.  With `prefetch`, one background thread reads the next batch's items (`dataset[i]`: the scenes' file bytes) while the
    caller runs the current one; `collate` (the PNG decode on the device) stays on the caller's thread and current stream, in order."""

    def __init__(self, dataset, samples_per_gpu, device=None, prefetch=True, indices=None):
        self.dataset, self.samples_per_gpu, self.device, self.prefetch = dataset, samples_per_gpu, device, prefetch
        rank, world = _dist_info()
        if indices is not None:
            self.indices = list(indices)
        elif dist.is_available() and dist.is_initialized():
            self.indices = scene_indices(len(dataset), rank, world, samples_per_gpu)
        else:
            self.indices = list(range(len(dataset)))

    def _groups(self):
        spg = self.samples_per_gpu
        return [self.indices[i:i + spg] for i in range(0, len(self.indices), spg)]

    def _read(self, ids):
        return [self.dataset[i] for i in ids]

    def __iter__(self):
        groups = self._groups()
        if not self.prefetch:
            for ids in groups:
                yield collate(self._read(ids), self.device)
            return
        with ThreadPoolExecutor(max_workers=1) as pool:
            pending = pool.submit(self._read, groups[0]) if groups else None
            for k in range(len(groups)):
                items = pending.result()
                if k + 1 < len(groups):
                    pending = pool.submit(self._read, groups[k + 1])
                yield collate(items, self.device)


def _feeds_reals(metric):
    """lib/apis/test.py:44: mmgen's FID / IS (and FIDKID, an FID) take generated images only"""
    return not isinstance(metric, FIDKID)


def _model_device(model):
    """mmgen `get_module_device` [mmgen-memory]: the device of the model's first parameter"""
    try:
        return next(model.parameters()).device
    except StopIteration:
        raise ValueError('evaluate_3d: the model has no parameters to take the device from') from None


def evaluate_3d(model, batches, metrics=None, feed_batch_size=32, viz_dir=None, viz_step=1, sample_kwargs={}):
    """lib/apis/test.py:12-73 over `batches` (an iterable of collated batches, e.g. `SceneBatches`): returns the `log_vars` averaged
    over every scene this run evaluated.  One process: `np.average` with the batches' `num_samples` as weights.  Distributed: float32
    sums of `num_samples`-weighted values all-reduced over the ranks, as the reference does.  Metrics are fed but not summarised."""
    rank, _ = _dist_info()
    log_vars, batch_size_list = {}, []
    for i, data in enumerate(batches):
        kwargs = deepcopy(sample_kwargs)
        if viz_dir is not None and i % viz_step == 0:
            kwargs.update(viz_dir=viz_dir)
        outputs = model.val_step(data, show_pbar=rank == 0, **kwargs)
        for k, v in outputs['log_vars'].items():
            log_vars.setdefault(k, []).append(v)
        batch_size_list.append(outputs['num_samples'])
        if metrics:
            pred = outputs['pred_imgs']
            pred_imgs = pred.reshape(-1, *pred.shape[2:]).split(feed_batch_size, dim=0)
            real_imgs = None
            for metric in metrics:
                if 'test_imgs' in data and _feeds_reals(metric) and real_imgs is None:
                    real = data['test_imgs'].permute(0, 1, 4, 2, 3)
                    real_imgs = real.reshape(-1, *real.shape[2:]).split(feed_batch_size, dim=0)
                for batch_id, batch_imgs in enumerate(pred_imgs):
                    metric.feed(batch_imgs * 2 - 1, 'fakes')
                    if _feeds_reals(metric) and real_imgs is not None:
                        metric.feed(real_imgs[batch_id] * 2 - 1, 'reals')
    if dist.is_available() and dist.is_initialized():
        device = _model_device(model)
        weights = torch.tensor(batch_size_list, dtype=torch.float, device=device)
        weight_sum = torch.sum(weights)
        dist.all_reduce(weight_sum, op=dist.ReduceOp.SUM)
        for k, v in log_vars.items():
            weighted = torch.sum(torch.tensor(v, dtype=torch.float, device=device) * weights)
            dist.all_reduce(weighted, op=dist.ReduceOp.SUM)
            log_vars[k] = float(weighted / weight_sum)
    else:
        for k, v in log_vars.items():
            log_vars[k] = np.average(v, weights=batch_size_list)
    return log_vars
