"""The training runner of the reference's tools/train.py -> lib/apis/train.py:train_model, without mmcv / mmgen: an iteration-based
runner (mmcv `IterBasedRunner` / mmgen `DynamicIterBasedRunner` with `pass_training_status=True` [mmcv-memory, mmgen-memory]) and
the hooks the shipped training configs name, run in mmcv's priority order.

Each iteration: `before_train_iter` hooks -> `model.train_step(batch, optimizers, running_status=dict(iteration=, epoch=))` -> the
log buffer takes `log_vars` weighted by `num_samples` -> `after_train_iter` hooks, until `total_iters`.  Hooks by priority (ties in
registration order): LR (VERY_HIGH), EMA (VERY_HIGH), checkpoint / SaveCache / ModelUpdater / DirCopy / MeanCache (NORMAL),
evaluation (LOW), loggers (VERY_LOW).
"""
import datetime
import json
import logging
import os
import shutil
import time
import warnings

import numpy as np
import torch
import torch.distributed as dist

from .ema import ExponentialMovingAverageHook
from .evaluation import SceneBatches, _dist_info, evaluate_3d
from .nerf import rgetattr, rsetattr
from .sharding import disjoint_first_batch, train_indices

PRIORITIES = dict(HIGHEST=0, VERY_HIGH=10, HIGH=30, ABOVE_NORMAL=40, NORMAL=50, BELOW_NORMAL=60, LOW=70, VERY_LOW=90, LOWEST=100)


# --------------------------------------------------------------------------------------------------------------------- optimizers
def build_optimizers(model, cfgs):
    """lib/core/optimizer/builder.py: a dict of dicts gives one `torch.optim.<type>` per key over `rgetattr(model, key)`'s
    parameters (e.g. `diffusion`, `decoder`); a single dict gives one optimizer over the whole model"""
    def build(module, cfg):
        cfg = dict(cfg)
        kind = cfg.pop('type')
        if not hasattr(torch.optim, kind):
            raise ValueError(f'optimizer type {kind!r} is not in torch.optim')
        return getattr(torch.optim, kind)(module.parameters(), **cfg)
    model = getattr(model, 'module', model)
    if all(isinstance(v, dict) for v in cfgs.values()):
        return {key: build(rgetattr(model, key), cfg) for key, cfg in cfgs.items()}
    return build(model, cfgs)


# --------------------------------------------------------------------------------------------------------------------- data
class TrainLoader:
    """The training loader of lib/datasets/builder.py behind mmcv's `IterLoader`: endless batches of `samples_per_gpu` scenes,
    collated on `device`, the epoch advancing each time the order runs out.  One process takes `torch.utils.data.RandomSampler`'s
    order (what `DataLoader(shuffle=True)` draws, from torch's global generator); a distributed run takes the reference's
    `DistributedSampler` order (`sharding.train_indices`, seeded `seed + epoch`, `split_data` as configured).  The last batch of an
    epoch may be partial.  With `check_batch_disjoint` each epoch's first batch is kept disjoint from the previous epoch's last
    (`sharding.disjoint_first_batch`); the reference's one-process loader ignores the option, here it applies there too, because a
    configuration that writes scene files back while training (`save_dir` = the dataset's `code_dir`) needs it with any number of
    processes.  Batches are read by `SceneBatches`' prefetch thread."""

    def __init__(self, dataset, samples_per_gpu, device=None, seed=0, split_data=False, check_batch_disjoint=False, prefetch=True):
        self.dataset, self.samples_per_gpu, self.device, self.prefetch = dataset, samples_per_gpu, device, prefetch
        self.seed, self.split_data, self.check_batch_disjoint = seed if seed is not None else 0, split_data, check_batch_disjoint
        self.last_batch = set()
        self.rank, self.world_size = _dist_info()
        self.distributed = dist.is_available() and dist.is_initialized()
        self.epoch, self.skip_iter = 0, 0
        self._it = None

    def indices(self, epoch):
        if self.distributed:
            return train_indices(len(self.dataset), epoch, self.seed, self.rank, self.world_size, self.samples_per_gpu,
                                 self.split_data)
        return list(torch.utils.data.RandomSampler(range(len(self.dataset))))

    def __len__(self):
        if self.distributed:
            return -(-len(train_indices(len(self.dataset), 0, self.seed, self.rank, self.world_size, self.samples_per_gpu,
                                        self.split_data)) // self.samples_per_gpu)
        return -(-len(self.dataset) // self.samples_per_gpu)

    def set_epoch(self, epoch):
        self.epoch = epoch

    def epoch_order(self):
        """the scene order of the current epoch, as the loader will read it (consumes `skip_iter` and updates `last_batch`)"""
        ids = self.indices(self.epoch)
        if self.check_batch_disjoint:
            ids, self.last_batch = disjoint_first_batch(ids, self.samples_per_gpu, self.last_batch)
        ids = ids[self.skip_iter:]
        self.skip_iter = 0
        return ids

    def _start(self):
        ids = self.epoch_order()
        return iter(SceneBatches(self.dataset, self.samples_per_gpu, self.device, prefetch=self.prefetch, indices=ids))

    def __next__(self):
        if self._it is None:
            self._it = self._start()
        try:
            return next(self._it)
        except StopIteration:
            self.epoch += 1
            self._it = self._start()
            return next(self._it)


class LogBuffer:
    """mmcv `LogBuffer`: per-iteration values and counts; `average(n)` fills `output` with the count-weighted means of the last n"""

    def __init__(self):
        self.val_history, self.n_history, self.output, self.ready = {}, {}, {}, False

    def update(self, vars, count=1):
        for k, v in vars.items():
            self.val_history.setdefault(k, []).append(float(v))
            self.n_history.setdefault(k, []).append(count)

    def average(self, n=0):
        for k in self.val_history:
            vals, nums = np.array(self.val_history[k][-n:]), np.array(self.n_history[k][-n:])
            self.output[k] = float(np.sum(vals * nums) / np.sum(nums))
        self.ready = True

    def clear_output(self):
        self.output, self.ready = {}, False


# --------------------------------------------------------------------------------------------------------------------- runner
class Runner:
    """Iteration-based runner.  `model` has `train_step(batch, optimizers, running_status)`; `optimizer` is the dict of
    `build_optimizers`; `meta` goes into every checkpoint."""

    def __init__(self, model, optimizer, work_dir, logger=None, meta=None, timestamp=None):
        self.model, self.optimizer, self.work_dir, self.meta = model, optimizer, os.path.abspath(work_dir), meta
        os.makedirs(self.work_dir, exist_ok=True)
        self.logger = logger or logging.getLogger('ssdnerf_b200')
        self.timestamp = timestamp or time.strftime('%Y%m%d_%H%M%S', time.localtime())
        self.rank, self.world_size = _dist_info()
        self.iter, self.epoch, self.inner_iter, self.max_iters = 0, 0, 0, 0
        self.hooks, self.log_buffer, self.data_loader, self.outputs = [], LogBuffer(), None, None

    def register_hook(self, hook, priority='NORMAL'):
        p = PRIORITIES[priority.upper()] if isinstance(priority, str) else int(priority)
        hook.priority_value = p
        i = len(self.hooks)
        while i > 0 and self.hooks[i - 1].priority_value > p:
            i -= 1
        self.hooks.insert(i, hook)

    def call_hook(self, name):
        for hook in self.hooks:
            fn = getattr(hook, name, None)
            if fn is not None:
                fn(self)

    def current_lr(self):
        return {k: [g['lr'] for g in o.param_groups] for k, o in self.optimizer.items()}

    def is_last_iter(self):
        return self.iter + 1 == self.max_iters

    def every_n_iters(self, n):
        return (self.iter + 1) % n == 0 if n > 0 else False

    def run(self, data_loader, workflow, max_iters):
        """mmcv `IterBasedRunner.run` for the one workflow every training config uses, `[('train', n)]`"""
        if len(workflow) != 1 or workflow[0][0] != 'train':
            raise NotImplementedError(f'workflow {workflow!r} is not supported: only [("train", n)] is')
        self.data_loader, self.max_iters = data_loader, max_iters
        self.call_hook('before_run')
        self.logger.info(f'workflow: {workflow}, max: {max_iters} iters')
        self.model.train()
        while self.iter < max_iters:
            self.train_iter()
        self.call_hook('after_run')

    def train_iter(self):
        t0 = time.time()
        batch = next(self.data_loader)
        self.epoch = self.data_loader.epoch
        self.data_time = time.time() - t0
        self.call_hook('before_train_iter')
        outputs = self.model.train_step(batch, self.optimizer, running_status=dict(iteration=self.iter, epoch=self.epoch))
        if not isinstance(outputs, dict):
            raise TypeError('model.train_step() must return a dict')
        if 'log_vars' in outputs:
            self.log_buffer.update(outputs['log_vars'], outputs['num_samples'])
        self.outputs = outputs
        self.log_buffer.update(dict(time=time.time() - t0, data_time=self.data_time))
        self.call_hook('after_train_iter')
        self.inner_iter += 1
        self.iter += 1

    # -- checkpoints
    def save_checkpoint(self, out_dir, filename_tmpl='iter_{}.pth', save_optimizer=True, create_symlink=True):
        """`<out_dir>/iter_{n}.pth` after n completed iterations and `latest.pth` beside it: dict(meta=dict(iter=n, epoch, seed,
        exp_name, config, time), state_dict=<CPU tensors, no `module.` prefix>, optimizer={name: state_dict}), readable by
        `torch.load(weights_only=True)`.  `meta['iter']` counts completed iterations, so a resumed run continues with the next;
        `meta['epoch']` is the current epoch plus one, as mmcv's iteration runner stores it (`resume` subtracts the one)."""
        meta = dict(self.meta or {})
        meta.update(iter=self.iter + 1, epoch=self.epoch + 1, time=time.asctime())
        model = getattr(self.model, 'module', self.model)
        ckpt = dict(meta=meta, state_dict={k: v.detach().cpu() for k, v in model.state_dict().items()})
        if save_optimizer:
            ckpt['optimizer'] = {k: _to_cpu(o.state_dict()) for k, o in self.optimizer.items()}
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, filename_tmpl.format(self.iter + 1))
        torch.save(ckpt, path)
        if create_symlink:
            dst = os.path.join(out_dir, 'latest.pth')
            if os.path.lexists(dst):
                os.remove(dst)
            try:
                os.symlink(os.path.basename(path), dst)
            except OSError:
                shutil.copy(path, dst)
        return path

    def load_checkpoint(self, filename):
        from .test import load_checkpoint
        return load_checkpoint(getattr(self.model, 'module', self.model), filename, self.logger)

    def resume(self, filename):
        """the model, every optimizer's state and the iteration / epoch of a `save_checkpoint` file"""
        self.load_checkpoint(filename)
        ckpt = torch.load(filename, map_location='cpu', weights_only=True)
        for k, o in self.optimizer.items():
            if k not in ckpt.get('optimizer', {}):
                raise KeyError(f'{filename}: no state for optimizer {k!r}')
            o.load_state_dict(ckpt['optimizer'][k])
        self.iter = self.inner_iter = int(ckpt['meta']['iter'])
        self.epoch = int(ckpt['meta']['epoch']) - 1
        self.logger.info(f'resumed from epoch: {self.epoch}, iter {self.iter}')


def _to_cpu(x):
    if torch.is_tensor(x):
        return x.detach().cpu()
    if isinstance(x, dict):
        return {k: _to_cpu(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_to_cpu(v) for v in x)
    return x


# --------------------------------------------------------------------------------------------------------------------- mmcv hooks
class LrUpdaterHook:
    """mmcv `LrUpdaterHook` by iteration [mmcv-memory] for every runner optimizer (not the per-scene code optimizers): policy
    `Fixed` (the base lr) or `step` (`base * gamma ** (number of milestones in `step` passed)`, `step` an int gives a period), and
    `warmup='linear'`: `regular * (1 - (1 - it / warmup_iters) * (1 - warmup_ratio))` for it < warmup_iters."""

    def __init__(self, policy, warmup=None, warmup_iters=0, warmup_ratio=0.1, by_epoch=False, step=None, gamma=0.1, min_lr=None,
                 warmup_by_epoch=False):
        policy = policy.title() if policy == policy.lower() else policy
        if policy not in ('Fixed', 'Step'):
            raise NotImplementedError(f'lr policy {policy!r} is not supported (Fixed and step are)')
        if warmup not in (None, 'linear'):
            raise NotImplementedError(f'lr warmup {warmup!r} is not supported (linear is)')
        if by_epoch or warmup_by_epoch:
            raise NotImplementedError('lr updates by epoch are not supported: the runner counts iterations')
        if policy == 'Step' and step is None:
            raise ValueError('the step lr policy needs `step`')
        self.policy, self.warmup, self.warmup_iters, self.warmup_ratio = policy, warmup, warmup_iters, warmup_ratio
        self.step, self.gamma, self.min_lr = step, gamma, min_lr
        self.base_lr = {}

    def get_lr(self, it, base_lr):
        if self.policy == 'Fixed':
            return base_lr
        if isinstance(self.step, int):
            exp = it // self.step
        else:
            exp = len(self.step)
            for i, s in enumerate(self.step):
                if it < s:
                    exp = i
                    break
        lr = base_lr * self.gamma ** exp
        return max(lr, self.min_lr) if self.min_lr is not None else lr

    def lrs(self, it):
        """{optimizer name: [lr per param group]} at iteration `it` (0-based)"""
        regular = {k: [self.get_lr(it, b) for b in base] for k, base in self.base_lr.items()}
        if self.warmup is None or it >= self.warmup_iters:
            return regular
        k = (1 - it / self.warmup_iters) * (1 - self.warmup_ratio)
        return {name: [lr * (1 - k) for lr in lrs] for name, lrs in regular.items()}

    def before_run(self, runner):
        for name, o in runner.optimizer.items():
            for g in o.param_groups:
                g.setdefault('initial_lr', g['lr'])
            self.base_lr[name] = [g['initial_lr'] for g in o.param_groups]

    def before_train_iter(self, runner):
        for name, lrs in self.lrs(runner.iter).items():
            for g, lr in zip(runner.optimizer[name].param_groups, lrs):
                g['lr'] = lr


class CheckpointHook:
    """mmcv `CheckpointHook` by iteration: every `interval` iterations (and after the last one with `save_last`) the runner's
    checkpoint goes to `<out_dir>/<basename(work_dir)>/`; with `max_keep_ckpts > 0` older `iter_*.pth` are deleted"""

    def __init__(self, interval=-1, by_epoch=False, save_optimizer=True, out_dir=None, max_keep_ckpts=-1, save_last=True, **kwargs):
        if by_epoch:
            raise NotImplementedError('checkpoints by epoch are not supported: the runner counts iterations')
        unknown = set(kwargs) - {'meta', 'sync_buffer', 'filename_tmpl', 'create_symlink'}
        if unknown:
            raise TypeError(f'CheckpointHook: unsupported arguments {sorted(unknown)}')
        self.interval, self.save_optimizer, self.out_dir = interval, save_optimizer, out_dir
        self.max_keep_ckpts, self.save_last = max_keep_ckpts, save_last
        self.filename_tmpl = kwargs.get('filename_tmpl', 'iter_{}.pth')
        self.create_symlink = kwargs.get('create_symlink', True)

    def before_run(self, runner):
        if not self.out_dir:
            self.out_dir = runner.work_dir
        if os.path.abspath(self.out_dir) != runner.work_dir:
            self.out_dir = os.path.join(self.out_dir, os.path.basename(runner.work_dir.rstrip(os.sep)))

    def after_train_iter(self, runner):
        if not (runner.every_n_iters(self.interval) or (self.save_last and runner.is_last_iter())):
            return
        if runner.rank != 0:
            return
        runner.logger.info(f'Saving checkpoint at {runner.iter + 1} iterations')
        runner.save_checkpoint(self.out_dir, self.filename_tmpl, self.save_optimizer, self.create_symlink)
        if self.max_keep_ckpts > 0:
            current = runner.iter + 1
            for step in range(current - self.max_keep_ckpts * self.interval, 0, -self.interval):
                path = os.path.join(self.out_dir, self.filename_tmpl.format(step))
                if not os.path.exists(path):
                    break
                os.remove(path)


class LoggerHook:
    """mmcv's `TextLoggerHook` and `TensorboardLoggerHook` over one log buffer: every `interval` iterations (and when an evaluation
    left results) the averaged log vars, one lr per optimizer, the iteration time and the peak device memory go to the console,
    `<work_dir>/<timestamp>.log`, `<work_dir>/<timestamp>.log.json` (one dict per line) and, when `torch.utils.tensorboard`
    imports, `<work_dir>/tf_logs`"""

    def __init__(self, interval=10, text=True, tensorboard=False):
        self.interval, self.text, self.tensorboard = interval, text, tensorboard
        self.writer, self.json_path, self.start = None, None, None

    def before_run(self, runner):
        self.start, self.start_iter = time.time(), runner.iter
        if self.text and runner.rank == 0:
            self.json_path = os.path.join(runner.work_dir, f'{runner.timestamp}.log.json')
        if self.tensorboard and runner.rank == 0:
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.writer = SummaryWriter(os.path.join(runner.work_dir, 'tf_logs'))
            except ImportError as e:
                warnings.warn(f'TensorboardLoggerHook: torch.utils.tensorboard does not import ({e}); no tensorboard logs are written')

    def after_train_iter(self, runner):
        buf = runner.log_buffer
        if runner.every_n_iters(self.interval) or runner.is_last_iter():
            buf.average(self.interval)
        if buf.ready:
            if runner.rank == 0:
                self.log(runner, buf.output)
            buf.clear_output()

    def log(self, runner, out):
        lrs = {k: v[0] for k, v in runner.current_lr().items()}
        record = dict(mode='train', epoch=runner.epoch + 1, iter=runner.iter + 1, lr=lrs)
        if torch.cuda.is_available() and torch.cuda.is_initialized():
            record['memory'] = int(torch.cuda.max_memory_allocated() // (1024 * 1024))
            torch.cuda.reset_peak_memory_stats()
        record.update(out)
        if self.text:
            done = runner.iter + 1 - self.start_iter
            eta = (time.time() - self.start) / max(done, 1) * (runner.max_iters - runner.iter - 1)
            items = [f'lr_{k}: {v:.3e}' for k, v in lrs.items()] + [f'eta: {datetime.timedelta(seconds=int(eta))}']
            items += [f'{k}: {v:.4f}' if isinstance(v, float) else f'{k}: {v}' for k, v in record.items()
                      if k not in ('mode', 'epoch', 'iter', 'lr')]
            runner.logger.info(f'Iter [{runner.iter + 1}/{runner.max_iters}]\t' + ', '.join(items))
            with open(self.json_path, 'a') as f:
                f.write(json.dumps(record) + '\n')
        if self.writer is not None:
            for k, v in lrs.items():
                self.writer.add_scalar(f'learning_rate/{k}', v, runner.iter + 1)
            for k, v in out.items():
                if isinstance(v, (int, float)):
                    self.writer.add_scalar(f'train/{k}', v, runner.iter + 1)
            self.writer.flush()

    def after_run(self, runner):
        if self.writer is not None:
            self.writer.close()


# --------------------------------------------------------------------------------------------------------------------- reference hooks
class SaveCacheHook:
    """lib/runner/hooks/cache.py:14-68: every `interval` iterations (and after the last with `save_last`) each cached scene goes to
    `<out_dir>/<scene_name>.pth`, and every `viz_step`-th one is visualised into `viz_dir`"""

    def __init__(self, interval=-1, by_epoch=False, out_dir=None, save_last=True, viz_dir=None, viz_step=32):
        if by_epoch:
            raise NotImplementedError('SaveCacheHook by epoch is not supported: the runner counts iterations')
        self.interval, self.out_dir, self.save_last, self.viz_dir, self.viz_step = interval, out_dir, save_last, viz_dir, viz_step
        if _dist_info()[0] == 0:
            os.makedirs(self.out_dir, exist_ok=True)
            if self.viz_dir is not None:
                os.makedirs(self.viz_dir, exist_ok=True)

    def _save(self, module):
        if torch.cuda.is_available():
            torch.cuda.synchronize()                 # the cache entries are filled by asynchronous device-to-host copies
        for i, out in enumerate(module.cache.values()):
            if out is None:
                continue
            torch.save(out, os.path.join(self.out_dir, out['scene_name'] + '.pth'))
            if i % self.viz_step == 0 and self.viz_dir is not None:
                device = next(module.parameters()).device
                code = module.code_activation(out['param']['code_'].to(device=device, dtype=torch.float32))
                module.decoder.visualize(code[None], [out['scene_name']], self.viz_dir,
                                         code_range=module.test_cfg.get('clip_range', [-1, 1]))

    def after_train_iter(self, runner):
        if runner.every_n_iters(self.interval) or (self.save_last and runner.is_last_iter()):
            runner.logger.info(f'Saving cache files at {runner.iter + 1} iterations')
            self._save(getattr(runner.model, 'module', runner.model))


class ModelUpdaterHook:
    """lib/runner/hooks/model_updater.py: when the iteration passes `step[i]`, the settings `cfgs[i]` (dotted names into the model,
    e.g. `train_cfg.extra_scene_step`) are set"""

    def __init__(self, step, cfgs, by_epoch=True):
        if not (isinstance(step, list) and isinstance(cfgs, list) and isinstance(cfgs[0], dict)):
            raise TypeError('ModelUpdaterHook: step must be a list and cfgs a list of dicts')
        if by_epoch:
            raise NotImplementedError('ModelUpdaterHook by epoch is not supported: the runner counts iterations')
        self.step, self.cfgs, self.current_step_id = step, cfgs, 0

    def get_step_id(self, runner):
        step_id = len(self.step)
        for i, s in enumerate(self.step):
            if runner.iter < s:
                step_id = i
                break
        if step_id > self.current_step_id:
            for key, value in self.cfgs[step_id - 1].items():
                rsetattr(getattr(runner.model, 'module', runner.model), key, value)
            self.current_step_id = step_id

    def before_train_iter(self, runner):
        self.get_step_id(runner)


def mean_cache(load_from, code_activation, device=None):
    """lib/runner/hooks/cache.py:186-211: the mean activated code over the scene files in `load_from` -> (file names, mean code on
    the CPU); `code_activation` runs on `device`"""
    files = os.listdir(load_from)
    sum_code, count = None, 0
    for f in files:
        cache = torch.load(os.path.join(load_from, f), map_location='cpu', weights_only=True)
        if 'code_' in cache['param']:
            code = code_activation(cache['param']['code_'].to(device=device, dtype=torch.float32)).cpu()
        elif 'code' in cache['param']:
            code = cache['param']['code'].float()
        else:
            raise ValueError(f'{os.path.join(load_from, f)}: no code_ or code in the scene file')
        if sum_code is None:
            sum_code = torch.zeros_like(code)
        sum_code += code
        count += 1
    return files, sum_code / count


class MeanCacheHook:
    """lib/runner/hooks/cache.py:175-228: at the iterations in `step`, every scene file of `load_from` is replaced in the model's
    `cache_load_from` by the mean code with a fresh density grid, and the cache is reloaded on the next visit"""

    def __init__(self, step, load_from=None, by_epoch=True):
        if not isinstance(step, list):
            raise TypeError('MeanCacheHook: step must be a list')
        if by_epoch:
            raise NotImplementedError('MeanCacheHook by epoch is not supported: the runner counts iterations')
        self.step, self.load_from = step, load_from

    def _update(self, runner):
        module = getattr(runner.model, 'module', runner.model)
        if runner.rank == 0:
            with torch.no_grad():
                files, mean_code = mean_cache(self.load_from, module.code_activation, next(module.parameters()).device)
            out = dict(param=dict(code=mean_code, density_grid=module.get_init_density_grid(None, 'cpu'),
                                  density_bitfield=module.get_init_density_bitfield(None, 'cpu')))
            for f in files:
                torch.save(out, os.path.join(module.train_cfg['cache_load_from'], f))
        if dist.is_available() and dist.is_initialized():
            dist.barrier()
        module.scene_cache.loaded = False

    def before_train_iter(self, runner):
        if runner.iter in self.step:
            runner.logger.info('Resetting cache files to their mean value...')
            self._update(runner)


class DirCopyHook:
    """lib/runner/hooks/filesystem.py: every `interval` iterations (and after the last with `save_last`) rank 0 copies `in_dir`
    into `out_dir`"""

    def __init__(self, interval=-1, by_epoch=False, in_dir=None, out_dir=None, save_last=True):
        if by_epoch:
            raise NotImplementedError('DirCopyHook by epoch is not supported: the runner counts iterations')
        self.interval, self.in_dir, self.out_dir, self.save_last = interval, in_dir, out_dir, save_last

    def after_train_iter(self, runner):
        if runner.every_n_iters(self.interval) or (self.save_last and runner.is_last_iter()):
            runner.logger.info(f'Backing up cache files at {runner.iter + 1} iterations')
            if runner.rank == 0:
                shutil.copytree(self.in_dir, self.out_dir, dirs_exist_ok=True)


class GenerativeEvalHook3D:
    """lib/core/evaluation/eval_hooks.py: every `interval` iterations the model is evaluated (`evaluation.evaluate_3d` over
    `dataloader`, then the metrics' `summary()`); results are logged as `<data>_<name>`, the metrics cleared and the model put back
    in training mode.  With `save_best_ckpt` (mmgen's default) rank 0 keeps `<work_dir>/best_<name>_iter_<n>.pth` for each name of
    `best_metric`, replacing it whenever the evaluation improves on the best so far (lower for fid / kid / test_lpips, higher for
    the others), as mmgen's `GenerativeEvalHook._save_best_ckpt` [mmgen-memory] does."""
    less_keys = ('loss', 'fid', 'kid', 'test_lpips')
    supported_best_metrics = ('fid', 'kid', 'is', 'test_ssim', 'test_psnr', 'test_lpips')

    def __init__(self, dataloader, interval=1, dist=True, metrics=None, sample_kwargs=None, save_best_ckpt=True, best_metric='fid',
                 data='', viz_dir=None, feed_batch_size=32, viz_step=32):
        from .test import build_metric
        if not isinstance(interval, int):
            raise NotImplementedError('GenerativeEvalHook3D: only an integer interval is supported')
        best_metric = [best_metric] if isinstance(best_metric, str) else list(best_metric)
        unknown = [m for m in best_metric if m not in self.supported_best_metrics]
        if save_best_ckpt and unknown:
            raise ValueError(f'GenerativeEvalHook3D: best_metric {unknown} not in {self.supported_best_metrics}')
        metrics = [] if metrics is None else [metrics] if isinstance(metrics, dict) else list(metrics)
        self.dataloader, self.interval, self.data, self.viz_dir = dataloader, interval, data, viz_dir
        self.feed_batch_size, self.viz_step, self.sample_kwargs = feed_batch_size, viz_step, dict(sample_kwargs or {})
        self.save_best_ckpt, self.best_metric = save_best_ckpt, best_metric
        self.best = {}                  # name -> (score, checkpoint path)
        self.metrics = [build_metric(m) for m in metrics]

    def before_run(self, runner):
        for m in self.metrics:
            m.prepare()

    def save_best(self, runner, name, score):
        """keep `best_<name>_iter_<n>.pth` if `score` improves on the best so far (rank 0)"""
        if not (self.save_best_ckpt and name in self.best_metric):
            return
        best = self.best.get(name)
        better = best is None or (score < best[0] if name in self.less_keys else score > best[0])
        if not better:
            return
        filename = f'best_{name}_iter_{runner.iter + 1}.pth'
        if best is not None and os.path.isfile(best[1]):
            os.remove(best[1])
        path = runner.save_checkpoint(runner.work_dir, filename, create_symlink=False)
        self.best[name] = (score, path)
        runner.logger.info(f'Now best checkpoint is saved as {filename}; best {name} is {score:.4f} at iteration {runner.iter + 1}')

    @torch.no_grad()
    def after_train_iter(self, runner):
        if not runner.every_n_iters(self.interval):
            return
        runner.model.eval()
        log_vars = evaluate_3d(runner.model, self.dataloader, self.metrics, self.feed_batch_size, self.viz_dir, self.viz_step,
                               self.sample_kwargs)
        if runner.rank == 0:
            for metric in self.metrics:
                metric.summary()
                for name, val in metric._result_dict.items():
                    runner.log_buffer.output[self.data + '_' + name] = val
                    self.save_best(runner, name, float(val))
            for name, val in log_vars.items():
                runner.logger.info(f'{self.data}_{name} = {val}')
                runner.log_buffer.output[self.data + '_' + name] = float(val)
                self.save_best(runner, name, float(val))
            runner.log_buffer.ready = True
        runner.model.train()
        for metric in self.metrics:
            metric.clear()


HOOKS = dict(ExponentialMovingAverageHook=ExponentialMovingAverageHook, SaveCacheHook=SaveCacheHook, ModelUpdaterHook=ModelUpdaterHook,
             MeanCacheHook=MeanCacheHook, DirCopyHook=DirCopyHook)


def build_hook(cfg):
    cfg = dict(cfg)
    kind = cfg.pop('type')
    if kind not in HOOKS:
        raise NotImplementedError(f'hook type {kind!r} is not supported ({", ".join(sorted(HOOKS))} are)')
    return HOOKS[kind](**cfg)


# --------------------------------------------------------------------------------------------------------------------- train_model
def train_model(model, dataset, cfg, distributed=False, validate=False, timestamp=None, meta=None, logger=None, device=None):
    """lib/apis/train.py:train_model: loader, optimizers, runner and hooks from `cfg`, then `run` to `cfg.total_iters`; returns the
    runner"""
    from .registry import build_dataset
    if cfg.get('apex_amp', None):
        raise NotImplementedError('apex_amp is not supported')
    if cfg.get('fp16', None) is not None:
        raise NotImplementedError('fp16 training (an fp16 optimizer hook) is not supported')
    rank, _ = _dist_info()
    data_cfg = cfg['data']
    loader_cfg = dict(samples_per_gpu=data_cfg['samples_per_gpu'], **data_cfg.get('train_dataloader', {}))
    unknown = set(loader_cfg) - {'samples_per_gpu', 'workers_per_gpu', 'persistent_workers', 'split_data', 'check_batch_disjoint'}
    if unknown:
        raise NotImplementedError(f'train_dataloader options {sorted(unknown)} are not supported')
    loader = TrainLoader(dataset, loader_cfg['samples_per_gpu'], device, seed=cfg.get('seed'),
                         split_data=loader_cfg.get('split_data', False),
                         check_batch_disjoint=loader_cfg.get('check_batch_disjoint', False))
    optimizer = build_optimizers(model, cfg['optimizer']) if cfg.get('optimizer') else {}
    if not isinstance(optimizer, dict):
        optimizer = dict(model=optimizer)
    runner = Runner(model, optimizer, cfg['work_dir'], logger=logger, meta=meta, timestamp=timestamp)

    if cfg.get('lr_config') is not None:
        runner.register_hook(LrUpdaterHook(**cfg['lr_config']), 'VERY_HIGH')
    if cfg.get('checkpoint_config') is not None:
        ck = dict(cfg['checkpoint_config'])
        ck['out_dir'] = os.path.join(cfg['work_dir'], ck.get('out_dir', 'ckpt'))
        runner.register_hook(CheckpointHook(**ck), 'NORMAL')
    log_cfg = cfg.get('log_config')
    if log_cfg is not None:
        kinds = [h['type'] for h in log_cfg.get('hooks', [])]
        unknown = set(kinds) - {'TextLoggerHook', 'TensorboardLoggerHook'}
        if unknown:
            raise NotImplementedError(f'logger hooks {sorted(unknown)} are not supported')
        runner.register_hook(LoggerHook(log_cfg.get('interval', 10), text='TextLoggerHook' in kinds,
                                        tensorboard='TensorboardLoggerHook' in kinds), 'VERY_LOW')
    if validate and cfg.get('evaluation') is not None:
        from .test import eval_plan
        if not isinstance(cfg['evaluation'], (list, tuple)):
            raise TypeError('cfg.evaluation must be a list of evaluation hooks')
        for ev, entry in zip(cfg['evaluation'], eval_plan(cfg)):
            ev = dict(ev)
            if ev.pop('type', 'GenerativeEvalHook3D') != 'GenerativeEvalHook3D':
                raise NotImplementedError('only GenerativeEvalHook3D evaluations are supported')
            priority = ev.pop('priority', 'LOW')
            batches = SceneBatches(build_dataset(entry['dataset']), entry['samples_per_gpu'], device)
            runner.register_hook(GenerativeEvalHook3D(batches, dist=distributed, **ev), priority)
    for hook_cfg in cfg.get('custom_hooks', None) or []:
        hook_cfg = dict(hook_cfg)
        priority = hook_cfg.pop('priority', 'NORMAL')
        runner.register_hook(build_hook(hook_cfg), priority)

    if cfg.get('resume_from'):
        runner.resume(cfg['resume_from'])
        loader.set_epoch(runner.epoch)
        if distributed:
            loader.skip_iter = runner.iter % len(loader)
        elif rank == 0:
            warnings.warn('Dataloader resuming is currently not supported for non-distributed training')
    elif cfg.get('load_from'):
        runner.load_checkpoint(cfg['load_from'])
    runner.run(loader, cfg['workflow'], cfg['total_iters'])
    return runner
