"""Exponential moving average of model weights: mmgen's `ExponentialMovingAverageHook` [mmgen-memory] as every training config
registers it (`interp_mode='lerp'`, `momentum_policy='rampup'`, `interval=1`, `start_iter=0`), on the fused kernel of csrc/ema.cu.

mmgen updates each state entry as `ema = src + (ema - src) * m` with three separately rounded torch kernels per tensor, then
`load_state_dict`s the result.  `ema_lerp_` does the same arithmetic, bit for bit, for a whole state in one launch: `m` is the rampup
momentum for entries whose source is a parameter that requires grad, and `momentum_nontrainable` (0: a copy) for buffers and frozen
modules.  The kernel writes the EMA tensors in place without bumping `Parameter._version`, so the hook calls `refresh_weights()` on
every updated module that caches packed weights (the UNet's fp16 engine and captured DDIM graphs, the decoder's weight blob)."""
import torch

from . import _lib as N


def rampup_momentum(iteration, ema_kimg=10, ema_rampup=0.05, batch_size=4, eps=1e-8):
    """mmgen `ExponentialMovingAverageHook.rampup` [mmgen-memory] after iteration `iteration` (0-based): the EMA half-life is
    `ema_kimg` thousand images, shortened to `ema_rampup` of the images seen so far; computed in double (the kernel rounds it to
    float once, as torch does when it multiplies an fp32 tensor by a Python float)"""
    cur_nimg = (iteration + 1) * batch_size
    ema_nimg = ema_kimg * 1000
    if ema_rampup is not None:
        ema_nimg = min(ema_nimg, cur_nimg * ema_rampup)
    return 0.5 ** (batch_size / max(ema_nimg, eps))


def ema_lerp_(ema, src, trainable, momentum, momentum_nontrainable=0.0):
    """ema[i] <- src[i] + (ema[i] - src[i]) * m for every pair, in one launch on the current stream; m = `momentum` where
    `trainable[i]`, else `momentum_nontrainable`.  Tensors: fp32, contiguous, on the current CUDA device, pairs of equal shape."""
    if not (len(ema) == len(src) == len(trainable)):
        raise ValueError(f'ema_lerp_: {len(ema)} EMA tensors, {len(src)} sources and {len(trainable)} trainable flags')
    table = (N.EmaTensor * max(len(ema), 1))()
    for i, (e, s, tr) in enumerate(zip(ema, src, trainable)):
        if e.shape != s.shape:
            raise ValueError(f'ema_lerp_: tensor {i}: EMA shape {tuple(e.shape)} != source shape {tuple(s.shape)}')
        for t in (e, s):
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f'ema_lerp_: tensor {i} must be contiguous fp32 (got {t.dtype}, contiguous={t.is_contiguous()})')
        N.require_cuda(e, s)
        table[i].ema, table[i].src, table[i].n, table[i].trainable = e.data_ptr(), s.data_ptr(), e.numel(), int(bool(tr))
    N.check(N.lib().ssdnerf_ema_lerp_f32(table, len(ema), float(momentum), float(momentum_nontrainable),
                                         N.stream_ptr() if ema else None))


def refresh_cached_weights(module):
    """drop the packed-weight caches of `module` and its submodules (after writes that bypass `Parameter._version`)"""
    for m in module.modules():
        if hasattr(m, 'refresh_weights'):
            m.refresh_weights()


class ExponentialMovingAverageHook:
    """mmgen's hook for `module_keys` such as ('diffusion_ema', 'decoder_ema'): after every `interval`-th iteration, each
    `<name>_ema` module follows `<name>` with the rampup momentum of `momentum_cfg` (`rampup_momentum`'s arguments).  Only the lerp
    interpolation, the rampup policy and `start_iter=0` -- what every shipped config uses -- are built; anything else raises."""
    priority = 'VERY_HIGH'

    def __init__(self, module_keys, interp_mode='lerp', interp_cfg=None, interval=-1, start_iter=0, momentum_policy='fixed',
                 momentum_cfg=None):
        module_keys = (module_keys,) if isinstance(module_keys, str) else tuple(module_keys)
        for k in module_keys:
            if not k.endswith('_ema'):
                raise ValueError(f'ExponentialMovingAverageHook: module key {k!r} does not end with "_ema"')
        if interp_mode != 'lerp':
            raise NotImplementedError(f'ExponentialMovingAverageHook: interp_mode={interp_mode!r} is not supported (lerp is)')
        if momentum_policy != 'rampup':
            raise NotImplementedError(f'ExponentialMovingAverageHook: momentum_policy={momentum_policy!r} is not supported (rampup is)')
        if start_iter > 0:
            raise NotImplementedError(f'ExponentialMovingAverageHook: start_iter={start_iter} is not supported (0 is)')
        self.module_keys, self.interval, self.start_iter = module_keys, interval, start_iter
        self.momentum_cfg = dict(momentum_cfg or {})
        self.momentum_nontrainable = float(dict(interp_cfg or {}).get('momentum_nontrainable', 0.0))

    def every_n_iters(self, iteration):
        return (iteration + 1 - self.start_iter) % self.interval == 0 if self.interval > 0 else False

    @torch.no_grad()
    def update(self, model, iteration):
        """one EMA step of every module key after iteration `iteration` (0-based); returns the momentum used"""
        momentum = rampup_momentum(iteration, **self.momentum_cfg)
        for key in self.module_keys:
            ema_net, net = getattr(model, key), getattr(model, key[:-4])
            states_ema = ema_net.state_dict(keep_vars=True)
            ema, src, trainable = [], [], []
            for k, v in net.state_dict(keep_vars=True).items():
                if k not in states_ema:
                    raise KeyError(f'ExponentialMovingAverageHook: {key} has no state entry {k!r}')
                e = states_ema[k]
                for name, t in ((key[:-4], v), (key, e)):
                    if t.dtype != torch.float32 or not t.is_contiguous():
                        raise ValueError(f'ExponentialMovingAverageHook: {name}.{k} must be contiguous fp32 '
                                         f'(got {t.dtype}, contiguous={t.is_contiguous()})')
                ema.append(e)
                src.append(v)
                trainable.append(v.requires_grad)
            ema_lerp_(ema, src, trainable, momentum, self.momentum_nontrainable)
            refresh_cached_weights(ema_net)
        return momentum

    def after_train_iter(self, runner):
        if self.every_n_iters(runner.iter):
            runner.ema_momentum = self.update(runner.model, runner.iter)
