"""How far may a native DDPM chain sit from the fp32 oracle?  CPU experiment: the fp32 oracle chain (oracle/ddpm_port.py) with the native
path's fp16 roundings injected into every UNet evaluation -- GEMM / convolution operands (activations incl. the UNet input, weights), the
convolution outputs that feed a GroupNorm, the residual stream, as tests/perf/precision_probe.py does for one evaluation -- against
the same chain without them, fed the same noise.  Prints rel-L2 of the final sample; tests/test_ddpm_gpu.py sets its bars at twice
these values.  TEST INFRASTRUCTURE (imports oracle/).

  python tests/perf/ddpm_precision_probe.py [small|cars|guided]...
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
import torch.nn.functional as F

from oracle import ddpm_port as dp
from oracle import unet_port as up

torch.set_num_threads(os.cpu_count())
ROUND = [False]
rt = lambda x: x.half().float() if ROUND[0] else x
_conv2d, _conv1d, _res, _attn = F.conv2d, F.conv1d, up.res_block, up.attention


class _F:      # torch.nn.functional inside unet_port with fp16-rounded convolution operands
    def __getattr__(self, k):
        if k == 'conv2d':
            return lambda x, w, b=None, **kw: _conv2d(rt(x), rt(w), b, **kw)
        if k == 'conv1d':
            return lambda x, w, b=None, **kw: _conv1d(rt(x), rt(w), b, **kw)
        return getattr(F, k)


def res_block(sd, b, x, emb):
    k = b['key']
    sc = up.F.conv2d(x, sd[k + '.shortcut.weight'], sd[k + '.shortcut.bias']) if b['cin'] != b['cout'] else x
    h = rt(up.F.conv2d(F.silu(up._gn(sd, k + '.conv_1.0', x)), sd[k + '.conv_1.2.weight'], sd[k + '.conv_1.2.bias'], padding=1))
    e = F.linear(F.silu(emb), sd[k + '.norm_with_embedding.embedding_layer.1.weight'], sd[k + '.norm_with_embedding.embedding_layer.1.bias'])[:, :, None, None]
    scale, shift = torch.chunk(e, 2, dim=1)
    h = up._gn(sd, k + '.norm_with_embedding.norm', h) * (1 + scale) + shift
    h = up.F.conv2d(F.silu(h), sd[k + '.conv_2.1.weight'], sd[k + '.conv_2.1.bias'], padding=1)
    return rt(h + sc)


up.F, up.res_block, up.attention = _F(), res_block, lambda sd, b, x, nh: rt(_attn(sd, b, x, nh))


def probe(name, cfg, B, steps, seed, guided=False):
    spec = up.unet_spec(**cfg)
    sd = up.random_state_dict(spec, seed=seed, std=0.02 if cfg.get('base_channels', 128) == 128 else 0.04)
    dv = up.diffusion_vars(up.linear_betas())
    g = torch.Generator().manual_seed(seed + 1)
    res = cfg.get('image_size', 128)
    x = torch.randn(B, 18, res, res, generator=g)
    zs = [torch.randn(B, 18, res, res, generator=g) for _ in range(steps)]
    kw = dict(num_timesteps=steps, clip_range=(-2, 2))
    if guided:
        target = torch.randn(B, 18, res, res, generator=g)
        kw.update(grad_guide_fn=lambda x0: 0.5 * ((x0 - target) ** 2).mean() * x0.size(0), guidance_gain=37.5, snr_weight_power=0.25)
    den = lambda x, t: up.unet_forward(sd, spec, x, t)
    t0 = time.time()
    out = []
    for r in (False, True):
        ROUND[0] = r
        out.append(dp.ddpm_sample(den, x, dv, iter(zs), **kw))
    rel = float((out[1] - out[0]).norm() / out[0].norm())
    print(f'{name:8s} B={B} {steps:4d} steps: fp16-rounding probe rel-L2 {rel:.3e}  ({time.time() - t0:.0f} s)', flush=True)


SMALL = dict(image_size=32, base_channels=64, channels_cfg=(1, 2, 2), resblocks_per_downsample=1, num_heads=2, attention_res=(16, 8))
for which in sys.argv[1:] or ['small', 'guided', 'cars']:
    if which == 'small':
        probe('small', SMALL, 2, 1000, 21)
    elif which == 'guided':
        probe('guided', SMALL, 2, 10, 23, guided=True)
    elif which == 'cars':
        probe('cars', dict(), 2, 50, 25)
