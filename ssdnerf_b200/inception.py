"""Inception-v3 features of FID / KID on the package's own kernels (csrc/inception.cu): the StyleGAN Inception TorchScript
(`inception-2015-12-05.pt`) that the shipped configs' `FIDKID(inception_args=dict(type='StyleGAN', inception_path=...))` and mmgen's
`FID` name, i.e. the 2015-12-05 TF graph with pytorch-fid's `FIDInception*` block semantics.

* preprocessing (one launch): u8 quantisation as tools/inception_stat.py:101, bilinear resize to 299 x 299, (u - 128) / 128, fp16 NHWC
  padded to 16 channels;
* the 94 convolutions: implicit-GEMM wgmma with BatchNorm (eps 1e-3) folded into fp16 weights and an fp32 bias at load time and ReLU in
  the epilogue; each branch writes its channel slice of the block's concatenated output, so there are no concatenation copies;
* the 3 x 3 pools (max / stride 2; average / stride 1 / pad 1 excluding padding; max / stride 1 / pad 1 in Mixed_7c) and the global
  8 x 8 mean to fp32 [n, 2048].

Weights are an external asset and are never downloaded: `InceptionV3.load(path)` reads the TorchScript, `from_state_dict(sd)` takes
torchvision `Inception3`'s parameter names (fc and AuxLogits keys are ignored)."""
import os

import torch

from . import _lib as N

SIZE = 299
IN_CHANNELS = 16                         # the normalised RGB input, zero-padded to the convolution's 16-wide K step
EPS = 1e-3
DEFAULT_WORKSPACE_BYTES = 2 << 30
POOL_MAX_S2, POOL_AVG_S1, POOL_MAX_S1 = 0, 1, 2


def _conv_specs():
    """(prefix, cin, cout, kh, kw, stride, pad_h, pad_w) of the 94 convolutions in network order, under torchvision's names"""
    out = []

    def c(name, cin, cout, k=(1, 1), s=1, p=(0, 0)):
        out.append((name, cin, cout, k[0], k[1], s, p[0], p[1]))

    k3, k5, k17, k71, k13, k31 = (3, 3), (5, 5), (1, 7), (7, 1), (1, 3), (3, 1)
    c('Conv2d_1a_3x3', 3, 32, k3, 2)
    c('Conv2d_2a_3x3', 32, 32, k3)
    c('Conv2d_2b_3x3', 32, 64, k3, 1, (1, 1))
    c('Conv2d_3b_1x1', 64, 80)
    c('Conv2d_4a_3x3', 80, 192, k3)
    for b, cin, pf in (('Mixed_5b', 192, 32), ('Mixed_5c', 256, 64), ('Mixed_5d', 288, 64)):
        c(f'{b}.branch1x1', cin, 64)
        c(f'{b}.branch5x5_1', cin, 48)
        c(f'{b}.branch5x5_2', 48, 64, k5, 1, (2, 2))
        c(f'{b}.branch3x3dbl_1', cin, 64)
        c(f'{b}.branch3x3dbl_2', 64, 96, k3, 1, (1, 1))
        c(f'{b}.branch3x3dbl_3', 96, 96, k3, 1, (1, 1))
        c(f'{b}.branch_pool', cin, pf)
    c('Mixed_6a.branch3x3', 288, 384, k3, 2)
    c('Mixed_6a.branch3x3dbl_1', 288, 64)
    c('Mixed_6a.branch3x3dbl_2', 64, 96, k3, 1, (1, 1))
    c('Mixed_6a.branch3x3dbl_3', 96, 96, k3, 2)
    for b, c7 in (('Mixed_6b', 128), ('Mixed_6c', 160), ('Mixed_6d', 160), ('Mixed_6e', 192)):
        c(f'{b}.branch1x1', 768, 192)
        c(f'{b}.branch7x7_1', 768, c7)
        c(f'{b}.branch7x7_2', c7, c7, k17, 1, (0, 3))
        c(f'{b}.branch7x7_3', c7, 192, k71, 1, (3, 0))
        c(f'{b}.branch7x7dbl_1', 768, c7)
        c(f'{b}.branch7x7dbl_2', c7, c7, k71, 1, (3, 0))
        c(f'{b}.branch7x7dbl_3', c7, c7, k17, 1, (0, 3))
        c(f'{b}.branch7x7dbl_4', c7, c7, k71, 1, (3, 0))
        c(f'{b}.branch7x7dbl_5', c7, 192, k17, 1, (0, 3))
        c(f'{b}.branch_pool', 768, 192)
    c('Mixed_7a.branch3x3_1', 768, 192)
    c('Mixed_7a.branch3x3_2', 192, 320, k3, 2)
    c('Mixed_7a.branch7x7x3_1', 768, 192)
    c('Mixed_7a.branch7x7x3_2', 192, 192, k17, 1, (0, 3))
    c('Mixed_7a.branch7x7x3_3', 192, 192, k71, 1, (3, 0))
    c('Mixed_7a.branch7x7x3_4', 192, 192, k3, 2)
    for b, cin in (('Mixed_7b', 1280), ('Mixed_7c', 2048)):
        c(f'{b}.branch1x1', cin, 320)
        c(f'{b}.branch3x3_1', cin, 384)
        c(f'{b}.branch3x3_2a', 384, 384, k13, 1, (0, 1))
        c(f'{b}.branch3x3_2b', 384, 384, k31, 1, (1, 0))
        c(f'{b}.branch3x3dbl_1', cin, 448)
        c(f'{b}.branch3x3dbl_2', 448, 384, k3, 1, (1, 1))
        c(f'{b}.branch3x3dbl_3a', 384, 384, k13, 1, (0, 1))
        c(f'{b}.branch3x3dbl_3b', 384, 384, k31, 1, (1, 0))
        c(f'{b}.branch_pool', cin, 192)
    return tuple(out)


CONVS = _conv_specs()
SPEC = {s[0]: s for s in CONVS}
WEIGHT_SHAPES = tuple((co, ci, kh, kw) for _, ci, co, kh, kw, *_ in CONVS)

# BatchNorm tensors that may follow a convolution weight in a state dict, by leaf name: (gamma, beta, mean, var); None = absent
# (gamma 1).  A lone `bias` is a convolution whose BatchNorm is already folded.
_BN_SETS = {
    frozenset(('weight', 'bias', 'running_mean', 'running_var')): ('weight', 'bias', 'running_mean', 'running_var'),
    frozenset(('bias', 'running_mean', 'running_var')): (None, 'bias', 'running_mean', 'running_var'),
    frozenset(('gamma', 'beta', 'mean', 'var')): ('gamma', 'beta', 'mean', 'var'),
    frozenset(('beta', 'mean', 'var')): (None, 'beta', 'mean', 'var'),
    frozenset(('gamma', 'beta', 'moving_mean', 'moving_variance')): ('gamma', 'beta', 'moving_mean', 'moving_variance'),
    frozenset(('beta', 'moving_mean', 'moving_variance')): (None, 'beta', 'moving_mean', 'moving_variance'),
    frozenset(('bias',)): None,
}

# per-image fp16 elements of the workspace: two ping-pong maps (the largest is the 299 x 299 x 16 input), two branch scratch maps
# (the largest is 35 x 35 x 96) and the pool-branch scratch (35 x 35 x 288)
_PING = SIZE * SIZE * IN_CHANNELS
_SCRATCH = 35 * 35 * 96
_POOLED = 35 * 35 * 288


def image_bytes():
    return 2 * (2 * _PING + 2 * _SCRATCH + _POOLED)


def fold_bn(w, gamma, beta, mean, var, eps=EPS):
    """conv (no bias) then BatchNorm(eps) in eval mode -> (w', b') in float64"""
    w, beta, mean, var = (t.double() for t in (w, beta, mean, var))
    s = (gamma.double() if gamma is not None else torch.ones_like(var)) / torch.sqrt(var + eps)
    return w * s.reshape(-1, 1, 1, 1), beta - mean * s


def _groups(sd):
    """[(weight key, weight, [(key, 1-D tensor), ...])]: each 4-D tensor in state-dict order with the 1-D tensors of its output width
    that directly follow it (0-D counters are skipped; anything else ends the group)"""
    groups, open_ = [], False
    for k, t in sd.items():
        if not isinstance(t, torch.Tensor) or t.dim() == 0:
            continue
        if t.dim() == 4:
            groups.append((k, t, []))
            open_ = True
        elif open_ and t.dim() == 1 and t.shape[0] == groups[-1][1].shape[0]:
            groups[-1][2].append((k, t))
        else:
            open_ = False
    return groups


class _Act:
    """an NHWC fp16 map in a workspace buffer: pixel p, channel k at buf[off + p * stride + k]"""
    __slots__ = ('buf', 'off', 'h', 'w', 'c', 'stride')

    def __init__(self, buf, h, w, c, stride=None, off=0):
        self.buf, self.h, self.w, self.c, self.stride, self.off = buf, h, w, c, stride or c, off

    def ptr(self):
        return N.c_void_p(self.buf.data_ptr() + 2 * self.off)


class InceptionV3:
    """InceptionV3(folded)(images) -> [n, 2048] fp32.  Build with `from_state_dict(sd)` or `load(path)`.

    images: [n, 3, h, w] float in [-1, 1] on the current CUDA device.  They run `chunk` at a time from one workspace
    (chunk = workspace_bytes // image_bytes()); an image's features do not depend on the chunk it ran in and are bit-identical run
    to run."""

    def __init__(self, folded, workspace_bytes=DEFAULT_WORKSPACE_BYTES, source=None):
        self.source = source
        self.workspace_bytes = int(workspace_bytes)
        self._host = {}
        for name, cin, cout, kh, kw, *_ in CONVS:
            w, b = folded[name]
            w = w.double().permute(0, 2, 3, 1)                        # [cout][kh][kw][cin]
            if cin % 16:
                w = torch.nn.functional.pad(w, (0, IN_CHANNELS - cin))
            self._host[name] = (w.half().contiguous(), b.float().contiguous())
        self._dev = {}
        self._ws = None

    # ------------------------------------------------------------------ loading
    @classmethod
    def from_state_dict(cls, sd, **kw):
        """torchvision `Inception3` names: `{prefix}.conv.weight` and `{prefix}.bn.{weight,bias,running_mean,running_var}` for the 94
        convolutions (fc, AuxLogits and num_batches_tracked are ignored).  A missing key or a wrong shape is a ValueError naming it."""
        folded = {}
        for name, cin, cout, kh, kw_, *_ in CONVS:
            ts = {}
            for leaf, shape in (('conv.weight', (cout, cin, kh, kw_)), ('bn.weight', (cout,)), ('bn.bias', (cout,)),
                                ('bn.running_mean', (cout,)), ('bn.running_var', (cout,))):
                k = f'{name}.{leaf}'
                if k not in sd:
                    raise ValueError(f'InceptionV3: missing key {k!r}')
                if tuple(sd[k].shape) != shape:
                    raise ValueError(f'InceptionV3: key {k!r} has shape {tuple(sd[k].shape)}, expected {shape}')
                ts[leaf] = torch.as_tensor(sd[k])
            folded[name] = fold_bn(ts['conv.weight'], ts['bn.weight'], ts['bn.bias'], ts['bn.running_mean'], ts['bn.running_var'])
        return cls(folded, **kw)

    @classmethod
    def from_ordered_state_dict(cls, sd, where='state dict', **kw):
        """any naming: the state dict's 4-D tensors, in order, must have the 94 weight shapes in network order, and the 1-D tensors
        following each must be one BatchNorm set of _BN_SETS (by leaf name) or a lone bias.  ValueError naming the first mismatch."""
        groups = _groups(sd)
        folded = {}
        for i, (name, *_rest) in enumerate(CONVS):
            if i >= len(groups):
                raise ValueError(f'{where}: {len(groups)} convolution weights (4-D tensors), expected 94; the next expected shape is '
                                 f'{WEIGHT_SHAPES[i]}')
            k, w, bn = groups[i]
            if tuple(w.shape) != WEIGHT_SHAPES[i]:
                raise ValueError(f'{where}: key {k!r} has shape {tuple(w.shape)}, expected {WEIGHT_SHAPES[i]} (convolution {i}, {name})')
            leaves = {bk.rsplit('.', 1)[-1]: t for bk, t in bn}
            roles = _BN_SETS.get(frozenset(leaves), 'bad') if len(leaves) == len(bn) else 'bad'
            if roles == 'bad':
                raise ValueError(f'{where}: the 1-D tensors after {k!r} are {[bk for bk, _ in bn]}, not a BatchNorm set '
                                 f'({sorted(sorted(s) for s in _BN_SETS)})')
            if roles is None:
                folded[name] = (w.double(), leaves['bias'].double())
            else:
                g, b, m, v = (leaves[r] if r else None for r in roles)
                folded[name] = fold_bn(w, g, b, m, v)
        if len(groups) > len(CONVS):
            raise ValueError(f'{where}: unexpected convolution weight {groups[len(CONVS)][0]!r} after the 94 of the network')
        return cls(folded, **kw)

    @classmethod
    def load(cls, path, **kw):
        """the StyleGAN TorchScript (inception-2015-12-05.pt): its state dict mapped by order and shape (from_ordered_state_dict)"""
        if not os.path.isfile(path):
            raise FileNotFoundError(f'InceptionV3: {path} not found (the Inception TorchScript is an external asset and is never downloaded)')
        ts = torch.jit.load(path, map_location='cpu')
        return cls.from_ordered_state_dict(ts.state_dict(), where=path, source=path, **kw)

    # ------------------------------------------------------------------ running
    def _weights(self, device):
        if device not in self._dev:
            self._dev[device] = {k: (w.to(device), b.to(device)) for k, (w, b) in self._host.items()}
        return self._dev[device]

    def chunk(self):
        return max(1, self.workspace_bytes // image_bytes())

    def _conv(self, W, n, name, x, buf, stride=None, c0=0):
        _, cin, cout, kh, kw, s, ph, pw = SPEC[name]
        w, b = W[name]
        oh, ow = (x.h + 2 * ph - kh) // s + 1, (x.w + 2 * pw - kw) // s + 1
        y = _Act(buf, oh, ow, cout, stride, c0)
        N.check(N.lib().ssdnerf_incep_conv_f16(x.ptr(), N.c_u32(n), N.c_u32(x.h), N.c_u32(x.w), N.c_u32(x.c), N.c_u32(x.stride),
                                               N.ptr(w), N.ptr(b), N.c_u32(cout), N.c_u32(kh), N.c_u32(kw), N.c_u32(s), N.c_u32(ph),
                                               N.c_u32(pw), N.c_int(1), y.ptr(), N.c_u32(y.stride), N.stream_ptr()))
        return y

    @staticmethod
    def _pool(n, x, mode, buf, stride=None, c0=0):
        oh, ow = ((x.h - 3) // 2 + 1, (x.w - 3) // 2 + 1) if mode == POOL_MAX_S2 else (x.h, x.w)
        y = _Act(buf, oh, ow, x.c, stride, c0)
        N.check(N.lib().ssdnerf_incep_pool_f16(x.ptr(), N.c_u32(n), N.c_u32(x.h), N.c_u32(x.w), N.c_u32(x.c), N.c_u32(x.stride),
                                               N.c_int(mode), y.ptr(), N.c_u32(y.stride), N.stream_ptr()))
        return y

    def _network(self, W, n, bufs, out):
        """the 94 convolutions, pools and the global mean over the prepared input in bufs[0] -> out fp32 [n, 2048]"""
        P, S1, S2, S3 = bufs[:2], bufs[2], bufs[3], bufs[4]
        conv = lambda name, x, buf, stride=None, c0=0: self._conv(W, n, name, x, buf, stride, c0)
        pool = lambda x, mode, buf, stride=None, c0=0: self._pool(n, x, mode, buf, stride, c0)
        t = _Act(P[0], SIZE, SIZE, IN_CHANNELS)
        t = conv('Conv2d_1a_3x3', t, P[1])
        t = conv('Conv2d_2a_3x3', t, P[0])
        t = conv('Conv2d_2b_3x3', t, P[1])
        t = pool(t, POOL_MAX_S2, P[0])
        t = conv('Conv2d_3b_1x1', t, P[1])
        t = conv('Conv2d_4a_3x3', t, P[0])
        t = pool(t, POOL_MAX_S2, P[1])
        cur = 1
        for b in ('Mixed_5b', 'Mixed_5c', 'Mixed_5d'):           # InceptionA: 64 | 64 | 96 | pool features
            d, ct = P[1 - cur], 224 + SPEC[f'{b}.branch_pool'][2]
            conv(f'{b}.branch1x1', t, d, ct, 0)
            conv(f'{b}.branch5x5_2', conv(f'{b}.branch5x5_1', t, S1), d, ct, 64)
            conv(f'{b}.branch3x3dbl_3', conv(f'{b}.branch3x3dbl_2', conv(f'{b}.branch3x3dbl_1', t, S1), S2), d, ct, 128)
            conv(f'{b}.branch_pool', pool(t, POOL_AVG_S1, S3), d, ct, 224)
            t, cur = _Act(d, t.h, t.w, ct), 1 - cur
        d = P[1 - cur]                                            # InceptionB: 384 | 96 | max pool (288)
        y = conv('Mixed_6a.branch3x3', t, d, 768, 0)
        conv('Mixed_6a.branch3x3dbl_3', conv('Mixed_6a.branch3x3dbl_2', conv('Mixed_6a.branch3x3dbl_1', t, S1), S2), d, 768, 384)
        pool(t, POOL_MAX_S2, d, 768, 480)
        t, cur = _Act(d, y.h, y.w, 768), 1 - cur
        for b in ('Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e'):   # InceptionC: 192 each
            d = P[1 - cur]
            conv(f'{b}.branch1x1', t, d, 768, 0)
            conv(f'{b}.branch7x7_3', conv(f'{b}.branch7x7_2', conv(f'{b}.branch7x7_1', t, S1), S2), d, 768, 192)
            a = conv(f'{b}.branch7x7dbl_1', t, S1)
            a = conv(f'{b}.branch7x7dbl_2', a, S2)
            a = conv(f'{b}.branch7x7dbl_3', a, S1)
            a = conv(f'{b}.branch7x7dbl_4', a, S2)
            conv(f'{b}.branch7x7dbl_5', a, d, 768, 384)
            conv(f'{b}.branch_pool', pool(t, POOL_AVG_S1, S3), d, 768, 576)
            t, cur = _Act(d, t.h, t.w, 768), 1 - cur
        d = P[1 - cur]                                            # InceptionD: 320 | 192 | max pool (768)
        y = conv('Mixed_7a.branch3x3_2', conv('Mixed_7a.branch3x3_1', t, S1), d, 1280, 0)
        a = conv('Mixed_7a.branch7x7x3_1', t, S1)
        a = conv('Mixed_7a.branch7x7x3_2', a, S2)
        a = conv('Mixed_7a.branch7x7x3_3', a, S1)
        conv('Mixed_7a.branch7x7x3_4', a, d, 1280, 320)
        pool(t, POOL_MAX_S2, d, 1280, 512)
        t, cur = _Act(d, y.h, y.w, 1280), 1 - cur
        for b, mode in (('Mixed_7b', POOL_AVG_S1), ('Mixed_7c', POOL_MAX_S1)):   # InceptionE: 320 | 384 | 384 | 384 | 384 | 192
            d = P[1 - cur]
            conv(f'{b}.branch1x1', t, d, 2048, 0)
            a = conv(f'{b}.branch3x3_1', t, S1)
            conv(f'{b}.branch3x3_2a', a, d, 2048, 320)
            conv(f'{b}.branch3x3_2b', a, d, 2048, 704)
            a = conv(f'{b}.branch3x3dbl_2', conv(f'{b}.branch3x3dbl_1', t, S1), S2)
            conv(f'{b}.branch3x3dbl_3a', a, d, 2048, 1088)
            conv(f'{b}.branch3x3dbl_3b', a, d, 2048, 1472)
            conv(f'{b}.branch_pool', pool(t, mode, S3), d, 2048, 1856)
            t, cur = _Act(d, t.h, t.w, 2048), 1 - cur
        N.check(N.lib().ssdnerf_incep_mean_f16(t.ptr(), N.c_u32(n), N.c_u32(t.h * t.w), N.c_u32(2048), N.ptr(out), N.stream_ptr()))

    @torch.no_grad()
    def __call__(self, images):
        N.require_cuda(images)
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f'InceptionV3: images must be [n, 3, h, w], got {tuple(images.shape)}')
        images = images.float().contiguous()
        n, _, h, w = images.shape
        dev = images.device
        out = torch.empty(n, 2048, dtype=torch.float32, device=dev)
        if n == 0:
            return out
        W = self._weights(dev)
        cm = min(n, self.chunk())
        sizes = (_PING, _PING, _SCRATCH, _SCRATCH, _POOLED)
        if self._ws is None or self._ws.device != dev or self._ws.numel() < cm * sum(sizes):
            self._ws = torch.empty(cm * sum(sizes), dtype=torch.float16, device=dev)
        bufs, o = [], 0
        for s in sizes:
            bufs.append(self._ws[o:o + cm * s])
            o += cm * s
        for j0 in range(0, n, cm):
            m = min(cm, n - j0)
            N.check(N.lib().ssdnerf_incep_prep_f16(N.ptr(images[j0:j0 + m]), N.c_u32(m), N.c_u32(h), N.c_u32(w), N.ptr(bufs[0]), None,
                                                   N.stream_ptr()))
            self._network(W, m, bufs, out[j0:j0 + m])
        return out
