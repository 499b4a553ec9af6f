"""CPU / PyTorch restatement of the StyleGAN Inception-v3 feature extractor of FID / KID (TEST INFRASTRUCTURE): the preprocessing of
tools/inception_stat.py:101 plus the TorchScript's resize and normalisation, and the 2015-12-05 TF graph as pytorch-fid's
`FIDInception{A,C,E_1,E_2}` blocks restate it (94 convolutions with BatchNorm eps 1e-3 and ReLU, the pool variants, the global mean).

What is pinned and what is not:
  * The network is pinned (tests/golden/reference_inception_v1.npz) to an EXECUTION of torchvision 0.26's `Inception3` blocks with the
    FID differences applied (count_include_pad=False in the average pools of Mixed_5*, Mixed_6b-e and Mixed_7b, a max pool in Mixed_7c),
    on seeded He-scaled weights whose BatchNorm statistics were calibrated on images.  It is NOT pinned to the StyleGAN TorchScript
    (inception-2015-12-05.pt), which is an external asset: only tests/test_inception_gpu.py's asset test, skipped without the file,
    compares against it.
  * The resize rule is restated from memory of the TorchScript's code (affine_grid / grid_sample(bilinear, border,
    align_corners=False) with theta[0, 2] += 1/w - 1/299): `resize_affine_grid` is that composition and `resize_closed_form` the
    closed form the kernel implements (source coordinate o * in / 299, clamped to the last pixel).  The CPU tests show the two agree;
    neither is checked against the asset here.
Images are [n, 3, h, w] in [-1, 1]; features [n, 2048]."""
import math

import numpy as np
import torch
import torch.nn.functional as F

SIZE = 299
EPS = 1e-3


def _block_specs():
    """(prefix, cin, cout, kh, kw, stride, pad_h, pad_w) of the 94 convolutions in network order (torchvision's names)"""
    out = []

    def c(name, cin, cout, k=1, s=1, p=0):
        kh, kw = (k, k) if isinstance(k, int) else k
        ph, pw = (p, p) if isinstance(p, int) else p
        out.append((name, cin, cout, kh, kw, s, ph, pw))

    c('Conv2d_1a_3x3', 3, 32, 3, 2)
    c('Conv2d_2a_3x3', 32, 32, 3)
    c('Conv2d_2b_3x3', 32, 64, 3, 1, 1)
    c('Conv2d_3b_1x1', 64, 80)
    c('Conv2d_4a_3x3', 80, 192, 3)
    for name, cin, pf in (('Mixed_5b', 192, 32), ('Mixed_5c', 256, 64), ('Mixed_5d', 288, 64)):
        c(f'{name}.branch1x1', cin, 64)
        c(f'{name}.branch5x5_1', cin, 48)
        c(f'{name}.branch5x5_2', 48, 64, 5, 1, 2)
        c(f'{name}.branch3x3dbl_1', cin, 64)
        c(f'{name}.branch3x3dbl_2', 64, 96, 3, 1, 1)
        c(f'{name}.branch3x3dbl_3', 96, 96, 3, 1, 1)
        c(f'{name}.branch_pool', cin, pf)
    c('Mixed_6a.branch3x3', 288, 384, 3, 2)
    c('Mixed_6a.branch3x3dbl_1', 288, 64)
    c('Mixed_6a.branch3x3dbl_2', 64, 96, 3, 1, 1)
    c('Mixed_6a.branch3x3dbl_3', 96, 96, 3, 2)
    for name, c7 in (('Mixed_6b', 128), ('Mixed_6c', 160), ('Mixed_6d', 160), ('Mixed_6e', 192)):
        c(f'{name}.branch1x1', 768, 192)
        c(f'{name}.branch7x7_1', 768, c7)
        c(f'{name}.branch7x7_2', c7, c7, (1, 7), 1, (0, 3))
        c(f'{name}.branch7x7_3', c7, 192, (7, 1), 1, (3, 0))
        c(f'{name}.branch7x7dbl_1', 768, c7)
        c(f'{name}.branch7x7dbl_2', c7, c7, (7, 1), 1, (3, 0))
        c(f'{name}.branch7x7dbl_3', c7, c7, (1, 7), 1, (0, 3))
        c(f'{name}.branch7x7dbl_4', c7, c7, (7, 1), 1, (3, 0))
        c(f'{name}.branch7x7dbl_5', c7, 192, (1, 7), 1, (0, 3))
        c(f'{name}.branch_pool', 768, 192)
    c('Mixed_7a.branch3x3_1', 768, 192)
    c('Mixed_7a.branch3x3_2', 192, 320, 3, 2)
    c('Mixed_7a.branch7x7x3_1', 768, 192)
    c('Mixed_7a.branch7x7x3_2', 192, 192, (1, 7), 1, (0, 3))
    c('Mixed_7a.branch7x7x3_3', 192, 192, (7, 1), 1, (3, 0))
    c('Mixed_7a.branch7x7x3_4', 192, 192, 3, 2)
    for name, cin in (('Mixed_7b', 1280), ('Mixed_7c', 2048)):
        c(f'{name}.branch1x1', cin, 320)
        c(f'{name}.branch3x3_1', cin, 384)
        c(f'{name}.branch3x3_2a', 384, 384, (1, 3), 1, (0, 1))
        c(f'{name}.branch3x3_2b', 384, 384, (3, 1), 1, (1, 0))
        c(f'{name}.branch3x3dbl_1', cin, 448)
        c(f'{name}.branch3x3dbl_2', 448, 384, 3, 1, 1)
        c(f'{name}.branch3x3dbl_3a', 384, 384, (1, 3), 1, (0, 1))
        c(f'{name}.branch3x3dbl_3b', 384, 384, (3, 1), 1, (1, 0))
        c(f'{name}.branch_pool', cin, 192)
    return out


CONVS = _block_specs()
assert len(CONVS) == 94
SPEC = {s[0]: s for s in CONVS}


# ---------------------------------------------------------------- preprocessing
def quantize(x):
    """tools/inception_stat.py:101 on fp32: (x * 127.5 + 128).clamp(0, 255).to(torch.uint8)"""
    return (x.float() * 127.5 + 128).clamp(0, 255).to(torch.uint8)


def _taps(n_in, dtype):
    """source indices i0, i1 and weight f of the 299 output positions along an axis of n_in pixels"""
    num = torch.arange(SIZE) * n_in
    i0, f = num // SIZE, (num % SIZE).double() / SIZE
    last = i0 >= n_in - 1
    i0, f = i0.clamp(max=n_in - 1), torch.where(last, torch.zeros_like(f), f)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    return i0, i1, f.to(dtype)


def resize_closed_form(u):
    """[n, c, h, w] float -> [n, c, 299, 299]: output index o samples source coordinate o * in / 299 bilinearly, clamped to the last
    pixel (what the affine_grid / grid_sample composition below works out to; the kernel computes this)"""
    y0, y1, fy = _taps(u.shape[2], u.dtype)
    x0, x1, fx = _taps(u.shape[3], u.dtype)
    fy, fx = fy[:, None], fx[None, :]
    a, b = u[:, :, y0][:, :, :, x0], u[:, :, y0][:, :, :, x1]
    c, d = u[:, :, y1][:, :, :, x0], u[:, :, y1][:, :, :, x1]
    return (1 - fy) * ((1 - fx) * a + fx * b) + fy * ((1 - fx) * c + fx * d)


def resize_affine_grid(u):
    """the TorchScript's resize as remembered: identity theta shifted by 1/w - 1/299 (columns) and 1/h - 1/299 (rows), affine_grid and
    grid_sample(bilinear, padding_mode='border', align_corners=False) to 299 x 299"""
    n, ch, h, w = u.shape
    theta = torch.eye(2, 3, dtype=u.dtype).unsqueeze(0).repeat(n, 1, 1)
    theta[:, 0, 2] += 1.0 / w - 1.0 / SIZE
    theta[:, 1, 2] += 1.0 / h - 1.0 / SIZE
    grid = F.affine_grid(theta, [n, ch, SIZE, SIZE], align_corners=False)
    return F.grid_sample(u, grid, mode='bilinear', padding_mode='border', align_corners=False)


def preprocess(x, dtype=torch.float64):
    """[n, 3, h, w] in [-1, 1] -> network input [n, 3, 299, 299] in `dtype`: quantise, resize when the size differs, (u - 128) / 128"""
    u = quantize(x).to(dtype)
    if tuple(u.shape[2:]) != (SIZE, SIZE):
        u = resize_closed_form(u)
    return (u - 128) / 128


# ---------------------------------------------------------------- weights
def fold_bn(w, gamma, beta, mean, var, eps=EPS):
    """conv (no bias) then BatchNorm(eps) in eval mode -> (w', b') of one biased convolution"""
    s = gamma / torch.sqrt(var + eps)
    return w * s.reshape(-1, 1, 1, 1), beta - mean * s


def random_weights(seed):
    """seeded He-scaled convolution weights and BatchNorm affine parameters under torchvision's names; running statistics not included"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, cin, cout, kh, kw, *_ in CONVS:
        sd[f'{name}.conv.weight'] = torch.randn(cout, cin, kh, kw, generator=g, dtype=torch.float64) * math.sqrt(2.0 / (cin * kh * kw))
        sd[f'{name}.bn.weight'] = 1 + 0.2 * (torch.rand(cout, generator=g, dtype=torch.float64) - 0.5)
        sd[f'{name}.bn.bias'] = 0.1 * torch.randn(cout, generator=g, dtype=torch.float64)
    return sd


def folded_params(sd):
    """torchvision-named state dict (conv weight, bn weight / bias / running_mean / running_var) -> {prefix: (w, b)} in float64"""
    out = {}
    for name, *_ in CONVS:
        f = lambda k: torch.as_tensor(sd[f'{name}.{k}']).double()
        out[name] = fold_bn(f('conv.weight'), f('bn.weight'), f('bn.bias'), f('bn.running_mean'), f('bn.running_var'))
    return out


def fixture_images(z, key):
    """the fixture's u8 images [n, 3, h, w] as float32 inputs in [-1, 1]: (u + 0.5 - 128) / 127.5, the middle of u's quantisation bin,
    which `quantize` maps back to u exactly"""
    u = torch.as_tensor(np.asarray(z[key])).double()
    return ((u + 0.5 - 128) / 127.5).float()


def fixture_state_dict(z):
    """torchvision-named state dict of a fixture: random_weights(seed) plus its calibrated running statistics"""
    sd = random_weights(int(z['seed']))
    o = 0
    for name, _, cout, *_ in CONVS:
        sd[f'{name}.bn.running_mean'] = torch.from_numpy(z['bn_mean'][o:o + cout].copy()).double()
        sd[f'{name}.bn.running_var'] = torch.from_numpy(z['bn_var'][o:o + cout].copy()).double()
        o += cout
    return sd


# ---------------------------------------------------------------- network
def forward(params, x, fp16=False, taps=None):
    """network input [n, 3, 299, 299] -> features [n, 2048] in x's dtype.  params {prefix: (w, b)} folded.
    fp16=True rounds where the native path stores fp16: the input, the folded weights, every convolution / pool output.
    taps: optional dict that receives each block's output (e.g. taps['Mixed_5d'])."""
    dt = x.dtype
    r = (lambda t: t.half().to(dt)) if fp16 else (lambda t: t)

    def conv(name, t):
        _, _, _, kh, kw, s, ph, pw = SPEC[name]
        w, b = params[name]
        return r(F.relu(F.conv2d(t, r(w.to(dt)), b.to(dt), stride=s, padding=(ph, pw))))

    avg = lambda t: r(F.avg_pool2d(t, 3, 1, 1, count_include_pad=False))
    maxs2 = lambda t: F.max_pool2d(t, 3, 2)

    def block_a(p, t):
        b1 = conv(f'{p}.branch1x1', t)
        b5 = conv(f'{p}.branch5x5_2', conv(f'{p}.branch5x5_1', t))
        b3 = conv(f'{p}.branch3x3dbl_3', conv(f'{p}.branch3x3dbl_2', conv(f'{p}.branch3x3dbl_1', t)))
        return torch.cat([b1, b5, b3, conv(f'{p}.branch_pool', avg(t))], 1)

    def block_c(p, t):
        b1 = conv(f'{p}.branch1x1', t)
        b7 = conv(f'{p}.branch7x7_3', conv(f'{p}.branch7x7_2', conv(f'{p}.branch7x7_1', t)))
        d = t
        for i in range(1, 6):
            d = conv(f'{p}.branch7x7dbl_{i}', d)
        return torch.cat([b1, b7, d, conv(f'{p}.branch_pool', avg(t))], 1)

    def block_e(p, t, pool):
        b1 = conv(f'{p}.branch1x1', t)
        a = conv(f'{p}.branch3x3_1', t)
        d = conv(f'{p}.branch3x3dbl_2', conv(f'{p}.branch3x3dbl_1', t))
        return torch.cat([b1, conv(f'{p}.branch3x3_2a', a), conv(f'{p}.branch3x3_2b', a),
                          conv(f'{p}.branch3x3dbl_3a', d), conv(f'{p}.branch3x3dbl_3b', d), conv(f'{p}.branch_pool', pool(t))], 1)

    taps = {} if taps is None else taps
    t = r(x)
    for name in ('Conv2d_1a_3x3', 'Conv2d_2a_3x3', 'Conv2d_2b_3x3'):
        t = conv(name, t)
    t = conv('Conv2d_4a_3x3', conv('Conv2d_3b_1x1', maxs2(t)))
    t = maxs2(t)
    for p in ('Mixed_5b', 'Mixed_5c', 'Mixed_5d'):
        t = taps[p] = block_a(p, t)
    b3 = conv('Mixed_6a.branch3x3', t)
    d = conv('Mixed_6a.branch3x3dbl_3', conv('Mixed_6a.branch3x3dbl_2', conv('Mixed_6a.branch3x3dbl_1', t)))
    t = taps['Mixed_6a'] = torch.cat([b3, d, maxs2(t)], 1)
    for p in ('Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e'):
        t = taps[p] = block_c(p, t)
    a = conv('Mixed_7a.branch3x3_2', conv('Mixed_7a.branch3x3_1', t))
    d = t
    for i in range(1, 5):
        d = conv(f'Mixed_7a.branch7x7x3_{i}', d)
    t = taps['Mixed_7a'] = torch.cat([a, d, maxs2(t)], 1)
    t = taps['Mixed_7b'] = block_e('Mixed_7b', t, avg)
    t = taps['Mixed_7c'] = block_e('Mixed_7c', t, lambda v: F.max_pool2d(v, 3, 1, 1))
    return t.mean(dim=(2, 3))


def features(params, images, dtype=torch.float64, fp16=False, taps=None):
    """[n, 3, h, w] in [-1, 1] -> [n, 2048]: preprocess, then the network"""
    return forward(params, preprocess(images, dtype), fp16=fp16, taps=taps)


def shape_gflop():
    """multiply-adds x 2 of the 94 convolutions at 299 x 299, in GFLOP per image"""
    # output extents follow the network: trace it on meta tensors, counting each convolution's output x its kernel volume
    params = {n: (torch.empty(co, ci, kh, kw, device='meta'), torch.empty(co, device='meta')) for n, ci, co, kh, kw, *_ in CONVS}
    flops = [0.0]

    orig = F.conv2d

    def counting(t, w, b=None, stride=1, padding=0):
        o = orig(t, w, b, stride=stride, padding=padding)
        flops[0] += 2.0 * o.shape[1] * o.shape[2] * o.shape[3] * w.shape[1] * w.shape[2] * w.shape[3]
        return o

    F.conv2d = counting
    try:
        forward(params, torch.empty(1, 3, SIZE, SIZE, device='meta'))
    finally:
        F.conv2d = orig
    return flops[0] / 1e9
