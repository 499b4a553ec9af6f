"""LPIPS(VGG16) of lpips 0.1.4 (`lpips.LPIPS(net='vgg', version='0.1')`, the reference's `test_lpips`, lib/core/evaluation/metrics.py:58-71)
on the package's own kernels: the 13 VGG16 convolutions run on the wgmma implicit-GEMM convolution with the ReLU in its epilogue, and the
scaling layer, the five taps (channel normalisation, squared difference, lin{k}, spatial mean) and the max-pools on csrc/eval_metrics.cu.

The weights are external assets and are never downloaded here:
  * torchvision's ImageNet VGG16, `vgg16-397923af.pth` (keys `features.{0,2,5,...,28}.{weight,bias}`), looked for in
    `torch.hub.get_dir()/checkpoints/` where torchvision / lpips cache it;
  * lpips' linear heads, `weights/v0.1/vgg.pth` inside an installed `lpips` package (keys `lin{0..4}.model.1.weight`, [1, C, 1, 1]),
    located with `importlib.util.find_spec` (lpips is not imported).
Either can be passed explicitly: `LPIPS(vgg_path=..., lin_path=...)`."""
import importlib.util
import os

import torch

from . import _lib as N
from . import unet_ops as U

VGG_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)          # vgg16.features indices of the 13 convolutions
VGG_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAP_AFTER = (1, 3, 6, 9, 12)            # convolutions whose ReLU output is tapped (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3)
TAP_CHANNELS = (64, 128, 256, 512, 512)
IN_CHANNELS = 16                        # the scaled RGB input, zero-padded for the narrow-channel GEMM family
DEFAULT_WORKSPACE_BYTES = 1 << 30


def default_paths():
    """(vgg_path, lin_path) where torchvision / lpips keep the weights; lin_path is None when lpips is not installed"""
    vgg = os.path.join(torch.hub.get_dir(), 'checkpoints', 'vgg16-397923af.pth')
    spec = importlib.util.find_spec('lpips')
    lin = None
    if spec is not None and spec.origin:
        lin = os.path.join(os.path.dirname(spec.origin), 'weights', 'v0.1', 'vgg.pth')
    return vgg, lin


def default_files_exist():
    vgg, lin = default_paths()
    return lin is not None and os.path.isfile(vgg) and os.path.isfile(lin)


def _load(path, expected):
    """state dict of `path` with every key of `expected` ({key: shape}) present at that shape (other keys are ignored)"""
    sd = torch.load(path, map_location='cpu', weights_only=True)
    if not isinstance(sd, dict):
        raise ValueError(f'{path}: expected a state dict, got {type(sd).__name__}')
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f'{path}: missing key {k!r}')
        if tuple(sd[k].shape) != tuple(shape):
            raise ValueError(f'{path}: key {k!r} has shape {tuple(sd[k].shape)}, expected {tuple(shape)}')
    return {k: sd[k].float() for k in expected}


def _levels(h, w):
    return [(h >> l, w >> l) for l in range(5)]


def supported(h, w):
    """the five VGG levels are whole (h, w multiples of 16) and every level's convolution boxes tile it (128-pixel boxes)"""
    if h <= 0 or w <= 0 or h % 16 or w % 16:
        return False
    for l, (hl, wl) in enumerate(_levels(h, w)):
        b1, b2, b3 = U._conv_boxes(hl, wl, narrow=l == 0)
        if b1 * b2 * b3 != 128:
            return False
        if l == 0:
            b1, b2, b3 = U._conv_boxes(hl, wl)
            if b1 * b2 * b3 != 128:
                return False
    return True


def pair_bytes(h, w):
    """workspace bytes per (pred, target) pair: two ping-pong maps of the largest level (64 channels at h x w, fp16) per image"""
    return 2 * 2 * h * w * 64 * 2


class LPIPS:
    """LPIPS(vgg_path=None, lin_path=None)(pred, target) -> [n] fp32.

    pred, target: [n, h, w, 3] fp32 in [0, 1] (channels-last, as the renderer writes them) on the current CUDA device.  Pairs run
    `chunk` at a time, with chunk = workspace_bytes // pair_bytes(h, w); a pair's result does not depend on the chunk it ran in."""

    def __init__(self, vgg_path=None, lin_path=None, workspace_bytes=DEFAULT_WORKSPACE_BYTES):
        dv, dl = default_paths()
        vgg_path = vgg_path or dv
        lin_path = lin_path or dl
        if lin_path is None:
            raise FileNotFoundError('LPIPS: no lin_path given and the lpips package (which ships weights/v0.1/vgg.pth) is not installed')
        for p in (vgg_path, lin_path):
            if not os.path.isfile(p):
                raise FileNotFoundError(f'LPIPS: weight file {p} not found')
        expect, cin = {}, 3
        for i, cout in zip(VGG_CONVS, VGG_CHANNELS):
            expect[f'features.{i}.weight'] = (cout, cin, 3, 3)
            expect[f'features.{i}.bias'] = (cout,)
            cin = cout
        vgg = _load(vgg_path, expect)
        lin = _load(lin_path, {f'lin{k}.model.1.weight': (1, c, 1, 1) for k, c in enumerate(TAP_CHANNELS)})
        self.vgg_path, self.lin_path = vgg_path, lin_path
        self.workspace_bytes = int(workspace_bytes)
        self._host = dict(
            w=[U.pack_conv_weight(vgg[f'features.{i}.weight'], cin_pad=IN_CHANNELS, narrow=True) if li == 0 else
               U.pack_conv_weight(vgg[f'features.{i}.weight']) for li, i in enumerate(VGG_CONVS)],
            b=[vgg[f'features.{i}.bias'].contiguous() for i in VGG_CONVS],
            lin=[lin[f'lin{k}.model.1.weight'].reshape(-1).contiguous() for k in range(5)])
        self._dev = {}
        self._ws = None

    def _weights(self, device):
        if device not in self._dev:
            self._dev[device] = {k: [t.to(device) for t in v] for k, v in self._host.items()}
        return self._dev[device]

    def chunk(self, h, w):
        return max(1, self.workspace_bytes // pair_bytes(h, w))

    @torch.no_grad()
    def __call__(self, pred, target):
        N.require_cuda(pred, target)
        if pred.shape != target.shape or pred.dim() != 4 or pred.shape[-1] != 3:
            raise ValueError(f'LPIPS: pred and target must both be [n, h, w, 3], got {tuple(pred.shape)} and {tuple(target.shape)}')
        n, h, w, _ = pred.shape
        if not supported(h, w):
            raise NotImplementedError(f'LPIPS: {h} x {w} images are not supported (h and w must be multiples of 16 whose five VGG levels '
                                      'the 128-pixel convolution boxes tile, e.g. 128 x 128, 64 x 64, 32 x 32)')
        pred, target = pred.float().contiguous(), target.float().contiguous()
        dev = pred.device
        W = self._weights(dev)
        out = torch.zeros(n, dtype=torch.float32, device=dev)
        cm = min(n, self.chunk(h, w))
        per_img = h * w * 64
        if self._ws is None or self._ws.device != dev or self._ws.numel() < 2 * 2 * cm * per_img:
            self._ws = torch.empty(2 * 2 * cm * per_img, dtype=torch.float16, device=dev)
        bufs = (self._ws[:2 * cm * per_img], self._ws[2 * cm * per_img:4 * cm * per_img])
        L, s = N.lib(), N.stream_ptr()
        npart = max(L.ssdnerf_lpips_tap_partials(N.c_u32(cm), N.c_u32(hl), N.c_u32(wl), N.c_u32(c), N.c_int(int(k < 4)))
                    for k, ((hl, wl), c) in enumerate(zip(_levels(h, w), TAP_CHANNELS)))
        partial = torch.empty(npart, dtype=torch.float32, device=dev)
        for j0 in range(0, n, cm):
            m = min(cm, n - j0)
            B = 2 * m
            cur = 0
            N.check(L.ssdnerf_lpips_prep_f16(N.ptr(pred[j0:j0 + m]), N.ptr(target[j0:j0 + m]), N.c_u32(m), N.c_u32(h), N.c_u32(w),
                                             N.ptr(bufs[cur]), s))
            hl, wl, cin, tap = h, w, IN_CHANNELS, 0
            for li, cout in enumerate(VGG_CHANNELS):
                x = bufs[cur][:B * hl * wl * cin].view(B, hl, wl, cin)
                y = bufs[1 - cur][:B * hl * wl * cout].view(B, hl, wl, cout)
                U.conv3x3_f16(x, W['w'][li], cout, bias=W['b'][li], out=y, narrow=li == 0, relu=True)
                cur, cin = 1 - cur, cout
                if li in TAP_AFTER:
                    pool = tap < 4
                    pooled = bufs[1 - cur] if pool else None
                    N.check(L.ssdnerf_lpips_tap_f16(N.ptr(y), N.c_u32(m), N.c_u32(hl), N.c_u32(wl), N.c_u32(cout), N.ptr(W['lin'][tap]),
                                                    N.ptr(partial), N.ptr(pooled), N.ptr(out[j0:j0 + m]), s))
                    if pool:
                        cur, hl, wl = 1 - cur, hl // 2, wl // 2
                    tap += 1
        return out
