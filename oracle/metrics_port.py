"""CPU restatements of the reference's evaluation metrics (TEST INFRASTRUCTURE): SSIM and LPIPS(VGG16) as
lib/core/evaluation/metrics.py:58-71 calls them from lib/models/autodecoders/base_nerf.py:555-572.

Provenance: neither skimage nor lpips is installed here, so no fixture could come from executing them.  Both functions are pinned to the
published formulas of the versions the reference requires, not to an execution:
  * skimage >= 0.19 `structural_similarity(p, t, channel_axis=0, data_range=1)`: 7 x 7 `scipy.ndimage.uniform_filter` (mode 'reflect'),
    sample covariance (49 / 48), C1 = (0.01)^2, C2 = (0.03)^2, mean of S over [3:h-3, 3:w-3] per channel, then over the channels.
    With float32 inputs skimage computes in float32 (the filters accumulate in double but store float32), as `ssim_skimage(..., np.float32)` does.
  * lpips 0.1.4 `LPIPS(net='vgg', version='0.1')`: ScalingLayer on 2 x - 1, torchvision VGG16 features[0:30] tapped after relu1_2, relu2_2,
    relu3_3, relu4_3, relu5_3, per-pixel channel normalisation f / (sqrt(sum_c f^2) + 1e-10), squared difference, 1 x 1 `lin{k}` (no
    bias), spatial mean, sum over the taps.
Images are channels-last [n, h, w, 3] in [0, 1], as the package's renderer writes them."""
import numpy as np
import torch
import torch.nn.functional as F
from scipy.ndimage import uniform_filter

VGG_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)          # torchvision vgg16.features indices of the 13 convolutions
VGG_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAP_AFTER = (1, 3, 6, 9, 12)                                           # conv position (0-based) whose ReLU output is a tap
TAP_CHANNELS = (64, 128, 256, 512, 512)
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)


def ssim_skimage(p, t, dtype=np.float64):
    """per-image SSIM of p, t [n, h, w, 3] (numpy or torch) in `dtype` -> float64 [n]"""
    p, t = (np.asarray(torch.as_tensor(a).cpu().numpy() if isinstance(a, torch.Tensor) else a) for a in (p, t))
    n = p.shape[0]
    out = np.empty(n, np.float64)
    NP = 49
    cov_norm = NP / (NP - 1)
    C1, C2 = (0.01 * 1) ** 2, (0.03 * 1) ** 2
    for i in range(n):
        vals = []
        for c in range(3):
            X, Y = p[i, :, :, c].astype(dtype), t[i, :, :, c].astype(dtype)
            ux, uy = uniform_filter(X, size=7), uniform_filter(Y, size=7)
            uxx, uyy, uxy = uniform_filter(X * X, size=7), uniform_filter(Y * Y, size=7), uniform_filter(X * Y, size=7)
            vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
            A1, A2, B1, B2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
            S = (A1 * A2) / (B1 * B2)
            vals.append(S[3:-3, 3:-3].mean(dtype=np.float64))
        out[i] = np.mean(vals)
    return out


def vgg_layers(vgg_sd, lin_sd, dtype=torch.float64):
    """(conv weights, biases, lin weights) from torchvision's vgg16 state dict and lpips' v0.1 vgg.pth"""
    ws = [vgg_sd[f'features.{i}.weight'].to(dtype) for i in VGG_CONVS]
    bs = [vgg_sd[f'features.{i}.bias'].to(dtype) for i in VGG_CONVS]
    lins = [lin_sd[f'lin{k}.model.1.weight'].to(dtype) for k in range(5)]
    return ws, bs, lins


def lpips_vgg(p, t, vgg_sd, lin_sd, dtype=torch.float64, fp16_storage=False):
    """per-image LPIPS of p, t [n, h, w, 3] in [0, 1] -> [n] (torch, `dtype`).
    fp16_storage: round what the GPU path stores in fp16 -- the scaled input, every post-ReLU map and the conv weights -- to fp16 (a
    precision probe of the native path; arithmetic stays in `dtype`)."""
    rt = (lambda x: x.half().to(dtype)) if fp16_storage else (lambda x: x)
    ws, bs, lins = vgg_layers(vgg_sd, lin_sd, dtype)
    shift = torch.tensor(SHIFT, dtype=dtype).view(1, 3, 1, 1)
    scale = torch.tensor(SCALE, dtype=dtype).view(1, 3, 1, 1)

    def feats(img):
        x = torch.as_tensor(img).cpu().to(dtype).permute(0, 3, 1, 2)
        x = rt(((2 * x - 1) - shift) / scale)
        taps = []
        for li, (w, b) in enumerate(zip(ws, bs)):
            if li in (2, 4, 7, 10):
                x = F.max_pool2d(x, 2, 2)
            x = rt(F.relu(F.conv2d(x, rt(w), b, padding=1)))
            if li in TAP_AFTER:
                taps.append(x)
        return taps

    fp, ft = feats(p), feats(t)
    total = 0
    for a, b, lw in zip(fp, ft, lins):
        na = a / (a.square().sum(dim=1, keepdim=True).sqrt() + 1e-10)
        nb = b / (b.square().sum(dim=1, keepdim=True).sqrt() + 1e-10)
        total = total + F.conv2d((na - nb).square(), lw).mean(dim=(2, 3))[:, 0]
    return total


def random_weights(seed=0):
    """VGG16 / lin state dicts in the two on-disk key formats: Kaiming-normal fan-out weights (torchvision's VGG initialisation, so
    activations keep a realistic scale), small random biases (so the bias path is exercised) and non-negative lin heads; for tests and
    timing, where the pretrained values do not matter"""
    g = torch.Generator().manual_seed(seed)
    vgg, cin = {}, 3
    for i, cout in zip(VGG_CONVS, VGG_CHANNELS):
        std = (2.0 / (cout * 9)) ** 0.5
        vgg[f'features.{i}.weight'] = torch.randn(cout, cin, 3, 3, generator=g) * std
        vgg[f'features.{i}.bias'] = torch.randn(cout, generator=g) * 0.01
        cin = cout
    lin = {f'lin{k}.model.1.weight': torch.rand(1, c, 1, 1, generator=g) * (4.0 / c) for k, c in enumerate(TAP_CHANNELS)}
    return vgg, lin


def synthetic_pairs(n, h, w, seed=0):
    """(pred, target) float32 [n, h, w, 3] in [0, 1]: smooth random targets (low-frequency sinusoids), predictions = an 8-bit-quantised
    blurred, noisy copy -- the statistics of a rendered test view against its ground truth"""
    g = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing='ij')
    tgt = np.empty((n, h, w, 3), np.float64)
    for i in range(n):
        for c in range(3):
            f = 0.5 + 0.1 * g.standard_normal()
            for _ in range(4):
                kx, ky, ph = g.uniform(0.5, 6, size=2).tolist() + [g.uniform(0, 2 * np.pi)]
                f = f + 0.12 * g.standard_normal() * np.sin(2 * np.pi * (kx * xx + ky * yy) + ph)
            tgt[i, :, :, c] = f
    tgt = np.clip(tgt, 0, 1)
    pred = uniform_filter(tgt, size=(1, 3, 3, 1)) + 0.03 * g.standard_normal(tgt.shape)
    pred = np.round(np.clip(pred, 0, 1) * 255) / 255
    return pred.astype(np.float32), tgt.astype(np.float32)
