"""Writes tests/golden/reference_inception_v1.npz by EXECUTING torchvision's `Inception3` blocks (torchvision 0.26) in float64 on the CPU,
with the FID differences of the 2015-12-05 graph applied around them: the average pools of Mixed_5b-d, Mixed_6b-e and Mixed_7b exclude
padding from the count, and Mixed_7c's pool branch is a 3 x 3 / stride 1 / pad 1 MAX pool (pytorch-fid's FIDInceptionA / C / E_1 / E_2).

Weights: `oracle.inception_port.random_weights(SEED)` (He-scaled convolutions, BatchNorm affine parameters near identity).  BatchNorm
running statistics are calibrated in one pass over calibration images: a forward pre-hook on every BatchNorm sets its running mean /
(biased) variance to the statistics of its input, so every layer's activations stay O(1) as in a trained network.  The fixture stores
the seed and those statistics, not the weights.

Inputs go through the StyleGAN preprocessing as `oracle.inception_port.resize_affine_grid` states it (u8 quantisation, affine_grid /
grid_sample to 299, (u - 128) / 128).  The preprocessing keeps only each input's u8 quantisation, so the fixture stores the images as u8
(`u128` [2, 3, 128, 128]; `u299` [1, 3, 299, 299], a 23 x 23 image in 13 x 13 blocks, which compresses well).
`oracle.inception_port.fixture_images` turns them back into [-1, 1] inputs at the middle of each quantisation bin, which quantise to
exactly those bytes.  Also stored: the seed, the statistics (float32; the features are computed with the float32-rounded values), the
features [3, 2048] (float64) and channels 0..7 of image 0's Mixed_5d output [35, 35, 8] (float32).  The whole file is about 290 KB.

Run: python tests/golden/make_golden_inception.py"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import inception_port as ip  # noqa: E402

SEED = 20151205
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'reference_inception_v1.npz')


def fid_inception3():
    """torchvision Inception3 with the FID block semantics patched around the blocks' own forward code"""
    import torchvision
    from torchvision.models import inception as tvi
    net = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=False, transform_input=False).double().eval()
    avg_orig = F.avg_pool2d

    def avg_excl(x, kernel_size, stride=None, padding=0, ceil_mode=False, count_include_pad=True, divisor_override=None):
        return avg_orig(x, kernel_size, stride, padding, ceil_mode, False, divisor_override)

    def max_instead(x, kernel_size, stride=None, padding=0, ceil_mode=False, count_include_pad=True, divisor_override=None):
        return F.max_pool2d(x, kernel_size, stride, padding)

    def patch(block, fn):
        orig = block.forward

        def fwd(x):
            tvi.F.avg_pool2d = fn
            try:
                return orig(x)
            finally:
                tvi.F.avg_pool2d = avg_orig
        block.forward = fwd

    for name in ('Mixed_5b', 'Mixed_5c', 'Mixed_5d', 'Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e', 'Mixed_7b'):
        patch(getattr(net, name), avg_excl)
    patch(net.Mixed_7c, max_instead)
    return net


def main():
    torch.set_grad_enabled(False)
    net = fid_inception3()
    sd = ip.random_weights(SEED)
    missing, _ = net.load_state_dict({k: v for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if k.endswith('conv.weight') or k.endswith('bn.weight') or k.endswith('bn.bias')], missing

    g = torch.Generator().manual_seed(SEED + 1)

    def smooth_images(n, h, w):
        # low-frequency colour fields plus noise, in [-1, 1]: image-like inputs for calibration and the fixture
        base = F.interpolate(torch.rand(n, 3, 8, 8, generator=g, dtype=torch.float64) * 2 - 1, size=(h, w), mode='bicubic',
                             align_corners=False)
        return (base + 0.15 * torch.randn(n, 3, h, w, generator=g, dtype=torch.float64)).clamp(-1, 1).float()

    def prep(x):
        u = ip.quantize(x).double()
        if tuple(u.shape[2:]) != (ip.SIZE, ip.SIZE):
            u = ip.resize_affine_grid(u)
        return (u - 128) / 128

    hooks = []

    def calib(mod, inp):
        x = inp[0]
        mod.running_mean.copy_(x.mean(dim=(0, 2, 3)))
        mod.running_var.copy_(x.var(dim=(0, 2, 3), unbiased=False))

    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eps = ip.EPS
            hooks.append(m.register_forward_pre_hook(calib))
    net(prep(smooth_images(6, 128, 128)))
    for h in hooks:
        h.remove()
    for m in net.modules():                 # the fixture stores float32 statistics: compute with exactly those
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.copy_(m.running_mean.float().double())
            m.running_var.copy_(m.running_var.float().double())

    feats = {}
    net.avgpool.register_forward_hook(lambda m, i, o: feats.__setitem__('f', o.flatten(1)))
    net.Mixed_5d.register_forward_hook(lambda m, i, o: feats.__setitem__('m5d', o))
    u128 = ip.quantize(smooth_images(2, 128, 128)).numpy()
    # 299 = 23 x 13: a 23 x 23 image blown up into 13 x 13 blocks (sharp block edges, and a fixture that stays small)
    u299 = ip.quantize(smooth_images(1, 23, 23)).repeat_interleave(13, 2).repeat_interleave(13, 3).numpy()
    x128 = ip.fixture_images(dict(u128=u128), 'u128')
    x299 = ip.fixture_images(dict(u299=u299), 'u299')
    net(prep(x128))
    f128, m5d = feats['f'].clone(), feats['m5d'][0, :8].permute(1, 2, 0).clone()
    net(prep(x299))
    f299 = feats['f'].clone()

    st = net.state_dict()
    names = [c[0] for c in ip.CONVS]
    np.savez_compressed(
        OUT, seed=np.int64(SEED),
        bn_mean=np.concatenate([st[f'{n}.bn.running_mean'].float().numpy() for n in names]),
        bn_var=np.concatenate([st[f'{n}.bn.running_var'].float().numpy() for n in names]),
        u128=u128, u299=u299, feat128=f128.numpy(), feat299=f299.numpy(), mixed_5d=m5d.float().numpy(),
        torchvision=np.array(__import__('torchvision').__version__))
    print(OUT, os.path.getsize(OUT), 'bytes, feature norms', f128.norm(dim=1).tolist(), f299.norm(dim=1).tolist())


if __name__ == '__main__':
    main()
