"""Generates tests/golden/reference_tiled_v1.npz by RUNNING THE REFERENCE'S OWN DenoisingUnetMod at a tiled-triplane-style shape
(build container only: `python tests/golden/make_golden_tiled.py`; the fixture is committed).

It loads lib/models/architecture/ddpm/{modules,denoising}.py from the reference with mmcv / mmgen stubbed exactly as
tests/golden/make_golden_ref.py does (same stubs, same [mmgen-memory] caveat: the constructor, the block wiring, the skip concat
order, the attention placement from min(image_size) and the legacy head layout are the reference's own code; the bodies of the
mmgen-inherited blocks are the memory restatement of SURVEY.md Appendix B).  The model has what sets the tiled config
(configs/new_cfgs/ssdnerf_cars_recons1v_tiled.py) apart from the paper configs, at a size a CPU runs in seconds:

  widths 80 / 160 (multiples of 16, not of 64), GroupNorm(16) (groups of 5 and 10 channels), a non-square 16 x 48 input with
  image_size [16, 48], attention at 16 x 48 (head width 40, T = 768) and 8 x 24 (head width 80, T = 192), 6 input channels.

Stored: state-dict keys / shapes and the weight seed (tests/common.py:seeded_weights regenerates the weights), the input, the
timesteps, the forward output and d (out . r) / d x.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden_ref import load_reference, seeded_state_dict  # noqa: E402

TILED_CFG = dict(image_size=[16, 48], in_channels=6, base_channels=80, channels_cfg=[1, 2], resblocks_per_downsample=1, dropout=0.0,
                 use_scale_shift_norm=True, downsample_conv=True, upsample_conv=True, num_heads=2, attention_res=[16, 8],
                 norm_cfg=dict(type='GN', num_groups=16))
SEED = 13


def main():
    mods, den, gd, sm = load_reference()
    torch.manual_seed(0)
    unet = den.DenoisingUnetMod(**TILED_CFG)
    sd = seeded_state_dict(unet, seed=SEED)
    unet.load_state_dict(sd)
    unet.eval()
    out = {}
    keys = list(sd.keys())
    out['keys'] = np.array(keys)
    out['shapes'] = np.array([','.join(map(str, sd[k].shape)) for k in keys])
    out['weight_seed'] = np.array(SEED)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 6, 16, 48, generator=g)
    t = torch.tensor([999, 17])
    with torch.no_grad():
        out['x'], out['t'] = x.numpy(), t.numpy()
        out['y'] = unet(x, t).numpy()
    xr = x.clone().requires_grad_(True)
    r = torch.randn(2, 6, 16, 48, generator=g)
    (unet(xr, t) * r).sum().backward()
    out['r'], out['dx'] = r.numpy(), xr.grad.numpy()
    np.savez_compressed(os.path.join(HERE, 'reference_tiled_v1.npz'), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
