"""The tiled-triplane denoiser's oracle and state-dict layout pinned to the reference's own DenoisingUnetMod
(tests/golden/reference_tiled_v1.npz, written by tests/golden/make_golden_tiled.py: widths 80 / 160, GroupNorm(16), a 16 x 48
input with image_size [16, 48], attention at head widths 40 and 80).  Same [mmgen-memory] caveat as tests/test_reference_pin_cpu.py:
the reference's constructor and forward wiring are pinned, the inner bodies of the mmgen-inherited blocks are a restatement."""
import os

import numpy as np
import torch

from oracle import unet_port as up
from tests import unet_tiled_oracle as uto
from tests.common import GOLDEN, parse_shapes, seeded_weights

CFG = dict(image_size=[16, 48], in_channels=6, base_channels=80, channels_cfg=[1, 2], resblocks_per_downsample=1, num_heads=2,
           attention_res=[16, 8], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True)


def _fixture():
    return np.load(os.path.join(GOLDEN, 'reference_tiled_v1.npz'))


def _spec():
    return up.unet_spec(image_size=16, in_channels=6, base_channels=80, channels_cfg=(1, 2), resblocks_per_downsample=1,
                        attention_res=(16, 8), num_heads=2)


def _weights(z):
    return seeded_weights(list(z['keys']), parse_shapes(z['shapes']), int(z['weight_seed']))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def test_package_state_dict_keys_match_reference():
    """DenoisingUnetMod of this package, built from the same constructor arguments, has the reference's keys and shapes in order"""
    from ssdnerf_b200.unet import DenoisingUnetMod
    z = _fixture()
    sd = DenoisingUnetMod(**CFG).state_dict()
    assert list(sd.keys()) == list(z['keys'])
    assert [tuple(v.shape) for v in sd.values()] == parse_shapes(z['shapes'])
    assert sum(1 for b in _spec()['in_blocks'] + [_spec()['mid']] + _spec()['out_blocks'] for l in b if l['type'] == 'attn') == \
        sum(1 for k in z['keys'] if k.endswith('.qkv.weight'))


def test_tiled_oracle_forward_matches_reference():
    z = _fixture()
    sd = _weights(z)
    with torch.no_grad():
        y = uto.unet_forward(sd, _spec(), torch.from_numpy(z['x']), torch.from_numpy(z['t']))
    assert _rel(y, z['y']) < 1e-5, _rel(y, z['y'])


def test_tiled_oracle_input_gradient_matches_reference():
    z = _fixture()
    sd = _weights(z)
    x = torch.from_numpy(z['x']).clone().requires_grad_(True)
    (uto.unet_forward(sd, _spec(), x, torch.from_numpy(z['t'])) * torch.from_numpy(z['r'])).sum().backward()
    assert _rel(x.grad, z['dx']) < 1e-5, _rel(x.grad, z['dx'])


def test_tiled_oracle_needs_the_group_count():
    """the fixture discriminates GroupNorm(16) from the paper configs' GroupNorm(32)-style normalisation over other groupings"""
    z = _fixture()
    sd = _weights(z)
    with torch.no_grad():
        y8 = uto.unet_forward(sd, _spec(), torch.from_numpy(z['x']), torch.from_numpy(z['t']), groups=8)
    assert _rel(y8, z['y']) > 1e-3
