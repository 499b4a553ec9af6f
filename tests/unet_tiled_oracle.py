"""fp32 forward of the reference's denoising UNet with a GroupNorm group count other than 32 and any input size the downsampling
divides -- the tiled-triplane config's GroupNorm(16) over 6 x 128 x 384 latents.  TEST INFRASTRUCTURE ONLY.

It is `oracle/unet_port.unet_forward` (same wiring, same [mmgen-memory] block bodies, same `unet_spec` block list) with the group count
as a parameter; the spec comes from `unet_port.unet_spec(image_size=min(H, W), ...)`, which places attention the way the reference
does (from min(image_size)).  tests/test_reference_pin_tiled_cpu.py pins it to the reference's own DenoisingUnetMod executed by
tests/golden/make_golden_tiled.py (widths 80 / 160, GroupNorm(16), a 16 x 48 input, head widths 40 and 80)."""
import math

import torch
import torch.nn.functional as F

from oracle import unet_port as up


def unet_forward(sd, spec, x_t, t, groups=16, num_timesteps=1000):
    """oracle/unet_port.unet_forward with GroupNorm(groups) instead of GroupNorm(32); same wiring, any input size"""
    gn = lambda key, x: F.group_norm(x, groups, sd[key + '.weight'], sd[key + '.bias'], eps=1e-5)
    emb = up.time_embedding(sd, t.float() * (1000.0 / num_timesteps), spec['base'])

    def res(b, x):
        k = b['key']
        sc = F.conv2d(x, sd[k + '.shortcut.weight'], sd[k + '.shortcut.bias']) if b['cin'] != b['cout'] else x
        h = F.conv2d(F.silu(gn(k + '.conv_1.0', x)), sd[k + '.conv_1.2.weight'], sd[k + '.conv_1.2.bias'], padding=1)
        e = F.linear(F.silu(emb), sd[k + '.norm_with_embedding.embedding_layer.1.weight'],
                     sd[k + '.norm_with_embedding.embedding_layer.1.bias'])[:, :, None, None]
        scale, shift = torch.chunk(e, 2, dim=1)
        h = gn(k + '.norm_with_embedding.norm', h) * (1 + scale) + shift
        return F.conv2d(F.silu(h), sd[k + '.conv_2.1.weight'], sd[k + '.conv_2.1.bias'], padding=1) + sc

    def attn(b, x):
        k, heads = b['key'], spec['num_heads']
        bsz, c, *sp = x.shape
        xf = x.reshape(bsz, c, -1)
        T = xf.size(-1)
        qkv = F.conv1d(gn(k + '.norm', xf), sd[k + '.qkv.weight'], sd[k + '.qkv.bias']).reshape(bsz * heads, -1, T)
        ch = qkv.shape[1] // 3
        q, kk, v = torch.chunk(qkv, 3, dim=1)
        s = 1 / math.sqrt(math.sqrt(ch))
        w = torch.softmax(torch.einsum('bct,bcs->bts', q * s, kk * s), dim=-1)
        h = torch.einsum('bts,bcs->bct', w, v).reshape(bsz, -1, T)
        return (F.conv1d(h, sd[k + '.proj.weight'], sd[k + '.proj.bias']) + xf).reshape(bsz, c, *sp)

    def run(layers, h):
        for b in layers:
            if b['type'] == 'conv_in':
                h = F.conv2d(h, sd[b['key'] + '.weight'], sd[b['key'] + '.bias'], padding=1)
            elif b['type'] == 'res':
                h = res(b, h)
            elif b['type'] == 'attn':
                h = attn(b, h)
            elif b['type'] == 'down':
                h = F.conv2d(h, sd[b['key'] + '.downsample.weight'], sd[b['key'] + '.downsample.bias'], stride=2, padding=1)
            elif b['type'] == 'up':
                h = F.conv2d(F.interpolate(h, scale_factor=2, mode='nearest'), sd[b['key'] + '.conv.weight'], sd[b['key'] + '.conv.bias'],
                             padding=1)
        return h

    h, hs = x_t, []
    for layers in spec['in_blocks']:
        h = run(layers, h)
        hs.append(h)
    h = run(spec['mid'], h)
    for layers in spec['out_blocks']:
        h = run(layers, torch.cat([h, hs.pop()], dim=1))
    return F.conv2d(F.silu(gn('out.gn', h)), sd['out.conv.weight'], sd['out.conv.bias'], padding=1)
