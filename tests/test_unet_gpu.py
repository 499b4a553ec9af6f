"""UNet / DDIM on the GPU (wgmma GEMMs, fp16 operands + activation storage, fp32 accumulation) vs the fp32 oracle
(oracle/unet_port.py, pinned to the reference's own code by tests/test_reference_pin_cpu.py).

Tolerance.  BASELINE.json north_star: "denoised triplanes within 1e-3 relative fp16 tolerance".  An fp32 oracle cannot be matched to
1e-3 by ANY single-pass 10/11-bit-mantissa tensor-core path: tests/perf/precision_probe.py injects
the roundings one at a time into the fp32 oracle at full size -- fp16 GEMM operands alone 1.28e-3, the reference's own default
(cuDNN TF32 convolutions, SURVEY.md Appendix C) 1.28e-3, fp16 storage of h1 +0.62e-3, of the residual stream +0.67e-3 (RSS total
1.54e-3).  The bars below are therefore stated against that floor: one evaluation <= 2.0e-3 relative L2,
i.e. within 1.2x of the reference's own TF32 deviation from fp32.  The quantity north_star actually names -- the
DENOISED TRIPLANE, i.e. the output of the whole 50-step chain -- is within 1e-3 at full size (the sampler is contractive,
per-evaluation noise does not accumulate), asserted below."""
import math

import numpy as np
import pytest
import torch

from oracle import unet_port as up

pytestmark = pytest.mark.gpu

SMALL = dict(image_size=32, in_channels=18, base_channels=64, channels_cfg=[1, 2, 2], resblocks_per_downsample=1,
             num_heads=2, attention_res=[16, 8], use_scale_shift_norm=True)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _build(cfg, sd, cuda):
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(**cfg)
    missing = m.load_state_dict(sd, strict=True)
    return m.to(cuda).eval()


def test_glue_kernels(cuda):
    """GroupNorm (+scale/shift, SiLU) over a channel concat, softmax vs torch"""
    from ssdnerf_b200 import _lib as N
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(0)
    B, H, W, C1, C2 = 3, 16, 16, 512, 256
    x1 = torch.randn(B, H, W, C1, generator=g).half().to(cuda)
    x2 = (torch.randn(B, H, W, C2, generator=g) * 2 + 0.5).half().to(cuda)
    C = C1 + C2
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    ss = torch.randn(B, 2 * C, generator=g).to(cuda) * 0.3
    stats = torch.zeros(B, 32, 2, device=cuda)
    out = torch.empty(B, H, W, C, dtype=torch.float16, device=cuda)
    L, s = N.lib(), N.stream_ptr()
    N.check(L.ssdnerf_gn_stats(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(32), N.ptr(stats), s))
    N.check(L.ssdnerf_gn_apply(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(32), N.ptr(stats),
                               N.ptr(gamma), N.ptr(beta), N.ptr(ss), N.c_longlong(2 * C), N.c_f32(1e-5), N.c_int(1), N.ptr(out), s))
    xc = torch.cat([x1, x2], -1).float().permute(0, 3, 1, 2)
    ref = F.group_norm(xc, 32, gamma, beta, 1e-5) * (1 + ss[:, :C, None, None]) + ss[:, C:, None, None]
    ref = F.silu(ref).permute(0, 2, 3, 1)
    assert (out.float() - ref).abs().max().item() < 2e-2 and _rel_l2(out.float().cpu(), ref.cpu()) < 2e-3
    S = torch.randn(64, 256, generator=g).to(cuda) * 4
    P = torch.empty(64, 256, dtype=torch.float16, device=cuda)
    N.check(L.ssdnerf_softmax_rows(N.ptr(S), N.c_u32(64), N.c_u32(256), N.ptr(P), s))
    assert (P.float() - torch.softmax(S, -1)).abs().max().item() < 1e-3


def test_attention_block_matches_oracle(cuda):
    spec = up.unet_spec(**{k: v for k, v in SMALL.items() if k != 'use_scale_shift_norm'})
    sd = up.random_state_dict(spec, seed=3, std=0.05)
    m = _build(SMALL, sd, cuda)
    eng = m.engine(2, cuda)
    kind, d = eng.mid_seq[1]
    assert kind == 'attn'
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 128, 8, 8, generator=g)
    xh = x.permute(0, 2, 3, 1).contiguous().half().to(cuda)
    xq = xh.float().view(2, 64, 32, 4)                 # quad statistics the producing GEMM epilogue would have emitted
    q = torch.stack([xq.sum(dim=(1, 3)), (xq * xq).sum(dim=(1, 3))], dim=-1).contiguous()
    y, _ = eng._attn(d, (xh, q), ('t',))
    ref = up.attention(sd, dict(key='mid_blocks.1', c=128), x.half().float(), 2)
    assert _rel_l2(y.float().cpu().permute(0, 3, 1, 2), ref) < 3e-3


@pytest.mark.parametrize('B', [1, 3])
def test_small_unet_forward(cuda, B):
    spec = up.unet_spec(**{k: v for k, v in SMALL.items() if k != 'use_scale_shift_norm'})
    sd = up.random_state_dict(spec, seed=1, std=0.04)
    m = _build(SMALL, sd, cuda)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, 18, 32, 32, generator=g)
    t = torch.tensor([999, 500, 19][:B])
    ref = up.unet_forward(sd, spec, x, t)
    out = m(x.to(cuda), t.to(cuda)).cpu()
    err = _rel_l2(out, ref)
    print('small unet rel l2', err)
    assert out.shape == ref.shape and err < 2e-3


def test_ddim_graph_equals_eager_and_tracks_oracle(cuda):
    from ssdnerf_b200.diffusion import GaussianDiffusion
    spec = up.unet_spec(**{k: v for k, v in SMALL.items() if k != 'use_scale_shift_norm'})
    sd = up.random_state_dict(spec, seed=5, std=0.04)
    m = _build(SMALL, sd, cuda)
    diff = GaussianDiffusion(m, betas_cfg=dict(type='linear'), num_timesteps=1000,
                             test_cfg=dict(num_timesteps=8, clip_range=[-2, 2])).to(cuda)
    g = torch.Generator().manual_seed(6)
    noise = torch.randn(2, 18, 32, 32, generator=g)
    a = diff(noise.to(cuda), return_loss=False, use_graph=True).cpu()
    b = diff(noise.to(cuda), return_loss=False, use_graph=False).cpu()
    # same kernels in the same order; only the fp32 atomics of the GroupNorm statistics are order-dependent
    assert _rel_l2(a, b) < 1e-3
    dv = up.diffusion_vars(up.linear_betas())
    ref = up.ddim_sample(lambda x, t: up.unet_forward(sd, spec, x, t), noise, dv, num_timesteps=8)
    err = _rel_l2(a, ref)
    print('ddim 8 steps rel l2', err)
    assert err < 1e-3          # north_star: denoised triplanes within 1e-3 relative
    # schedule tables equal the oracle's float64 restatement
    np.testing.assert_array_equal(diff.alphas_bar, dv['alphas_bar'])
    assert torch.equal(diff.ddim_timesteps(50), up.ddim_timesteps(1000, 50))


def test_full_unet_one_step_vs_oracle(cuda):
    """the 122.4 M-parameter UNet of ssdnerf_cars_uncond, one evaluation at B=1 against the fp32 CPU oracle"""
    full = dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
                num_heads=4, attention_res=[32, 16, 8], use_scale_shift_norm=True)
    spec = up.unet_spec()
    sd = up.random_state_dict(spec, seed=7, std=0.02)
    m = _build(full, sd, cuda)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(1, 18, 128, 128, generator=g)
    t = torch.tensor([659])
    out = m(x.to(cuda), t.to(cuda)).cpu()
    torch.set_num_threads(max(torch.get_num_threads(), 8))
    ref = up.unet_forward(sd, spec, x, t)
    err = _rel_l2(out, ref)
    print('full unet rel l2', err)
    assert err < 2e-3


def test_full_size_50_step_ddim_vs_fp32_oracle(cuda):
    """ssdnerf_cars_uncond UNet, the whole 50-step DDIM chain at B=1: captured-graph loop vs the fp32 oracle chain.  The oracle runs
    on the same GPU in strict fp32 (TF32 off): 50 x 218 GFLOP would take minutes on host cores."""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    full = dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
                num_heads=4, attention_res=[32, 16, 8], use_scale_shift_norm=True)
    spec = up.unet_spec()
    sd = up.random_state_dict(spec, seed=7, std=0.02)
    m = _build(full, sd, cuda)
    diff = GaussianDiffusion(m, betas_cfg=dict(type='linear'), num_timesteps=1000, test_cfg=dict(num_timesteps=50, clip_range=[-2, 2])).to(cuda)
    g = torch.Generator().manual_seed(9)
    noise = torch.randn(1, 18, 128, 128, generator=g)
    out = diff(noise.to(cuda), return_loss=False).cpu()
    up.fp32_reference_mode()
    sdg = up.state_dict_to(sd, cuda)
    dv = up.diffusion_vars(up.linear_betas())
    with torch.no_grad():
        # cross-check the GPU-resident oracle against the CPU oracle on one evaluation (same arithmetic, different library kernels)
        x1 = torch.randn(1, 18, 128, 128, generator=g)
        t1 = torch.tensor([400])
        a = up.unet_forward(sdg, spec, x1.to(cuda), t1.to(cuda)).cpu()
        b = up.unet_forward(sd, spec, x1, t1)
        assert _rel_l2(a, b) < 2e-5, _rel_l2(a, b)
        ref = up.ddim_sample(lambda x, t: up.unet_forward(sdg, spec, x, t.to(x.device)), noise.to(cuda), dv, num_timesteps=50, clip_range=(-2, 2)).cpu()
    err = _rel_l2(out, ref)
    print('full-size 50-step DDIM rel l2', err, 'max abs', float((out - ref).abs().max()), 'ref rms', float(ref.pow(2).mean().sqrt()))
    assert err < 1e-3          # north_star: denoised triplanes within 1e-3 relative


def test_fused_quad_stats_match_tensor(cuda):
    """GroupNorm statistics emitted by the GEMM epilogue (conv, 8x8 two-images-per-tile conv, flattened-row GEMM) == sums of the
    fp32 accumulator values (the statistics are taken before the fp16 rounding of the stored activation)"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(31)
    for (B, H, Cin, Cout) in [(3, 32, 128, 256), (5, 8, 256, 512), (2, 64, 64, 128)]:
        x = torch.randn(B, H, H, Cin, generator=g).half().to(cuda)
        w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
        q = torch.zeros(B, Cout // 4, 2, device=cuda)
        wp = U.pack_conv_weight(w).to(cuda)
        out = U.conv3x3_f16(x, wp, Cout, qstats=q)
        o = U.conv3x3_f16(x, wp, Cout, out_f32=True).view(B, H * H, Cout // 4, 4)
        assert torch.equal(out, o.half().view_as(out))
        ref = torch.stack([o.sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))], dim=-1)
        torch.testing.assert_close(q, ref, rtol=1e-3, atol=5e-3)
    B, T, c = 3, 64, 512
    a = torch.randn(B * T, c, generator=g).half().to(cuda)
    wl = U.pack_linear_weight(torch.randn(c, c, generator=g) * 0.05).to(cuda)
    q = torch.zeros(B, c // 4, 2, device=cuda)
    out = U.linear_f16(a, wl, n=c, qstats=q, stats_hw=T)
    o = U.linear_f16(a, wl, n=c, out_f32=True).view(B, T, c // 4, 4)
    assert torch.equal(out, o.half().view_as(out))
    ref = torch.stack([o.sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))], dim=-1)
    torch.testing.assert_close(q, ref, rtol=1e-3, atol=5e-3)


@pytest.mark.parametrize("T,heads,ch", [(1024, 4, 64), (256, 4, 128), (64, 2, 128), (128, 1, 64), (1024, 8, 128), (2048, 2, 64)])
def test_flash_attention_matches_fp32_reference(cuda, T, heads, ch):
    """fused attention (scores never materialised) vs fp32 softmax attention on the same fp16 qkv, legacy head layout
    (modules.py:36-48); tolerance = fp16 rounding of P and of the output (2e-3 relative to the output range)."""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    B, c = 3, heads * ch
    g = torch.Generator().manual_seed(T + ch)
    qkv = (torch.randn(B, T, 3 * c, generator=g) * 1.5).half()
    scale = 1.0 / math.sqrt(ch)
    out = U.flash_attn(qkv.to(cuda), heads, scale).float().cpu()
    x = qkv.float().view(B, T, heads, 3, ch)
    q, k, v = x[..., 0, :], x[..., 1, :], x[..., 2, :]                       # [B,T,heads,ch]
    w = torch.softmax(torch.einsum('bthc,bshc->bhts', q, k) * scale, dim=-1)
    ref = torch.einsum('bhts,bshc->bthc', w, v).reshape(B, T, c)
    assert (out - ref).abs().max().item() < 2e-3 * ref.abs().max().item() + 1e-3
    # and the unfused composition of this library agrees
    S = U.attn_scores(qkv.to(cuda), heads, scale)
    P = torch.empty(B, heads, T, T, dtype=torch.float16, device=cuda)
    N.check(N.lib().ssdnerf_softmax_rows(N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(P), N.stream_ptr()))
    vt = torch.empty(B, heads, ch, T, dtype=torch.float16, device=cuda)
    N.check(N.lib().ssdnerf_transpose_v(N.ptr(qkv.to(cuda)), N.c_u32(B), N.c_u32(T), N.c_u32(heads), N.c_u32(ch), N.ptr(vt), N.stream_ptr()))
    o2 = U.attn_pv(P, vt).float().cpu()
    assert (out - o2).abs().max().item() < 4e-3 * ref.abs().max().item() + 1e-3
