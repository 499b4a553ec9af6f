"""The tiled-triplane denoiser (configs/new_cfgs/ssdnerf_cars_recons1v_tiled.py) on the GPU: 80 / 160 / 320-channel UNet with
GroupNorm(16), attention heads of width 40 and 80, latents of 6 x 128 x 384.

Every GEMM of this model runs on the narrow-channel family of csrc/gemm_tc.cu (`algo` 3: K extents multiples of 8 with short last
K-slabs, N tiles of 16 / 40 / 48 / 80 / 160 / 256 columns).  The ops are checked against torch fp32 on the same fp16 operands, the
whole UNet, its DDIM chain and its input gradient against the fp32 GroupNorm(16) oracle of tests/unet_tiled_oracle.py (pinned to
the reference's own DenoisingUnetMod by tests/test_reference_pin_tiled_cpu.py; the engine is also checked against that fixture
directly).  The bars are those of tests/test_unet_gpu.py and tests/test_unet_bwd_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import unet_port as up
from tests import unet_tiled_oracle as uto

pytestmark = pytest.mark.gpu

TILED = dict(image_size=128, in_channels=6, base_channels=80, channels_cfg=[1, 1, 2, 2, 4, 4], resblocks_per_downsample=2,
             num_heads=4, attention_res=[16, 8, 4], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True)
HW = (128, 384)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _spec():
    return up.unet_spec(image_size=128, in_channels=6, base_channels=80, channels_cfg=(1, 1, 2, 2, 4, 4), resblocks_per_downsample=2,
                        attention_res=(16, 8, 4), num_heads=4)


def _build(sd, cuda):
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(**TILED)
    m.load_state_dict(sd, strict=True)
    return m.to(cuda).eval()


def _tc(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).half()


# ----------------------------------------------------------------------------------------------------------------------- ops
@pytest.mark.parametrize('B,H,W,C1,C2,Cout', [
    (2, 128, 384, 80, 0, 80),        # top level: K = N = 80 per tap
    (1, 64, 192, 80, 0, 160),        # 80 -> 160
    (2, 32, 96, 160, 0, 160),
    (3, 16, 48, 160, 160, 320),      # skip concat 160 + 160
    (4, 8, 24, 320, 320, 320),       # skip concat 320 + 320, two images per box
    (8, 4, 12, 320, 160, 320),       # 320 + 160, padded 16 x 4 boxes
    (2, 128, 384, 80, 80, 80),       # 80 + 80
    (2, 64, 192, 160, 80, 160),      # 160 + 80
    (2, 128, 384, 16, 0, 80),        # input convolution (6 channels padded to 16)
    (2, 128, 384, 80, 0, 6),         # output convolution, N = 6 -> 16-column tile
    (2, 8, 24, 320, 0, 320),
])
def test_narrow_conv3x3(cuda, B, H, W, C1, C2, Cout):
    """3x3 convolution (incl. the two-source skip concat) with fused quad statistics; the big shapes run several tiles per CTA"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(B * H + C1 + C2 + Cout)
    x1 = _tc(B, H, W, C1, g=g).to(cuda)
    x2 = _tc(B, H, W, C2, g=g).to(cuda) if C2 else None
    w = torch.randn(Cout, C1 + C2, 3, 3, generator=g) * 0.05
    b = torch.randn(Cout, generator=g).to(cuda)
    res = _tc(B, H, W, Cout, g=g).to(cuda)
    q = torch.zeros(B, (Cout + 3) // 4, 2, device=cuda) if Cout % 4 == 0 else None
    out = U.conv3x3_f16(x1, U.pack_conv_weight(w, narrow=True).to(cuda), Cout, bias=b, x2=x2, residual=res, qstats=q, narrow=True)
    xin = torch.cat([x1, x2], -1) if C2 else x1
    ref = F.conv2d(xin.float().permute(0, 3, 1, 2), w.half().float().to(cuda), b, padding=1).permute(0, 2, 3, 1) + res.float()
    assert _rel_l2(out.float(), ref) < 2e-3
    if q is not None:
        rq = ref.reshape(B, -1, Cout // 4, 4)
        torch.testing.assert_close(q, torch.stack([rq.sum(dim=(1, 3)), (rq * rq).sum(dim=(1, 3))], dim=-1), rtol=3e-3, atol=5e-2)


@pytest.mark.parametrize('B,H,W,C', [(2, 128, 384, 80), (2, 64, 192, 80), (2, 32, 96, 160), (3, 16, 48, 160), (4, 8, 24, 320)])
def test_narrow_stride2_and_upconv(cuda, B, H, W, C):
    """stride-2 convolution (DenoisingDownsample) and the four 2x2-tap phases of nearest-x2 + conv3x3 (DenoisingUpsample)"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(H + C)
    x = _tc(B, H, W, C, g=g).to(cuda)
    w = torch.randn(C, C, 3, 3, generator=g) * 0.05
    b = torch.randn(C, generator=g).to(cuda)
    q = torch.zeros(B, C // 4, 2, device=cuda)
    y = U.conv3x3_s2_f16(x, U.pack_conv_weight(w, narrow=True).to(cuda), C, bias=b, qstats=q, narrow=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.half().float().to(cuda), b, stride=2, padding=1).permute(0, 2, 3, 1)
    assert _rel_l2(y.float(), ref) < 2e-3
    rq = ref.reshape(B, -1, C // 4, 4)
    torch.testing.assert_close(q, torch.stack([rq.sum(dim=(1, 3)), (rq * rq).sum(dim=(1, 3))], dim=-1), rtol=3e-3, atol=5e-2)
    xs = x[:, :H // 2, :W // 2].contiguous()
    u = U.upconv3x3_f16(xs, U.pack_upconv_weight(w, narrow=True).to(cuda), C, bias=b, narrow=True)
    ref = F.conv2d(F.interpolate(xs.float().permute(0, 3, 1, 2), scale_factor=2, mode='nearest'), w.half().float().to(cuda), b,
                   padding=1).permute(0, 2, 3, 1)
    assert _rel_l2(u.float(), ref) < 3e-3


@pytest.mark.parametrize('M,K,N', [(8 * 768, 160, 480), (8 * 192, 320, 960), (8 * 48, 320, 320), (8 * 768, 160, 160),
                                   (8 * 4608, 80, 720), (8 * 1152, 160, 1440), (8 * 768, 480, 160), (4096, 240, 80), (4096, 640, 320)])
def test_narrow_linear(cuda, M, K, N):
    """1x1 GEMMs: qkv / proj projections, the stride-2 convolution's input-gradient GEMM (N = 9 c) and transposed weights (K = 3 c)"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(M + K + N)
    a = _tc(M, K, g=g, scale=0.5).to(cuda)
    w = torch.randn(N, K, generator=g) * 0.1
    bias = torch.randn(N, generator=g).to(cuda)
    res = _tc(M, N, g=g).to(cuda)
    out = U.linear_f16(a, U.pack_linear_weight(w, narrow=True).to(cuda), bias=bias, residual=res, n=N, narrow=True)
    ref = a.float() @ w.half().float().t().to(cuda) + bias + res.float()
    assert _rel_l2(out.float(), ref) < 2e-3


@pytest.mark.parametrize('B,H,W,Cin,Cout', [(2, 128, 384, 80, 80), (2, 64, 192, 80, 160), (3, 16, 48, 320, 160), (2, 128, 384, 80, 16)])
def test_narrow_input_gradient_conv(cuda, B, H, W, Cin, Cout):
    """dX = conv3x3(dY, W^T tap-flipped): K = Cout (80 / 160 / 16), N = Cin"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(Cin * Cout + H)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
    dy = _tc(B, H, W, Cout, g=g).to(cuda)
    dx = U.conv3x3_f16(dy, U.pack_conv_weight_dgrad(w, narrow=True).to(cuda), Cin, narrow=True)
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w.half().float().to(cuda), dy.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    assert _rel_l2(dx.float(), ref) < 2e-3


def test_narrow_family_is_opt_in(cuda):
    """the default family keeps its 64-multiple K contract; the narrow one accepts K = 80"""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    a = torch.randn(128, 80, device=cuda).half()
    w = torch.randn(64, 80, device=cuda).half()
    with pytest.raises(N.SSDNeRFNativeError):
        U.linear_f16(a, w)
    torch.testing.assert_close(U.linear_f16(a, w, narrow=True).float(), a.float() @ w.float().t(), rtol=2e-3, atol=2e-2)


# ----------------------------------------------------------------------------------------------------------------------- GroupNorm(16)
@pytest.mark.parametrize('C1,C2', [(80, 0), (160, 0), (320, 0), (80, 80), (160, 80), (320, 160), (320, 320)])
def test_groupnorm16_forward_backward(cuda, C1, C2):
    """GroupNorm(16) (+scale/shift, SiLU) over a channel concat: separate statistics pass (5 / 10 / 15 / 30 channels per group), backward
    split back into the two sources, against torch autograd in fp32"""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(C1 + C2)
    B, H, W, G = 2, 16, 48, 16
    C = C1 + C2
    x1 = _tc(B, H, W, C1, g=g).to(cuda)
    x2 = (torch.randn(B, H, W, C2, generator=g) * 2 + 0.5).half().to(cuda) if C2 else None
    gamma, beta = (1 + 0.1 * torch.randn(C, generator=g)).to(cuda), (0.1 * torch.randn(C, generator=g)).to(cuda)
    ss = (torch.randn(B, 2 * C, generator=g) * 0.3).to(cuda)
    st = torch.zeros(B, G, 2, device=cuda)
    out = torch.empty(B, H, W, C, dtype=torch.float16, device=cuda)
    L, s = N.lib(), N.stream_ptr()
    N.check(L.ssdnerf_gn_stats(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(st), s))
    N.check(L.ssdnerf_gn_apply(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(st),
                               N.ptr(gamma), N.ptr(beta), N.ptr(ss), N.c_longlong(2 * C), N.c_f32(1e-5), N.c_int(1), N.ptr(out), s))
    xc = (torch.cat([x1, x2], -1) if C2 else x1).float().permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.silu(F.group_norm(xc, G, gamma, beta, 1e-5) * (1 + ss[:, :C, None, None]) + ss[:, C:, None, None])
    assert _rel_l2(out.float().permute(0, 3, 1, 2), ref.detach()) < 2e-3
    dy = _tc(B, H, W, C, g=g).to(cuda)
    dx1 = torch.empty_like(x1)
    dx2 = torch.empty_like(x2) if C2 else None
    U.gn_bwd(x1, x2, (False, st, None), gamma, beta, dy, dx1, dx2, scale_shift_ptr=N.c_void_p(ss.data_ptr()), ss_batch_stride=2 * C,
             silu=True, groups=G)
    gref = torch.autograd.grad(ref, xc, dy.float().permute(0, 3, 1, 2))[0].permute(0, 2, 3, 1)
    got = torch.cat([dx1, dx2], -1) if C2 else dx1
    assert _rel_l2(got.float(), gref) < 3e-3


# ----------------------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize('ch,T', [(40, 768), (80, 192), (80, 48)])
def test_narrow_attention_forward_backward(cuda, ch, T):
    """the unfused composition (scores -> softmax -> P V) and its recomputing backward at the tiled config's head widths and lengths,
    legacy head layout, against fp32 autograd on the same fp16 qkv"""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    B, heads = 8, 4
    c = heads * ch
    g = torch.Generator().manual_seed(ch * T)
    qkv = _tc(B, T, 3 * c, g=g, scale=1.5).to(cuda)
    scale = 1.0 / math.sqrt(ch)
    S = U.attn_scores(qkv, heads, scale, narrow=True)
    P = torch.empty(B, heads, T, T, dtype=torch.float16, device=cuda)
    N.check(N.lib().ssdnerf_softmax_rows(N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(P), N.stream_ptr()))
    vt = torch.empty(B, heads, ch, T, dtype=torch.float16, device=cuda)
    N.check(N.lib().ssdnerf_transpose_v(N.ptr(qkv), N.c_u32(B), N.c_u32(T), N.c_u32(heads), N.c_u32(ch), N.ptr(vt), N.stream_ptr()))
    out = U.attn_pv(P, vt, narrow=True)
    x = qkv.float().view(B, T, heads, 3, ch).requires_grad_(True)
    q, k, v = x[..., 0, :], x[..., 1, :], x[..., 2, :]
    w = torch.softmax(torch.einsum('bthc,bshc->bhts', q, k) * scale, dim=-1)
    ref = torch.einsum('bhts,bshc->bthc', w, v).reshape(B, T, c)
    assert _rel_l2(out.float(), ref.detach()) < 3e-3
    d_o = _tc(B, T, c, g=g).to(cuda)
    ws = {}
    dqkv = U.attn_backward(qkv, d_o, heads, scale, lambda name, shape, dtype: ws.setdefault(name, torch.empty(shape, dtype=dtype, device=cuda)),
                           narrow=True)
    gref = torch.autograd.grad(ref, x, d_o.float())[0].reshape(B, T, 3 * c)
    assert _rel_l2(dqkv.float(), gref) < 5e-3


# ----------------------------------------------------------------------------------------------------------------------- whole model
def test_full_tiled_unet_one_step_vs_oracle(cuda):
    """the tiled config's UNet, one evaluation at B = 1 on a 6 x 128 x 384 latent against the fp32 oracle (on the GPU, TF32 off)"""
    spec = _spec()
    sd = up.random_state_dict(spec, seed=7, std=0.02)
    m = _build(sd, cuda)
    eng = m.engine(1, cuda, HW)
    assert eng.narrow and eng.groups == 16 and (eng.H, eng.W) == HW and eng.CPAD_IN == 16
    g = torch.Generator().manual_seed(8)
    x = torch.randn(1, 6, *HW, generator=g)
    t = torch.tensor([659])
    with torch.no_grad():
        out = m(x.to(cuda), t.to(cuda)).cpu()
    up.fp32_reference_mode()
    with torch.no_grad():
        ref = uto.unet_forward(up.state_dict_to(sd, cuda), spec, x.to(cuda), t.to(cuda)).cpu()
    err = _rel_l2(out, ref)
    print('tiled unet rel l2', err)
    assert out.shape == (1, 6, *HW) and err < 2e-3


def test_tiled_75_step_ddim_vs_fp32_oracle(cuda):
    """the whole DDIM chain at the config's num_timesteps = 75 through the captured graph, against the fp32 oracle chain"""
    from ssdnerf_b200.diffusion import GaussianDiffusion
    spec = _spec()
    sd = up.random_state_dict(spec, seed=7, std=0.02)
    m = _build(sd, cuda)
    diff = GaussianDiffusion(m, betas_cfg=dict(type='linear'), num_timesteps=1000, test_cfg=dict(num_timesteps=75, clip_range=[-2, 2])).to(cuda)
    g = torch.Generator().manual_seed(9)
    noise = torch.randn(1, 6, *HW, generator=g)
    out = diff(noise.to(cuda), return_loss=False).cpu()
    up.fp32_reference_mode()
    sdg = up.state_dict_to(sd, cuda)
    dv = up.diffusion_vars(up.linear_betas())
    with torch.no_grad():
        ref = up.ddim_sample(lambda x, t: uto.unet_forward(sdg, spec, x, t.to(x.device)), noise.to(cuda), dv, num_timesteps=75,
                             clip_range=(-2, 2)).cpu()
    err = _rel_l2(out, ref)
    print('tiled 75-step DDIM rel l2', err)
    assert err < 1e-3


def test_tiled_input_gradient_vs_oracle_autograd(cuda):
    """d (v . r) / d x_t through the native input-gradient pass against autograd through the fp32 oracle"""
    spec = _spec()
    sd = up.random_state_dict(spec, seed=11, std=0.02)
    m = _build(sd, cuda)
    for p in m.parameters():
        p.requires_grad_(False)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(1, 6, *HW, generator=g)
    r = torch.randn(1, 6, *HW, generator=g)
    t = torch.tensor([420])
    xg = x.to(cuda).requires_grad_(True)
    v = m(xg, t.to(cuda))
    (dx,) = torch.autograd.grad((v * r.to(cuda)).sum(), xg)
    up.fp32_reference_mode()
    xo = x.to(cuda).requires_grad_(True)
    vo = uto.unet_forward(up.state_dict_to(sd, cuda), spec, xo, t.to(cuda))
    (dxo,) = torch.autograd.grad((vo * r.to(cuda)).sum(), xo)
    err = _rel_l2(dx.cpu(), dxo.cpu())
    print('tiled input gradient rel l2', err)
    assert err < 4e-3


def test_tiled_training_is_refused(cuda):
    """the weight-gradient pass is not built for these widths: a training forward raises before it runs"""
    from ssdnerf_b200.unet import UNetEngine
    from ssdnerf_b200.unet_train import WeightGradPass
    spec = _spec()
    m = _build(up.random_state_dict(spec, seed=1), cuda).train()
    x = torch.randn(1, 6, *HW, device=cuda)
    with pytest.raises(NotImplementedError, match='80 / 160 / 320'):
        m(x, torch.tensor([10], device=cuda))
    with pytest.raises(NotImplementedError, match='80 / 160 / 320'):
        WeightGradPass(UNetEngine(m, 1, cuda, HW))


def test_engine_matches_reference_fixture(cuda):
    """the engine against the reference's own DenoisingUnetMod (tests/golden/reference_tiled_v1.npz): widths 80 / 160, GroupNorm(16),
    a 16 x 48 input, heads of width 40 (T = 768) and 80 (T = 192); forward and d (v . r) / d x"""
    import numpy as np
    from ssdnerf_b200.unet import DenoisingUnetMod
    from tests.common import GOLDEN, parse_shapes, seeded_weights
    z = np.load(f'{GOLDEN}/reference_tiled_v1.npz')
    sd = seeded_weights(list(z['keys']), parse_shapes(z['shapes']), int(z['weight_seed']))
    m = DenoisingUnetMod(image_size=[16, 48], in_channels=6, base_channels=80, channels_cfg=[1, 2], resblocks_per_downsample=1, num_heads=2,
                         attention_res=[16, 8], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True)
    m.load_state_dict(sd, strict=True)
    m = m.to(cuda).eval()
    for p in m.parameters():
        p.requires_grad_(False)
    x, t = torch.from_numpy(z['x']).to(cuda), torch.from_numpy(z['t']).to(cuda)
    with torch.no_grad():
        y = m(x, t).cpu()
    assert m.engine(2, cuda, (16, 48)).narrow
    err = _rel_l2(y, torch.from_numpy(z['y']))
    xg = x.clone().requires_grad_(True)
    (dx,) = torch.autograd.grad((m(xg, t) * torch.from_numpy(z['r']).to(cuda)).sum(), xg)
    gerr = _rel_l2(dx.cpu(), torch.from_numpy(z['dx']))
    print('reference fixture: forward rel l2', err, 'input gradient rel l2', gerr)
    assert err < 2e-3 and gerr < 4e-3


def test_training_refuses_groupnorm_other_than_32(cuda):
    """64-multiple widths with GroupNorm(16) run inference but the weight-gradient pass (built for GroupNorm(32)) refuses them"""
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(image_size=16, in_channels=18, base_channels=64, channels_cfg=[1, 2], resblocks_per_downsample=1, num_heads=2,
                         attention_res=[8], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True).to(cuda).train()
    x = torch.randn(1, 18, 16, 16, device=cuda)
    with pytest.raises(NotImplementedError, match='GroupNorm\\(16\\)'):
        m(x, torch.tensor([10], device=cuda))
    with torch.no_grad():
        assert torch.isfinite(m(x, torch.tensor([10], device=cuda))).all()


def test_engine_refuses_head_widths_off_the_8_grid(cuda):
    from ssdnerf_b200.unet import DenoisingUnetMod, UNetEngine
    m = DenoisingUnetMod(image_size=16, in_channels=6, base_channels=48, channels_cfg=[1, 2], resblocks_per_downsample=1, num_heads=4,
                         attention_res=[16], norm_cfg=dict(type='GN', num_groups=16), use_scale_shift_norm=True).to(cuda)
    with pytest.raises(NotImplementedError, match='head widths'):
        UNetEngine(m, 1, cuda, (16, 16))
