"""wgmma GEMM / implicit-GEMM conv (C-ABI ssdnerf_gemm_f16) vs PyTorch fp32 on the same fp16-rounded operands.

Some shapes have more than twice as many output tiles as an H100 has SMs, so the persistent kernels carry their pipelines
(stage phases, staged rows, weight tiles, statistics flushes) across several tiles per CTA."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _check(out, ref, tol=2e-3):
    err = (out.float() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
    assert err < tol, f'rel err {err}'


@pytest.mark.parametrize('M,N,K,bn', [(256, 128, 64, 128), (1000, 320, 192, 0), (128, 64, 128, 64), (4096, 512, 1024, 256), (8960, 512, 256, 128)])
def test_plain_gemm(cuda, M, N, K, bn):
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(M + N + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda)
    w = (torch.randn(N, K, generator=g) * 0.1).half().to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    res = torch.randn(M, N, generator=g).half().to(cuda)
    out = U.linear_f16(a, w, bias=bias, residual=res, bn=bn)
    ref = a.float() @ w.float().t() + bias + res.float()
    _check(out, ref)
    out32 = U.linear_f16(a, w, out_f32=True, alpha=0.25, bn=bn)
    _check(out32, 0.25 * (a.float() @ w.float().t()), 1e-3)


@pytest.mark.parametrize('B,H,W,Cin,Cout', [(2, 128, 128, 64, 128), (3, 64, 64, 128, 256), (2, 32, 32, 256, 256),
                                            (3, 16, 16, 512, 512), (5, 8, 8, 512, 512)])
def test_conv3x3(cuda, B, H, W, Cin, Cout):
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(B * H + Cin)
    x = (torch.randn(B, H, W, Cin, generator=g)).half().to(cuda)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05)
    b = torch.randn(Cout, generator=g).to(cuda)
    wp = U.pack_conv_weight(w).to(cuda)
    out = U.conv3x3_f16(x, wp, Cout, bias=b)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.half().float().to(cuda), b, padding=1).permute(0, 2, 3, 1)
    _check(out, ref)


def test_conv3x3_concat_and_residual(cuda):
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(11)
    B, H, W = 2, 32, 32
    x1 = torch.randn(B, H, W, 256, generator=g).half().to(cuda)
    x2 = torch.randn(B, H, W, 128, generator=g).half().to(cuda)
    w = torch.randn(256, 384, 3, 3, generator=g) * 0.03
    res = torch.randn(B, H, W, 256, generator=g).half().to(cuda)
    out = U.conv3x3_f16(x1, U.pack_conv_weight(w).to(cuda), 256, x2=x2, residual=res)
    xin = torch.cat([x1, x2], -1).float().permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xin, w.half().float().to(cuda), None, padding=1).permute(0, 2, 3, 1) + res.float()
    _check(out, ref)


def test_batched_attention_gemms(cuda):
    """S = q k^T over (batch, head) with strided q/k slices of a [B,T,3c] qkv tensor (legacy head layout)."""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(13)
    B, T, c, heads = 2, 256, 256, 4
    ch = c // heads
    qkv = torch.randn(B, T, 3 * c, generator=g).half().to(cuda)
    S = U.attn_scores(qkv, heads, scale=ch ** -0.5)
    q = qkv.float().view(B, T, heads, 3, ch)[:, :, :, 0]
    k = qkv.float().view(B, T, heads, 3, ch)[:, :, :, 1]
    ref = torch.einsum('bthc,bshc->bhts', q, k) * ch ** -0.5
    _check(S, ref, 1e-3)


@pytest.mark.parametrize('B,H,W,Cin,Cout,bn', [(3, 64, 64, 128, 256, 256), (2, 128, 128, 64, 128, 128), (5, 8, 8, 512, 512, 256), (1, 32, 32, 256, 256, 128),
                                              (5, 64, 64, 128, 256, 128)])
def test_conv3x3_forced_tile_width_and_quad_stats(cuda, B, H, W, Cin, Cout, bn):
    """a forced N tile with bias, residual and the fused quad statistics; odd tile counts and several tiles per CTA"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(B * H + Cin + 1)
    x = torch.randn(B, H, W, Cin, generator=g).half().to(cuda)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
    b = torch.randn(Cout, generator=g).to(cuda)
    res = torch.randn(B, H, W, Cout, generator=g).half().to(cuda)
    q = torch.zeros(B, Cout // 4, 2, device=cuda)
    out = U.conv3x3_f16(x, U.pack_conv_weight(w).to(cuda), Cout, bias=b, residual=res, bn=bn, qstats=q)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.half().float().to(cuda), b, padding=1).permute(0, 2, 3, 1) + res.float()
    _check(out, ref)
    rq = ref.reshape(B, -1, Cout // 4, 4)
    torch.testing.assert_close(q, torch.stack([rq.sum(dim=(1, 3)), (rq * rq).sum(dim=(1, 3))], dim=-1), rtol=2e-3, atol=2e-2)


def test_plain_gemm_nine_k_chunks_forced_wide_tile(cuda):
    """K = 576 = 9 x 64 (more k-blocks than pipeline stages at bn = 256) over seven row tiles, without bias or residual"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(77)
    M, N, K = 128 * 7, 512, 576
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda)
    w = (torch.randn(N, K, generator=g) * 0.1).half().to(cuda)
    out = U.linear_f16(a, w, bn=256)
    _check(out, a.float() @ w.float().t())


@pytest.mark.parametrize('B,H,C1,C2', [(2, 8, 128, 0), (1, 128, 64, 0), (3, 6, 128, 128), (2, 4, 256, 128), (5, 128, 64, 64)])
def test_conv3x3_row_pair_kernel(cuda, B, H, C1, C2):
    """128-pixel-wide rows, 128 output channels: row-pair kernel with halo reuse (algo 2) == generic tile kernel (algo 1) == fp32 conv,
    including image borders, the skip-concat second input, bias, residual and the fused quad statistics"""
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(B * 100 + H + C1 + C2)
    W, Cout = 128, 128
    x = torch.randn(B, H, W, C1, generator=g).half().to(cuda)
    x2 = torch.randn(B, H, W, C2, generator=g).half().to(cuda) if C2 else None
    w = torch.randn(Cout, C1 + C2, 3, 3, generator=g) * 0.05
    bias = torch.randn(Cout, generator=g).to(cuda)
    res = torch.randn(B, H, W, Cout, generator=g).half().to(cuda)
    wp = U.pack_conv_weight(w).to(cuda)
    outs, stats = {}, {}
    for algo in (1, 2):
        q = torch.zeros(B, Cout // 4, 2, device=cuda)
        outs[algo] = U.conv3x3_f16(x, wp, Cout, bias=bias, x2=x2, residual=res, qstats=q, algo=algo)
        stats[algo] = q
    xin = torch.cat([x, x2], dim=-1) if C2 else x
    ref = torch.nn.functional.conv2d(xin.float().permute(0, 3, 1, 2), w.half().float().to(cuda), bias, padding=1).permute(0, 2, 3, 1) + res.float()
    _check(outs[2], ref)
    _check(outs[1], ref)
    torch.testing.assert_close(outs[2].float(), outs[1].float(), rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(stats[2], stats[1], rtol=1e-3, atol=5e-2)


@pytest.mark.parametrize('B,H,C1,C2,use_ss', [(2, 8, 128, 0, False), (1, 128, 128, 0, True), (3, 6, 128, 128, False), (2, 4, 256, 128, True),
                                              (5, 128, 128, 128, True)])
def test_groupnorm_silu_from_quad_stats_then_conv3x3(cuda, B, H, C1, C2, use_ss):
    """GroupNorm(32) (+ scale/shift) + SiLU from the producers' quad statistics (gn_apply_q: channel concat of two sources, scale/shift rows at
    an offset with a batch stride) followed by the row-pair convolution vs fp32 PyTorch GroupNorm -> SiLU -> conv2d."""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + C1 + C2 + int(use_ss))
    W, Cout, C = 128, 128, C1 + C2
    x1 = (torch.randn(B, H, W, C1, generator=g) * 1.5 + 0.3).half().to(cuda)
    x2 = (torch.randn(B, H, W, C2, generator=g) * 0.7 - 0.2).half().to(cuda) if C2 else None

    def quads(x):
        xf = x.float().reshape(x.shape[0], -1, x.shape[-1] // 4, 4)
        return torch.stack([xf.sum(dim=(1, 3)), (xf * xf).sum(dim=(1, 3))], dim=-1).contiguous()
    q1, q2 = quads(x1), (quads(x2) if C2 else None)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(cuda)
    beta = (0.2 * torch.randn(C, generator=g)).to(cuda)
    ss = (0.3 * torch.randn(B, 2 * C + 64, generator=g)).to(cuda) if use_ss else None      # row b: [pad 64][scale C][shift C]
    ss_ptr = N.c_void_p(ss.data_ptr() + 4 * 64) if use_ss else None
    w = torch.randn(Cout, C, 3, 3, generator=g) * 0.05
    wp = U.pack_conv_weight(w).to(cuda)
    bias = torch.randn(Cout, generator=g).to(cuda)
    res = torch.randn(B, H, W, Cout, generator=g).half().to(cuda)
    y = torch.empty(B, H, W, C, dtype=torch.float16, device=cuda)
    N.check(N.lib().ssdnerf_gn_apply_q(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(32), N.ptr(q1), N.ptr(q2),
                                       N.ptr(gamma), N.ptr(beta), ss_ptr, N.c_longlong(ss.shape[1] if use_ss else 0), N.c_f32(1e-5), N.c_int(1),
                                       N.ptr(y), N.stream_ptr()))
    qo = torch.zeros(B, Cout // 4, 2, device=cuda)
    out = U.conv3x3_f16(y, wp, Cout, bias=bias, residual=res, qstats=qo)
    # fp32 reference
    xin = torch.cat([x1, x2], dim=-1) if C2 else x1
    xn = torch.nn.functional.group_norm(xin.float().permute(0, 3, 1, 2), 32, gamma, beta, eps=1e-5)
    if use_ss:
        xn = xn * (1 + ss[:, 64:64 + C, None, None]) + ss[:, 64 + C:64 + 2 * C, None, None]
    wr = w.half().float().to(cuda)
    ref = torch.nn.functional.conv2d(torch.nn.functional.silu(xn), wr, bias, padding=1).permute(0, 2, 3, 1) + res.float()
    _check(out, ref, tol=5e-3)
    # emitted statistics: those of the fp32 convolution of the fp16 activation the kernel read, and, to the fp16 rounding of that
    # activation, those of the all-fp32 chain
    ref_y = torch.nn.functional.conv2d(y.float().permute(0, 3, 1, 2), wr, bias, padding=1).permute(0, 2, 3, 1) + res.float()
    torch.testing.assert_close(qo, quads(ref_y), rtol=2e-3, atol=2e-2)
    qr = quads(ref)
    assert ((qo - qr).abs() / (qr.abs() + 0.05 * qr.abs().max())).max().item() < 2e-3


@pytest.mark.parametrize('B,H,C,Cout', [(2, 16, 128, 128), (3, 16, 512, 512), (1, 128, 128, 128), (2, 64, 256, 256), (5, 32, 256, 256)])
def test_stride2_conv_and_upsample_conv_without_intermediate_buffers(cuda, B, H, C, Cout):
    """DenoisingDownsample (conv3x3 stride 2) straight from the input through stride-2 TMA boxes, and DenoisingUpsample (nearest x2 + conv3x3)
    as four 2x2-tap phase convolutions of the low-resolution tensor, vs F.conv2d on the same fp16 operands; fused quad statistics too."""
    import torch.nn.functional as F
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(H + C)
    x = torch.randn(B, H, H, C, generator=g).half().to(cuda)
    w = torch.randn(Cout, C, 3, 3, generator=g) * 0.05
    bias = torch.randn(Cout, generator=g).to(cuda)
    xr = x.float().permute(0, 3, 1, 2)
    wr = w.half().float().to(cuda)
    # stride 2
    q = torch.zeros(B, Cout // 4, 2, device=cuda)
    y = U.conv3x3_s2_f16(x, U.pack_conv_weight(w).to(cuda), Cout, bias=bias, qstats=q)
    ref = F.conv2d(xr, wr, bias, stride=2, padding=1).permute(0, 2, 3, 1)
    assert y.shape == ref.shape
    assert (y.float() - ref).abs().max().item() < 2e-3 * ref.abs().max().item() + 2e-3
    rq = ref.reshape(B, -1, Cout // 4, 4)
    torch.testing.assert_close(q, torch.stack([rq.sum(dim=(1, 3)), (rq * rq).sum(dim=(1, 3))], dim=-1), rtol=2e-3, atol=2e-2)
    # nearest x2 + conv: the merged-tap weights are rounded to fp16 once (w1 + w2 -> fp16), so compare against the fp32-weight reference
    q2 = torch.zeros(B, Cout // 4, 2, device=cuda)
    y2 = U.upconv3x3_f16(x, U.pack_upconv_weight(w).to(cuda), Cout, bias=bias, qstats=q2)
    ref2 = F.conv2d(F.interpolate(xr, scale_factor=2, mode='nearest'), w.to(cuda), bias, padding=1).permute(0, 2, 3, 1)
    assert y2.shape == ref2.shape
    assert (y2.float() - ref2).abs().max().item() < 3e-3 * ref2.abs().max().item() + 3e-3
    assert float((y2.float() - ref2).norm() / ref2.norm()) < 1e-3
    # the fused statistics are those of the kernel's own fp32 accumulators (merged fp16 weights), summed over the four phase launches
    o2 = U.upconv3x3_f16(x, U.pack_upconv_weight(w).to(cuda), Cout, bias=bias, out=torch.empty(B, 2 * H, 2 * H, Cout, dtype=torch.float32, device=cuda))
    assert torch.equal(y2, o2.half())
    rq2 = o2.reshape(B, -1, Cout // 4, 4)
    torch.testing.assert_close(q2, torch.stack([rq2.sum(dim=(1, 3)), (rq2 * rq2).sum(dim=(1, 3))], dim=-1), rtol=1e-3, atol=2e-2)
