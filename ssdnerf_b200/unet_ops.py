"""Thin Python wrappers over the UNet building-block kernels (C ABI section 4, include/ssdnerf_b200.h).

Activations are NHWC fp16 tensors; weights are packed once (`pack_conv_weight`, `pack_linear_weight`).

`narrow=True` selects the narrow-channel GEMM family (`ssdnerf_gemm_args.algo = 3`, csrc/gemm_tc.cu): K extents per source that are
multiples of 8 rather than 64 (a source's last K chunk is a short slab, only its k-steps that hold data are issued) and N tiles of
16 / 40 / 48 / 80 / 160 / 256 columns fitted to N.  The tiled-triplane UNet (80 / 160 / 320 channels, 40 / 80-wide heads) runs on it;
every other caller keeps the default family and its 64-multiple K contract.
"""
import ctypes

import torch

from . import _lib as N

c_u64 = ctypes.c_uint64
c_ll = ctypes.c_longlong


class GemmArgs(ctypes.Structure):
    """mirror of `ssdnerf_gemm_args`"""
    _fields_ = [
        ('a1', N.c_void_p), ('a1_strides', c_u64 * 3), ('k1', N.c_u32),
        ('a2', N.c_void_p), ('a2_strides', c_u64 * 3), ('k2', N.c_u32),
        ('d1', N.c_u32), ('d2', N.c_u32), ('d3', N.c_u32), ('b1', N.c_u32), ('b2', N.c_u32), ('b3', N.c_u32),
        ('taps', N.c_u32),
        ('b', N.c_void_p), ('b_strides', c_u64 * 3), ('n', N.c_u32), ('n_rows_b', N.c_u32), ('bx2', N.c_u32), ('bx3', N.c_u32),
        ('b_batched', N.c_u32),
        ('bn', N.c_u32), ('alpha', N.c_f32), ('bias_n', N.c_void_p), ('residual', N.c_void_p),
        ('out', N.c_void_p), ('out_f32', N.c_u32), ('so1', c_ll), ('so2', c_ll), ('so3', c_ll),
        ('qstats', N.c_void_p), ('stats_hw', N.c_u32), ('algo', N.c_u32),
        ('tap_offsets', N.c_void_p), ('a_stride', N.c_u32),
    ]


ALGO_NARROW = 3     # ssdnerf_gemm_args.algo of the narrow-channel family


def _launch(a):
    N.check(N.lib().ssdnerf_gemm_f16(ctypes.byref(a), N.stream_ptr()))


def _pad_rows(w, mult=64):
    n = w.shape[-2]
    pad = (-n) % mult
    if pad:
        w = torch.cat([w, w.new_zeros(*w.shape[:-2], pad, w.shape[-1])], dim=-2)
    return w


def pack_linear_weight(w, narrow=False):
    """nn.Linear / 1x1-conv weight [N, K] -> fp16 [N_pad, K] (rows padded to a multiple of 64 so any N tile is in bounds).
    narrow: K a multiple of 8 (the narrow-channel GEMM family)."""
    w = w.detach().reshape(w.shape[0], -1).half()
    assert w.shape[1] % (8 if narrow else 64) == 0, 'K must be a multiple of 64 (narrow: of 8)'
    return _pad_rows(w).contiguous()


def pack_conv_weight(w, cin_pad=None, narrow=False):
    """Conv2d weight [Cout, Cin, 3, 3] -> fp16 [9][Cout_pad][Cin_pad] (tap = ky*3 + kx, K contiguous).
    Cin_pad defaults to the next multiple of 64 (narrow: of 8)."""
    cout, cin = w.shape[0], w.shape[1]
    m = 8 if narrow else 64
    cin_pad = cin_pad or ((cin + m - 1) // m * m)
    wp = w.detach().permute(2, 3, 0, 1).reshape(9, cout, cin).half()
    if cin_pad != cin:
        wp = torch.cat([wp, wp.new_zeros(9, cout, cin_pad - cin)], dim=-1)
    return _pad_rows(wp).contiguous()


def linear_f16(a, w, bias=None, residual=None, out=None, out_f32=False, alpha=1.0, bn=0, n=None, qstats=None, stats_hw=0, narrow=False):
    """out[M, N] = alpha * a[M, K] @ w[N, K]^T + bias + residual.  a fp16 [M, K] (row stride may exceed K)."""
    N.require_cuda(a, w)
    M, K = a.shape
    n = n if n is not None else w.shape[0]
    if out is None:
        out = torch.empty(M, n, dtype=torch.float32 if out_f32 else torch.float16, device=a.device)
    g = GemmArgs()
    g.a1, g.k1 = a.data_ptr(), K
    rs = a.stride(0) * 2
    g.a1_strides = (c_u64 * 3)(rs, rs * M, rs * M)
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = M, 1, 1, 128, 1, 1
    g.taps = 1
    g.b, g.n, g.n_rows_b, g.bx2, g.bx3 = w.data_ptr(), n, w.shape[0], 1, 1
    ws = w.stride(0) * 2
    g.b_strides = (c_u64 * 3)(ws, ws * w.shape[0], ws * w.shape[0])
    g.bn, g.alpha = bn, alpha
    g.bias_n = bias.data_ptr() if bias is not None else None
    g.residual = residual.data_ptr() if residual is not None else None
    g.out, g.out_f32 = out.data_ptr(), int(out.dtype == torch.float32)
    g.so1, g.so2, g.so3 = out.stride(0), 0, 0
    if qstats is not None:
        g.qstats, g.stats_hw = qstats.data_ptr(), stats_hw
    if narrow:
        g.algo = ALGO_NARROW
    _launch(g)
    return out


def _conv_boxes(H, W, narrow=False):
    if narrow:
        return _conv_boxes_narrow(H, W)
    bw = min(W, 128)
    bh = min(H, 128 // bw)
    nb = 128 // (bw * bh)
    return bw, bh, nb


def _pow2_floor(v):
    return 1 << (max(int(v), 1).bit_length() - 1)


def _conv_boxes_narrow(H, W):
    """128-pixel TMA boxes (bw x bh x nb images, powers of two) for any H x W: the widest power of two that divides W (no partial
    boxes along a row), rows filling the rest.  The fused quad statistics need every 64-pixel half of a box inside one image (nb <= 2);
    where that would not hold (4 x 12) the box is the next power of two above W and H, its tail zero-filled and masked."""
    bw = min(128, W & -W)
    bh = min(128 // bw, _pow2_floor(H))
    if 128 // (bw * bh) > 2:
        bw = min(128, 1 << (W - 1).bit_length())
        bh = min(128 // bw, 1 << (H - 1).bit_length())
    return bw, bh, 128 // (bw * bh)


def conv3x3_f16(x, wp, cout, bias=None, x2=None, residual=None, out=None, out_f32=False, taps=9, bn=0, qstats=None, algo=0, narrow=False):
    """3x3 (taps=9, pad 1, stride 1) or 1x1 (taps=1) convolution over NHWC fp16 x [B,H,W,C1] (+ x2 [B,H,W,C2] concatenated
    along channels).  wp: packed weight [taps][Cout_pad][C1+C2].  narrow: C1 / C2 multiples of 8 (narrow-channel family)."""
    N.require_cuda(x, wp)
    B, H, W, C1 = x.shape
    C2 = x2.shape[-1] if x2 is not None else 0
    assert x.is_contiguous() and (x2 is None or x2.is_contiguous())
    km = 8 if narrow else 64
    assert wp.shape[-1] == C1 + C2 and C1 % km == 0 and C2 % km == 0, (wp.shape, C1, C2)
    if narrow:
        algo = ALGO_NARROW
    if out is None:
        out = torch.empty(B, H, W, cout, dtype=torch.float32 if out_f32 else torch.float16, device=x.device)
    bw, bh, nb = _conv_boxes(H, W, narrow)
    g = GemmArgs()
    g.a1, g.k1 = x.data_ptr(), C1
    g.a1_strides = (c_u64 * 3)(C1 * 2, W * C1 * 2, H * W * C1 * 2)
    if x2 is not None:
        g.a2, g.k2 = x2.data_ptr(), C2
        g.a2_strides = (c_u64 * 3)(C2 * 2, W * C2 * 2, H * W * C2 * 2)
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = W, H, B, bw, bh, nb
    g.taps = taps
    ktot = C1 + C2
    rows = wp.shape[-2]
    g.b, g.n, g.n_rows_b, g.bx2, g.bx3 = wp.data_ptr(), cout, rows, taps, 1
    g.b_strides = (c_u64 * 3)(ktot * 2, rows * ktot * 2, taps * rows * ktot * 2)
    g.bn, g.alpha, g.algo = bn, 1.0, algo
    g.bias_n = bias.data_ptr() if bias is not None else None
    g.residual = residual.data_ptr() if residual is not None else None
    g.out, g.out_f32 = out.data_ptr(), int(out.dtype == torch.float32)
    co = out.shape[-1]
    g.so1, g.so2, g.so3 = co, W * co, H * W * co
    if qstats is not None:
        g.qstats, g.stats_hw = qstats.data_ptr(), 0
    _launch(g)
    return out


def conv3x3_s2_f16(x, wp, cout, bias=None, out=None, qstats=None, narrow=False):
    """3x3 stride-2 pad-1 convolution (mmgen DenoisingDownsample) over NHWC fp16 x [B,H,W,C] -> [B,H/2,W/2,cout] WITHOUT an im2col
    buffer: the same implicit GEMM as the stride-1 convolution, its TMA boxes traversing every second input pixel (a_stride = 2)."""
    N.require_cuda(x, wp)
    B, H, W, C = x.shape
    assert x.is_contiguous() and H % 2 == 0 and W % 2 == 0 and wp.shape[-1] == C and C % (8 if narrow else 64) == 0
    Ho, Wo = H // 2, W // 2
    if out is None:
        out = torch.empty(B, Ho, Wo, cout, dtype=torch.float16, device=x.device)
    bw, bh, nb = _conv_boxes(Ho, Wo, narrow)
    g = GemmArgs()
    g.a1, g.k1 = x.data_ptr(), C
    g.a1_strides = (c_u64 * 3)(C * 2, W * C * 2, H * W * C * 2)
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = Wo, Ho, B, bw, bh, nb
    g.taps, g.a_stride = 9, 2
    rows = wp.shape[-2]
    g.b, g.n, g.n_rows_b, g.bx2, g.bx3 = wp.data_ptr(), cout, rows, 9, 1
    g.b_strides = (c_u64 * 3)(C * 2, rows * C * 2, 9 * rows * C * 2)
    g.bn, g.alpha, g.algo = 0, 1.0, ALGO_NARROW if narrow else 1
    g.bias_n = bias.data_ptr() if bias is not None else None
    g.out, g.out_f32 = out.data_ptr(), int(out.dtype == torch.float32)
    g.so1, g.so2, g.so3 = cout, Wo * cout, Ho * Wo * cout
    if qstats is not None:
        g.qstats, g.stats_hw = qstats.data_ptr(), 0
    _launch(g)
    return out


_UP_ROWS = {0: ((-1, (0,)), (0, (1, 2))), 1: ((0, (0, 1)), (1, (2,)))}     # output parity -> ((source offset, merged kernel rows), ...)


def pack_upconv_weight(w, narrow=False):
    """nearest-x2 upsample followed by conv3x3 == four 2x2-tap convolutions of the LOW-resolution image, one per output parity
    (py, px): kernel rows / columns that read the same source pixel are summed.  w [Cout, Cin, 3, 3] -> fp16 [4 phases][4 taps][Cout_pad][Cin]
    (phase = py*2 + px, tap = iy*2 + ix) -- 16 tap-GEMMs at a quarter of the pixels = 4/9 of the flops, and no upsampled tensor."""
    w = w.detach().float()
    phases = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for _, kys in _UP_ROWS[py]:
                for _, kxs in _UP_ROWS[px]:
                    taps.append(sum(w[:, :, ky, kx] for ky in kys for kx in kxs))
            phases.append(torch.stack(taps))                     # [4, Cout, Cin]
    wp = torch.stack(phases).half()                              # [4, 4, Cout, Cin]
    assert wp.shape[-1] % (8 if narrow else 64) == 0
    return _pad_rows(wp).contiguous()


def upconv3x3_f16(x, wps, cout, bias=None, out=None, qstats=None, narrow=False):
    """conv3x3(nearest_x2(x)) (mmgen DenoisingUpsample) from the low-resolution x [B,H,W,C] -> [B,2H,2W,cout]; wps = pack_upconv_weight."""
    N.require_cuda(x, wps)
    B, H, W, C = x.shape
    assert x.is_contiguous() and wps.shape[-1] == C
    if out is None:
        out = torch.empty(B, 2 * H, 2 * W, cout, dtype=torch.float16, device=x.device)
    bw, bh, nb = _conv_boxes(H, W, narrow)
    rows = wps.shape[-2]
    esz = out.element_size()
    for py in (0, 1):
        for px in (0, 1):
            offs = (ctypes.c_int8 * 8)(*[v for oy, _ in _UP_ROWS[py] for ox, _ in _UP_ROWS[px] for v in (ox, oy)])
            g = GemmArgs()
            g.a1, g.k1 = x.data_ptr(), C
            g.a1_strides = (c_u64 * 3)(C * 2, W * C * 2, H * W * C * 2)
            g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = W, H, B, bw, bh, nb
            g.taps, g.a_stride = 4, 1
            g.tap_offsets = ctypes.cast(offs, ctypes.c_void_p)
            ph = py * 2 + px
            g.b = wps.data_ptr() + ph * 4 * rows * C * 2
            g.n, g.n_rows_b, g.bx2, g.bx3 = cout, rows, 4, 1
            g.b_strides = (c_u64 * 3)(C * 2, rows * C * 2, 4 * rows * C * 2)
            g.bn, g.alpha, g.algo = 0, 1.0, ALGO_NARROW if narrow else 1
            g.bias_n = bias.data_ptr() if bias is not None else None
            g.out = out.data_ptr() + (py * 2 * W + px) * cout * esz
            g.out_f32 = int(out.dtype == torch.float32)
            g.so1, g.so2, g.so3 = 2 * cout, 2 * (2 * W) * cout, 4 * H * W * cout
            if qstats is not None:
                g.qstats, g.stats_hw = qstats.data_ptr(), 0
            _launch(g)
    return out


def attn_scores(qkv, heads, scale, out=None, narrow=False):
    """S[b,h,t,s] = scale * q[b,t,h,:] . k[b,s,h,:] in fp32, q/k read in place from qkv [B,T,3c] with the reference's
    legacy head layout (head h owns channels [h*3ch, (h+1)*3ch) = q | k | v; lib/models/architecture/ddpm/modules.py:36-48).
    narrow: head widths that are multiples of 8 (40, 80), K = ch zero-filled to the next 16 by TMA."""
    B, T, c3 = qkv.shape
    c = c3 // 3
    ch = c // heads
    assert ch % (8 if narrow else 64) == 0
    if out is None:
        out = torch.empty(B, heads, T, T, dtype=torch.float32, device=qkv.device)
    g = GemmArgs()
    g.a1, g.k1 = qkv.data_ptr(), ch
    g.a1_strides = (c_u64 * 3)(c3 * 2, 3 * ch * 2, T * c3 * 2)              # t, head, batch
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = T, heads, B, 128, 1, 1
    g.taps = 1
    g.b = qkv.data_ptr() + ch * 2                                            # k slice of each head
    g.n, g.n_rows_b, g.bx2, g.bx3, g.b_batched = T, T, heads, B, 1
    g.b_strides = (c_u64 * 3)(c3 * 2, 3 * ch * 2, T * c3 * 2)
    g.bn, g.alpha = 0, scale
    g.out, g.out_f32 = out.data_ptr(), 1
    g.so1, g.so2, g.so3 = T, T * T, heads * T * T
    if narrow:
        g.algo = ALGO_NARROW
    _launch(g)
    return out


def attn_pv(P, vt, out=None, narrow=False):
    """O[b,t,h*ch + c] = sum_s P[b,h,t,s] * vt[b,h,c,s]   (P fp16 [B,heads,T,T], vt fp16 [B,heads,ch,T]) -> fp16 [B,T,heads*ch]"""
    B, heads, T, _ = P.shape
    ch = vt.shape[2]
    c = heads * ch
    assert T % (8 if narrow else 64) == 0
    if out is None:
        out = torch.empty(B, T, c, dtype=torch.float16, device=P.device)
    g = GemmArgs()
    g.a1, g.k1 = P.data_ptr(), T
    g.a1_strides = (c_u64 * 3)(T * 2, T * T * 2, heads * T * T * 2)
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = T, heads, B, 128, 1, 1
    g.taps = 1
    g.b, g.n, g.n_rows_b, g.bx2, g.bx3, g.b_batched = vt.data_ptr(), ch, ch, heads, B, 1
    g.b_strides = (c_u64 * 3)(T * 2, ch * T * 2, heads * ch * T * 2)
    g.bn, g.alpha = 0, 1.0
    g.out, g.out_f32 = out.data_ptr(), 0
    g.so1, g.so2, g.so3 = c, ch, T * c
    if narrow:
        g.algo = ALGO_NARROW
    _launch(g)
    return out


def flash_attn(qkv, heads, scale, out=None):
    """O[b,t,h*ch+d] = softmax_s(scale * q.k) v with the scores kept on chip (csrc/attention.cu). qkv fp16 [B,T,3c], legacy head layout."""
    N.require_cuda(qkv)
    B, T, c3 = qkv.shape
    c = c3 // 3
    ch = c // heads
    assert qkv.is_contiguous() and qkv.dtype == torch.float16
    if out is None:
        out = torch.empty(B, T, c, dtype=torch.float16, device=qkv.device)
    N.check(N.lib().ssdnerf_flash_attn(N.ptr(qkv), N.c_u32(B), N.c_u32(T), N.c_u32(heads), N.c_u32(ch), N.c_f32(scale), N.ptr(out),
                                       N.stream_ptr()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# input-gradient pass (C ABI section 4b): data gradients of the frozen UNet
# ---------------------------------------------------------------------------------------------------------------------
def pack_conv_weight_dgrad(w, cout_pad=None, narrow=False):
    """Conv2d weight [Cout, Cin, 3, 3] -> packed weight of the DATA-GRADIENT convolution: dX = conv3x3(dY, W^T with flipped taps),
    i.e. a 3x3 stride-1 convolution whose input channels are Cout (zero-padded to `cout_pad`) and whose outputs are Cin."""
    return pack_conv_weight(w.detach().transpose(0, 1).flip(2, 3), cin_pad=cout_pad, narrow=narrow)


def pack_linear_weight_dgrad(w, narrow=False):
    """Linear / 1x1-conv weight [N, K] -> packed [K_pad, N] so that dX[M, K] = dY[M, N] @ W."""
    w = w.detach().reshape(w.shape[0], -1)
    return pack_linear_weight(w.t(), narrow=narrow)


class GnBwdArgs(ctypes.Structure):
    """mirror of `ssdnerf_gn_bwd_args`"""
    _fields_ = [
        ('x1', N.c_void_p), ('C1', N.c_u32), ('x2', N.c_void_p), ('C2', N.c_u32), ('B', N.c_u32), ('HW', N.c_u32), ('groups', N.c_u32),
        ('stats', N.c_void_p), ('stats2', N.c_void_p), ('quad_stats', N.c_int), ('gamma', N.c_void_p), ('beta', N.c_void_p),
        ('scale_shift', N.c_void_p), ('ss_batch_stride', c_ll), ('eps', N.c_f32), ('do_silu', N.c_int),
        ('dy', N.c_void_p), ('add', N.c_void_p), ('group_sums', N.c_void_p), ('dx1', N.c_void_p), ('dx2', N.c_void_p),
        ('channel_sums', N.c_void_p),
    ]


def gn_bwd(x1, x2, stats, gamma, beta, dy, dx1, dx2=None, add=None, scale_shift_ptr=None, ss_batch_stride=0, silu=True, gsum=None, eps=1e-5,
           csum=None, groups=32):
    """GroupNorm(groups)(+scale/shift)(+SiLU) backward over the channel concat of x1 (+x2); stats = (quad_flag, s1, s2) as the forward used.
    csum (fp32 [B, C, 2], overwritten): per-(image, channel) sums the affine / scale-shift parameter gradients are built from."""
    N.require_cuda(x1, dy, dx1)
    B, H, W, C1 = x1.shape
    a = GnBwdArgs()
    a.x1, a.C1 = x1.data_ptr(), C1
    if x2 is not None:
        a.x2, a.C2 = x2.data_ptr(), x2.shape[-1]
    a.B, a.HW, a.groups = B, H * W, groups
    quad, s1, s2 = stats
    a.stats, a.quad_stats = s1.data_ptr(), int(quad)
    a.stats2 = s2.data_ptr() if s2 is not None else None
    a.gamma, a.beta = gamma.data_ptr(), beta.data_ptr()
    if scale_shift_ptr is not None:
        a.scale_shift, a.ss_batch_stride = scale_shift_ptr, ss_batch_stride
    a.eps, a.do_silu = eps, int(silu)
    a.dy = dy.data_ptr()
    a.add = add.data_ptr() if add is not None else None
    if gsum is None:
        gsum = torch.empty(B * groups * 2, dtype=torch.float32, device=x1.device)
    a.group_sums = gsum.data_ptr()
    a.dx1 = dx1.data_ptr()
    a.dx2 = dx2.data_ptr() if dx2 is not None else None
    a.channel_sums = csum.data_ptr() if csum is not None else None
    N.check(N.lib().ssdnerf_gn_bwd(ctypes.byref(a), N.stream_ptr()))
    return dx1, dx2


class WgradArgs(ctypes.Structure):
    """mirror of `ssdnerf_wgrad_args`"""
    _fields_ = [
        ('gy', N.c_void_p), ('gy_stride', N.c_u32), ('gy_c0', N.c_u32),
        ('x', N.c_void_p), ('x_stride', N.c_u32), ('x_c0', N.c_u32),
        ('dw', N.c_void_p), ('dw_stride', N.c_u32), ('dw_c0', N.c_u32),
        ('batch', N.c_u32), ('out_h', N.c_u32), ('out_w', N.c_u32), ('in_h', N.c_u32), ('in_w', N.c_u32),
        ('cout', N.c_u32), ('cin', N.c_u32), ('taps', N.c_u32), ('stride', N.c_u32), ('up', N.c_int), ('ksplit', N.c_u32),
    ]


def conv_wgrad(gy, x, dw, cout, cin, taps=1, stride=1, up=False, gy_c0=0, x_c0=0, dw_c0=0, ksplit=0):
    """dw[co, tap, dw_c0 + ci] += sum_pixels gy[..., gy_c0 + co] * x[shifted pixel, x_c0 + ci]  (header section 4c).
    gy fp16 [B,Ho,Wo,Cg]; x fp16 [B,Hi,Wi,Cx]; dw fp32 [cout, taps, K] contiguous."""
    N.require_cuda(gy, x, dw)
    assert gy.dtype == torch.float16 and x.dtype == torch.float16 and dw.dtype == torch.float32 and dw.is_contiguous()
    B, Ho, Wo, Cg = gy.shape
    _, Hi, Wi, Cx = x.shape
    a = WgradArgs()
    a.gy, a.gy_stride, a.gy_c0 = gy.data_ptr(), Cg, gy_c0
    a.x, a.x_stride, a.x_c0 = x.data_ptr(), Cx, x_c0
    a.dw, a.dw_stride, a.dw_c0 = dw.data_ptr(), dw.shape[-1], dw_c0
    a.batch, a.out_h, a.out_w, a.in_h, a.in_w = B, Ho, Wo, Hi, Wi
    a.cout, a.cin, a.taps, a.stride, a.up, a.ksplit = cout, cin, taps, stride, int(up), ksplit
    N.check(N.lib().ssdnerf_conv_wgrad_f16(ctypes.byref(a), N.stream_ptr()))
    return dw


def colsum(src, channels, out, c0=0):
    """out[c] += sum over rows of src[..., c0 + c]; src fp16 [..., stride] contiguous, out fp32 [channels]"""
    N.require_cuda(src, out)
    stride = src.shape[-1]
    N.check(N.lib().ssdnerf_colsum_f16(N.ptr(src), c_u64(src.numel() // stride), N.c_u32(stride), N.c_u32(c0), N.c_u32(channels),
                                       N.ptr(out), N.stream_ptr()))
    return out


def transpose_f16(src_ptr, dst, rows, cols, row_stride, stride1, n1, stride2, n2):
    N.check(N.lib().ssdnerf_transpose_f16(N.c_void_p(src_ptr), N.ptr(dst), N.c_u32(rows), N.c_u32(cols), c_ll(row_stride), c_ll(stride1),
                                          N.c_u32(n1), c_ll(stride2), N.c_u32(n2), N.stream_ptr()))
    return dst


def _bgemm(a_ptr, a_strides, k, b_ptr, b_strides, n, T, heads, B, out_ptr, out_strides, out_f32, alpha, narrow=False):
    """batched GEMM over (head, batch): out[b,h,t,:n] = alpha * A[b,h,t,:k] @ Bm[b,h,:n,:k]^T (strides in bytes for A / Bm, elements for out)"""
    g = GemmArgs()
    g.a1, g.k1 = a_ptr, k
    g.a1_strides = (c_u64 * 3)(*a_strides)
    g.d1, g.d2, g.d3, g.b1, g.b2, g.b3 = T, heads, B, 128, 1, 1
    g.taps = 1
    g.b, g.n, g.n_rows_b, g.bx2, g.bx3, g.b_batched = b_ptr, n, n, heads, B, 1
    g.b_strides = (c_u64 * 3)(*b_strides)
    g.bn, g.alpha = 0, alpha
    g.out, g.out_f32 = out_ptr, int(out_f32)
    g.so1, g.so2, g.so3 = out_strides
    if narrow:
        g.algo = ALGO_NARROW
    _launch(g)


def attn_backward(qkv, d_o, heads, scale, ws, narrow=False):
    """Attention data gradient (softmax(scale q k^T) v, legacy head layout of modules.py:36-48) by recomputation on the tensor cores:
    qkv fp16 [B,T,3c] (saved by the forward), d_o fp16 [B,T,c] -> dqkv fp16 [B,T,3c].  `ws(name, shape, dtype)` supplies scratch."""
    B, T, c3 = qkv.shape
    c = c3 // 3
    ch = c // heads
    L, s = N.lib(), N.stream_ptr
    S = attn_scores(qkv, heads, scale, out=ws('S', (B, heads, T, T), torch.float32), narrow=narrow)
    P = ws('P', (B, heads, T, T), torch.float16)
    N.check(L.ssdnerf_softmax_rows(N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(P), s()))
    qp, dop = qkv.data_ptr(), d_o.data_ptr()
    TT = T * T
    # dP[b,h,t,s] = d_o[b,t,h,:] . v[b,s,h,:]   (into the score buffer, which is dead after the softmax)
    _bgemm(dop, (c * 2, ch * 2, T * c * 2), ch, qp + 2 * ch * 2, (c3 * 2, 3 * ch * 2, T * c3 * 2), T, T, heads, B,
           S.data_ptr(), (T, TT, heads * TT), True, 1.0, narrow)
    dS = ws('dS', (B, heads, T, T), torch.float16)
    N.check(L.ssdnerf_softmax_bwd_rows(N.ptr(P), N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(dS), s()))
    Pt = transpose_f16(P.data_ptr(), ws('Pt', (B, heads, T, T), torch.float16), T, T, T, TT, heads, heads * TT, B)
    dSt = transpose_f16(dS.data_ptr(), ws('dSt', (B, heads, T, T), torch.float16), T, T, T, TT, heads, heads * TT, B)
    qt = transpose_f16(qp, ws('qt', (B, heads, ch, T), torch.float16), T, ch, c3, 3 * ch, heads, T * c3, B)
    kt = transpose_f16(qp + ch * 2, ws('kt', (B, heads, ch, T), torch.float16), T, ch, c3, 3 * ch, heads, T * c3, B)
    dot = transpose_f16(dop, ws('dot', (B, heads, ch, T), torch.float16), T, ch, c, ch, heads, T * c, B)
    dqkv = ws('dqkv', (B, T, c3), torch.float16)
    a_tt = (T * 2, TT * 2, heads * TT * 2)
    b_ct = (T * 2, ch * T * 2, heads * ch * T * 2)
    o_str = (c3, 3 * ch, T * c3)
    dp = dqkv.data_ptr()
    _bgemm(dS.data_ptr(), a_tt, T, kt.data_ptr(), b_ct, ch, T, heads, B, dp, o_str, False, scale, narrow)          # dq = scale dS k
    _bgemm(dSt.data_ptr(), a_tt, T, qt.data_ptr(), b_ct, ch, T, heads, B, dp + ch * 2, o_str, False, scale, narrow)  # dk = scale dS^T q
    _bgemm(Pt.data_ptr(), a_tt, T, dot.data_ptr(), b_ct, ch, T, heads, B, dp + 2 * ch * 2, o_str, False, 1.0, narrow)  # dv = P^T d_o
    return dqkv


def dropout_f16(x, seed, p):
    """in-place inverted dropout with the mask a pure function of (seed, element index)"""
    if p <= 0:
        return x
    N.require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    N.check(N.lib().ssdnerf_dropout_f16(N.ptr(x), ctypes.c_ulonglong(x.numel()), ctypes.c_ulonglong(seed & (2 ** 64 - 1)), N.c_f32(p),
                                        N.stream_ptr()))
    return x
