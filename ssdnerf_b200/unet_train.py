"""Weight-gradient pass of the denoising UNet (training of the denoiser: lib/models/autodecoders/diffusion_nerf.py:66-189,
`loss_diffusion.backward()` + `optimizer['diffusion'].step()`).

The input-gradient pass (`UNetEngine.backward_nhwc`, csrc/unet_bwd.cu) already produces d loss / d (output of every layer); this
module turns those into parameter gradients while the walker still holds them:

  convolution / linear weights   `ssdnerf_conv_wgrad_f16` (csrc/wgrad.cu): pixel-axis GEMM on mma.sync tensor cores, operands read as
                                 they lie in HBM (NHWC) and transposed by ldmatrix.trans; 3x3 taps, stride 2 and the nearest-x2
                                 upsample are loader address arithmetic
  their biases                   `ssdnerf_colsum_f16`
  GroupNorm gamma / beta and the per-sample (scale, shift) of NormWithEmbedding
                                 linear in the two per-(image, channel) sums `ssdnerf_gn_bwd` emits on request (`channel_sums`)
  time embedding MLP + every block's embedding Linear
                                 [B x 512]-sized: PyTorch autograd over the tiny graph emb -> (scale, shift) rows, fed with the d(scale,
                                 shift) assembled above

GroupNorm-applied activations are not kept by the forward (they live in shared scratch); the pass re-applies the norm from the saved
raw tensor + statistics right before the weight-gradient GEMM that needs it.  Gradients arrive loss-scaled in fp16 (see unet_bwd.cu) and
are un-scaled in fp32 at the end (`finish`).
"""
import math

import torch

from . import _lib as N
from . import unet_ops as U


def _pad64(c):
    return (c + 63) // 64 * 64


def check_trainable(m):
    """the weight-gradient pass covers what every paper config uses: widths that are multiples of 64 and GroupNorm(32).  Anything else
    (the tiled-triplane config's 80 / 160 / 320 channels with GroupNorm(16)) raises naming itself; its sampling, guidance and
    guide_optim run natively."""
    from .unet import is_narrow, unet_widths
    if is_narrow(m) or m.num_groups != 32:
        raise NotImplementedError(f'training the denoiser with channel widths {unet_widths(m)} and GroupNorm({m.num_groups}) is not built: the '
                                  f'weight-gradient pass covers widths that are multiples of 64 with GroupNorm(32), not the tiled-triplane '
                                  f'config\'s 80 / 160 / 320 channels with GroupNorm(16); sampling, guidance and guide_optim run natively')


class WeightGradPass:
    """Collects parameter gradients during one walk of the tape.  `grads[param] = fp32 tensor in the parameter's shape`.
    Models outside `check_trainable` are refused."""

    def __init__(self, eng):
        check_trainable(eng.m)
        self.eng = eng
        self.grads = {}
        self.d_ss = torch.zeros(eng.B, eng.ss_total, dtype=torch.float32, device=eng.dev)

    # ------------------------------------------------------------------ helpers
    def csum(self, C):
        return self.eng._buf(('wg', 'csum', C), (self.eng.B, C, 2), torch.float32)

    def _add(self, param, g):
        """g: a tensor this pass owns (fresh buffer or a view of one) -- stored as is, no defensive copy"""
        g = g.reshape(param.shape)
        old = self.grads.get(param)
        self.grads[param] = g if old is None else old.add_(g)

    def _conv(self, weight, bias, gy, xs, taps=1, stride=1, up=False):
        """gy fp16 [B,Ho,Wo,Cg>=cout]; xs = list of (tensor [B,Hi,Wi,Cx], channels used) concatenated along the input-channel axis"""
        cout, cin = weight.shape[0], weight.shape[1]
        cout_p = _pad64(cout)
        assert gy.shape[-1] >= cout_p, (gy.shape, cout)
        k_total = sum(_pad64(c) for _, c in xs)
        dw = torch.zeros(cout_p, taps, k_total, dtype=torch.float32, device=self.eng.dev)
        off, cols = 0, []
        for x, c in xs:
            cp = _pad64(c)
            assert x.shape[-1] >= cp
            U.conv_wgrad(gy, x, dw, cout_p, cp, taps=taps, stride=stride, up=up, dw_c0=off)
            cols.append((off, c))
            off += cp
        parts = [dw[:cout, :, o:o + c] for o, c in cols]
        g = parts[0] if len(parts) == 1 else torch.cat(parts, dim=2)          # [cout, taps, cin]
        assert g.shape[2] == cin
        if taps == 9:
            g = g.view(cout, 3, 3, cin).permute(0, 3, 1, 2)                   # -> [cout, cin, ky, kx]
        self._add(weight, g.contiguous())
        if bias is not None:
            db = torch.zeros(cout_p, dtype=torch.float32, device=self.eng.dev)
            U.colsum(gy, cout_p, db)
            self._add(bias, db[:cout])

    def _norm(self, norm, cs, ss_off=None):
        """GroupNorm affine (+ NormWithEmbedding scale / shift) gradients from the channel sums cs [B, C, 2] = (sum dy', sum dy' * xhat)"""
        r1, r2 = cs[..., 0], cs[..., 1]
        if ss_off is None:
            self._add(norm.weight, r2.sum(0))
            self._add(norm.bias, r1.sum(0))
            return
        C = cs.shape[1]
        one_s = 1.0 + self.eng.ss_cur[:, ss_off:ss_off + C]
        self._add(norm.weight, (one_s * r2).sum(0))
        self._add(norm.bias, (one_s * r1).sum(0))
        gam, bet = norm.weight.detach().float(), norm.bias.detach().float()
        self.d_ss[:, ss_off:ss_off + C] = gam * r2 + bet * r1            # y = (xhat * gamma + beta) * (1 + scale) + shift
        self.d_ss[:, ss_off + C:ss_off + 2 * C] = r1

    def _gn_apply(self, x1, x2, st, gamma, beta, out, silu, ss_off=None):
        """re-apply a GroupNorm of the forward from its saved statistics descriptor (no statistics pass)"""
        eng = self.eng
        B, H, W, C1 = x1.shape
        C2 = x2.shape[-1] if x2 is not None else 0
        L, s = N.lib(), N.stream_ptr()
        ss = N.c_void_p(eng.ss_cur.data_ptr() + 4 * ss_off) if ss_off is not None else None
        quad, s1, s2 = st
        if quad:
            N.check(L.ssdnerf_gn_apply_q(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(eng.groups), N.ptr(s1),
                                         N.ptr(s2), N.ptr(gamma), N.ptr(beta), ss, N.c_longlong(eng.ss_total), N.c_f32(1e-5),
                                         N.c_int(int(silu)), N.ptr(out), s))
        else:
            N.check(L.ssdnerf_gn_apply(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(eng.groups), N.ptr(s1),
                                       N.ptr(gamma), N.ptr(beta), ss, N.c_longlong(eng.ss_total), N.c_f32(1e-5), N.c_int(int(silu)),
                                       N.ptr(out), s))
        return out

    # ------------------------------------------------------------------ per-op hooks (called by UNetEngine.backward_nhwc)
    def out(self, r, g_v, cs):
        eng, m = self.eng, self.eng.m
        x = r['x']
        B, H, W, c = x.shape
        a = self._gn_apply(x, None, r['st'], eng.out_norm['g'], eng.out_norm['b'], eng._buf(('wg', 'a', H, c), (B, H, W, c)), True)
        self._conv(m.out.conv.weight, m.out.conv.bias, g_v, [(a, c)], taps=9)
        self._norm(m.out.gn, cs)

    def res_second(self, r, g, cs2):
        """second half of a ResBlock (conv_2, NormWithEmbedding): g = d loss / d block output, cs2 = channel sums of its norm backward"""
        eng = self.eng
        d, h1 = r['d'], r['h1']
        p = d['mod']
        B, H, W, cout = h1.shape
        ss_off = eng.ss_offsets[d['idx']]
        a2 = self._gn_apply(h1, None, r['st2'], d['g2'], d['b2'], eng._buf(('wg', 'a', H, cout), (B, H, W, cout)), True, ss_off)
        eng._dropout(a2, d['idx'])
        self._conv(p.conv_2[-1].weight, p.conv_2[-1].bias, g, [(a2, cout)], taps=9)
        self._norm(p.norm_with_embedding.norm, cs2, ss_off)

    def res_first(self, r, g, d_h1, cs1):
        """first half (conv_1, its GroupNorm over the skip concat, the 1x1 shortcut): d_h1 = d loss / d conv_1 output"""
        eng = self.eng
        d, x, sk = r['d'], r['x'], r['sk']
        p = d['mod']
        B, H, W, C1 = x.shape
        cin = d['cin']
        a = self._gn_apply(x, sk, r['st1'], d['g1'], d['b1'], eng._buf(('wg', 'a', H, cin), (B, H, W, cin)), True)
        self._conv(p.conv_1[2].weight, p.conv_1[2].bias, d_h1, [(a, cin)], taps=9)
        self._norm(p.conv_1[0], cs1)
        if hasattr(p, 'shortcut'):
            xs = [(x, C1)] + ([(sk, sk.shape[-1])] if sk is not None else [])
            self._conv(p.shortcut.weight, p.shortcut.bias, g, xs, taps=1)

    def attn(self, r, g, dqkv, cs):
        eng = self.eng
        d, x, qkv = r['d'], r['x'], r['qkv']
        p = d['mod']
        B, H, W, c = x.shape
        T, heads = H * W, d['heads']
        o = eng._attn_core(qkv.view(B * T, 3 * c), B, T, c, heads, ('wg', 'o', T, c))
        self._conv(p.proj.weight, p.proj.bias, g.view(B, H, W, c), [(o.view(B, H, W, c), c)], taps=1)
        xn = self._gn_apply(x, None, r['st'], d['g'], d['b'], eng._buf(('wg', 'a', H, c), (B, H, W, c)), False)
        self._conv(p.qkv.weight, p.qkv.bias, dqkv.view(B, H, W, 3 * c), [(xn, c)], taps=1)
        self._norm(p.norm, cs)

    def down(self, r, g):
        p = r['d']['mod']
        self._conv(p.downsample.weight, p.downsample.bias, g, [(r['x'], r['x'].shape[-1])], taps=9, stride=2)

    def up(self, r, g):
        p = r['d']['mod']
        self._conv(p.conv.weight, p.conv.bias, g, [(r['x'], r['x'].shape[-1])], taps=9, up=True)

    def conv_in(self, r, g):
        eng = self.eng
        conv = eng.m.in_blocks[0][0]
        self._conv(conv.weight, conv.bias, g, [(eng.x_in, eng.cin_total)], taps=9)

    # ------------------------------------------------------------------ wrap-up
    def finish(self, inv_scale):
        """un-scale (inv_scale: 0-dim device tensor = 1 / loss scale); returns (grads dict, d loss / d scale-shift rows [B, ss_total])"""
        torch._foreach_mul_(list(self.grads.values()), inv_scale)
        return self.grads, self.d_ss * inv_scale


class _UNetFullGrad(torch.autograd.Function):
    """v = UNet(x_t, t) with gradients w.r.t. x_t AND every parameter (`params` = list(module.parameters()), passed so autograd routes
    their gradients): input-gradient pass + weight-gradient pass in one walk of the tape."""

    @staticmethod
    def forward(ctx, x_t, module, t, *params):
        B = x_t.shape[0]
        eng = module.engine(B, x_t.device, x_t.shape[-2:])
        with torch.enable_grad():       # tiny differentiable graph: time embedding -> per-block (scale, shift) rows
            emb = module.embedding(t.to(x_t.device))
            ss = eng.scale_shift_rows(emb, live=True)
        eng.ss_cur.copy_(ss.detach())
        eng.load_input_nchw(x_t.detach().float().contiguous())
        eng.new_dropout_seed(module.training)
        v = eng.forward_nhwc(save=True)
        ctx.eng, ctx.token, ctx.ss, ctx.params, ctx.module = eng, eng.fwd_token, ss, params, module
        return v.permute(0, 3, 1, 2)[:, :module.out_channels].contiguous()

    @staticmethod
    def backward(ctx, grad_v):
        eng = ctx.eng
        if eng.fwd_token != ctx.token:
            raise RuntimeError('UNet gradient: the engine ran another forward before this backward (activations overwritten)')
        dx, grads, d_ss = eng.backward_nchw(grad_v.contiguous().float(), weight_grads=True)
        live = [p for p in ctx.params if p.requires_grad and p not in grads]
        emb_params = [p for p in live if ctx.ss.requires_grad]
        if emb_params:
            eg = torch.autograd.grad(ctx.ss, emb_params, d_ss, allow_unused=True)
            grads.update({p: g for p, g in zip(emb_params, eg) if g is not None})
        out = tuple(grads.get(p) if p.requires_grad else None for p in ctx.params)
        return (dx if ctx.needs_input_grad[0] else None, None, None) + out


def forward_with_weight_grads(module, x_t, t):
    check_trainable(module)       # refuse before the forward rather than in the backward
    if module.concat_cond_channels > 0:
        raise NotImplementedError('training with concat_cond (image_cond) is not built (unused by the shipped configs)')
    return _UNetFullGrad.apply(x_t, module, t, *module.parameters())
