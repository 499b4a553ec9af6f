"""The UNet's kernels at the value ranges of a trained network rather than of a random initialisation.

1. fp16 gradient headroom of the backward.  `UNetEngine.backward_nchw` loss-scales d loss / d v to max |g| = 1024 and stores every
   interior gradient in fp16 (max 65504): 64x headroom.  Coherent upstream gradients (the gradient of a mean loss is nearly constant),
   shifted output-convolution weights or a GroupNorm with a low-variance input and a large gamma amplify past it.  The fp32 oracle
   proves each construction crosses the headroom; the native input and weight gradients must stay finite and meet the bars of
   test_unet_bwd_gpu / test_unet_wgrad_gpu.
2. GroupNorm statistics are one-pass (E[x^2] - E[x]^2 from fp32 sums).  Each statistics source is run at group |mean| / std in
   {0, 10, 30, 100, 300} against float64 `F.group_norm` of the fp16 tensor the kernel reads: up to 30 the bars of test_glue_kernels /
   test_groupnorm_backward hold; at 100 and 300 the outputs are finite and within 2x of the error measured on an H100 (`ENVELOPE`).
3. Attention at near one-hot softmax rows (logit gaps of 30-50 after scaling), the max in the first or the last K tile, one row with
   two tied maxima: fused flash attention, the unfused narrow-head composition and the recomputing backward vs float64.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import unet_port as up
from tests.test_train_step_gpu import _diffusion_model
from tests.test_unet_bwd_gpu import SMALL, _build, _rel_l2
from tests.test_unet_wgrad_gpu import _weight_grad_case

pytestmark = pytest.mark.gpu

SPEC = up.unet_spec(**{k: v for k, v in SMALL.items() if k != 'use_scale_shift_norm'})
HEADROOM = 65504.0 / 1024.0


# ================================================================================================================ gradient headroom
def _coherent_out_conv(sd):
    """output-convolution weights shifted to mean 0.5: its data gradient sums 18 x 9 = 162 same-signed products of a constant grad_v"""
    sd = dict(sd)
    sd['out.conv.weight'] = sd['out.conv.weight'] + 0.5
    return sd


def _low_variance_groupnorm(sd):
    """the last ResBlock's output scaled by 0.005 (its conv_2 and shortcut) feeding out.gn with gamma x 4: the GroupNorm backward
    multiplies by gamma * rstd ~ 4 / (0.005 std).  (A larger gamma makes the fp16 storage of the forward alone cost more than the
    4e-3 bar: gamma x 20 over a 0.02 std reaches 4.6e-3 in the oracle with its activations rounded to fp16.)"""
    sd = dict(sd)
    k = f'out_blocks.{len(SPEC["out_blocks"]) - 1}.0'
    for name in ('conv_2.1.weight', 'conv_2.1.bias', 'shortcut.weight', 'shortcut.bias'):
        sd[f'{k}.{name}'] = sd[f'{k}.{name}'] * 0.005
    sd['out.gn.weight'] = sd['out.gn.weight'] * 4
    return sd


CONSTRUCTIONS = dict(coherent_out_conv=_coherent_out_conv, low_variance_groupnorm=_low_variance_groupnorm)


class _GradPeak:
    """stands in for torch.nn.functional inside the oracle: every op output that requires a gradient records max |d loss / d output|"""

    def __init__(self):
        self.peak = 0.0

    def __getattr__(self, name):
        f = getattr(F, name)

        def op(*args, **kwargs):
            y = f(*args, **kwargs)
            if isinstance(y, torch.Tensor) and y.requires_grad:
                y.register_hook(self._record)
            return y
        return op

    def _record(self, g):
        self.peak = max(self.peak, float(g.abs().max()))


def _count_walks(monkeypatch):
    """-> dict counting backward_nchw calls ('calls') and the tape walks they made ('walks', 'checks': diagnostic walks)"""
    from ssdnerf_b200.unet import UNetEngine
    n = dict(calls=0, walks=0, checks=0)
    call, walk = UNetEngine.backward_nchw, UNetEngine.backward_nhwc

    def counted_call(self, *args, **kwargs):
        n['calls'] += 1
        return call(self, *args, **kwargs)

    def counted_walk(self, *args, **kwargs):
        n['checks' if kwargs.get('check') else 'walks'] += 1
        return walk(self, *args, **kwargs)
    monkeypatch.setattr(UNetEngine, 'backward_nchw', counted_call)
    monkeypatch.setattr(UNetEngine, 'backward_nhwc', counted_walk)
    return n


def _inputs(B=3):
    g = torch.Generator().manual_seed(12)
    return torch.randn(B, 18, 32, 32, generator=g), torch.tensor([999, 400, 19][:B])


@pytest.mark.parametrize('construction', sorted(CONSTRUCTIONS))
def test_input_gradient_beyond_fp16_headroom(cuda, monkeypatch, construction):
    sd = CONSTRUCTIONS[construction](up.random_state_dict(SPEC, seed=1, std=0.04))
    x, t = _inputs()
    gv = torch.full((3, 18, 32, 32), 0.37)              # d mean-loss / d v: constant
    rec = _GradPeak()
    with monkeypatch.context() as mp:
        mp.setattr(up, 'F', rec)
        xo = x.clone().requires_grad_(True)
        ref, = torch.autograd.grad(up.unet_forward(sd, SPEC, xo, t), xo, gv)
    amp = rec.peak / float(gv.abs().max())
    print(f'{construction}: largest interior gradient of the fp32 oracle = {amp:.0f} x max |grad_v|')
    assert amp > HEADROOM            # the construction really leaves the fp16 headroom of a single walk
    walks = _count_walks(monkeypatch)
    m = _build(SMALL, sd, cuda)
    xg = x.to(cuda).requires_grad_(True)
    with torch.enable_grad():
        got, = torch.autograd.grad(m(xg, t.to(cuda)), xg, gv.to(cuda))
    assert torch.isfinite(got).all()
    err = _rel_l2(got, ref)
    print(f'{construction}: d x_t rel l2 {err:.2e} after {walks["walks"]} walks')
    assert err < 4e-3
    assert walks['calls'] == 1 and walks['walks'] > 1 and walks['checks'] == 0


@pytest.mark.parametrize('construction', sorted(CONSTRUCTIONS))
def test_weight_gradients_beyond_fp16_headroom(cuda, monkeypatch, construction):
    sd = CONSTRUCTIONS[construction](up.random_state_dict(SPEC, seed=1, std=0.04))
    walks = _count_walks(monkeypatch)
    _weight_grad_case(SMALL, SPEC, sd, 3, 32, cuda, torch.device('cpu'), 2e-2, 6e-3, r=torch.full((3, 18, 32, 32), 0.37))
    assert walks['calls'] == 1 and walks['walks'] > 1


def test_stage2_train_step_beyond_fp16_headroom(cuda, monkeypatch):
    """`stage2_cars_uncond` (full-size UNet) with the output convolution shifted as in `_coherent_out_conv`: the MSE gradient of the
    coherent prediction crosses the headroom; the step's weight gradients and the weights after Adam stay finite"""
    model, _ = _diffusion_model(cuda, 'configs/paper_cfgs/stage2_cars_uncond.py')
    unet = model.diffusion.denoising
    with torch.no_grad():
        unet.out.conv.weight.add_(0.5)
    g = torch.Generator().manual_seed(1)
    stored = [dict(param=dict(code=torch.tanh(torch.randn(3, 6, 128, 128, generator=g)) * 0.8, density_grid=torch.zeros(64 ** 3).half(),
                              density_bitfield=torch.zeros(64 ** 3 // 8, dtype=torch.uint8))) for _ in range(2)]
    data = dict(scene_id=[0, 1], scene_name=['a', 'b'], code=stored)
    opt = dict(diffusion=torch.optim.Adam(model.diffusion.parameters(), lr=1e-4))
    walks = _count_walks(monkeypatch)
    out = model.train_step(data, opt)
    print('stage-2 step with a coherent output convolution: loss', out['log_vars']['loss_ddpm_mse'], 'backward walks', walks)
    bad = [k for k, p in unet.named_parameters() if p.grad is None or not torch.isfinite(p.grad).all() or not torch.isfinite(p).all()]
    assert not bad, bad[:8]
    assert walks['walks'] > walks['calls'] >= 1


def test_zero_upstream_gradient_gives_exact_zeros(cuda):
    sd = up.random_state_dict(SPEC, seed=1, std=0.04)
    x, t = _inputs()
    from ssdnerf_b200.unet import DenoisingUnetMod
    m = DenoisingUnetMod(**SMALL)
    m.load_state_dict(sd, strict=True)
    m = m.to(cuda).train()
    xg = x.to(cuda).requires_grad_(True)
    m(xg, t.to(cuda)).backward(torch.zeros(3, 18, 32, 32, device=cuda))
    assert int(torch.count_nonzero(xg.grad)) == 0
    nonzero = [k for k, p in m.named_parameters() if p.grad is None or int(torch.count_nonzero(p.grad))]
    assert not nonzero, nonzero[:8]


@pytest.mark.parametrize('bad', [float('inf'), float('nan')])
@pytest.mark.parametrize('train', [False, True])
def test_non_finite_upstream_gradient_stays_non_finite(cuda, monkeypatch, bad, train):
    """as in fp32 autograd: no retry, nothing hidden"""
    sd = up.random_state_dict(SPEC, seed=1, std=0.04)
    x, t = _inputs()
    gv = torch.randn(3, 18, 32, 32, generator=torch.Generator().manual_seed(2))
    gv[1, 4, 7, 9] = bad
    xo = x.clone().requires_grad_(True)
    ref, = torch.autograd.grad(up.unet_forward(sd, SPEC, xo, t), xo, gv)
    assert not torch.isfinite(ref).all()
    m = _build(SMALL, sd, cuda)
    if train:
        m.requires_grad_(True).train()
    walks = _count_walks(monkeypatch)
    xg = x.to(cuda).requires_grad_(True)
    with torch.enable_grad():
        m(xg, t.to(cuda)).backward(gv.to(cuda))
    assert not torch.isfinite(xg.grad).all()
    if train:
        assert not all(torch.isfinite(p.grad).all() for p in m.parameters())
    assert walks == dict(calls=1, walks=1, checks=0)


def test_backward_that_never_fits_names_the_layer(cuda):
    """output-convolution weights of mean 1e4: its data gradient exceeds fp16 at every loss-scale target"""
    from ssdnerf_b200 import _lib as N
    sd = up.random_state_dict(SPEC, seed=1, std=0.04)
    sd['out.conv.weight'] = sd['out.conv.weight'] + 1e4
    x, t = _inputs()
    m = _build(SMALL, sd, cuda)
    xg = x.to(cuda).requires_grad_(True)
    with torch.enable_grad(), pytest.raises(N.SSDNeRFNativeError, match='at layer `out`'):
        torch.autograd.grad(m(xg, t.to(cuda)), xg, torch.ones(3, 18, 32, 32, device=cuda))


# ================================================================================================================ GroupNorm at offsets
RATIOS = [0, 10, 30, 100, 300]
SOURCES = ['gn_stats_c512', 'gn_stats_tiled80', 'rowpair_bias', 'rowpair_residual', 'generic_bias', 'generic_residual']
# relative L2 (forward output, backward dx) vs float64, measured on an H100 80GB HBM3 (700 W power limit); asserted with a factor 2.
# At <= 30 every source is at the fp16 output rounding (2.1e-4 .. 4.6e-4).  The separate-statistics pass over the tiled config's
# 5-channel groups of 128 x 384 pixels (245760 values per group) loses the most: fp32 sums of that many values.
ENVELOPE = {
    ('gn_stats_c512', 100): (7.0e-4, 7.3e-4), ('gn_stats_c512', 300): (4.4e-3, 4.6e-3),
    ('gn_stats_tiled80', 100): (4.2e-3, 4.3e-3), ('gn_stats_tiled80', 300): (4.4e-2, 4.5e-2),
    ('rowpair_bias', 100): (1.7e-3, 1.7e-3), ('rowpair_bias', 300): (1.3e-2, 1.4e-2),
    ('rowpair_residual', 100): (1.8e-3, 1.9e-3), ('rowpair_residual', 300): (1.2e-2, 1.2e-2),
    ('generic_bias', 100): (8.1e-4, 8.0e-4), ('generic_bias', 300): (4.1e-3, 4.2e-3),
    ('generic_residual', 100): (8.5e-4, 8.7e-4), ('generic_residual', 300): (4.1e-3, 4.1e-3),
}


def _group_signs(B, C, G, g):
    """+-1 per (image, group), expanded to channels: [B, C]"""
    s = torch.randint(0, 2, (B, G), generator=g).float() * 2 - 1
    return s.repeat_interleave(C // G, dim=1)


def _gn_source(source, ratio, cuda, g):
    """-> (x fp16 NHWC on the GPU, stats descriptor as UNetEngine._gn leaves it, groups)"""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    L, s = N.lib(), N.stream_ptr()
    if source.startswith('gn_stats'):
        B, H, W, C, G = (2, 16, 16, 512, 32) if source == 'gn_stats_c512' else (2, 128, 384, 80, 16)
        off = ratio * _group_signs(B, C, G, g)
        x = (torch.randn(B, H, W, C, generator=g) + off[:, None, None, :]).half().to(cuda)
        st = torch.zeros(B, G, 2, device=cuda)
        N.check(L.ssdnerf_gn_stats(N.ptr(x), N.c_u32(C), None, N.c_u32(0), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(st), s))
        return x, (False, st, None), G
    # fused quad statistics of a convolution epilogue: row-pair kernel (128-pixel rows, 128 output channels) or generic tile kernel
    B, H, Cin, Cout = (2, 128, 128, 128) if source.startswith('rowpair') else (2, 32, 128, 256)
    xin = torch.randn(B, H, H, Cin, generator=g).half().to(cuda)
    wp = U.pack_conv_weight(torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05).to(cuda)
    std = float(U.conv3x3_f16(xin, wp, Cout, out_f32=True).std())
    signs = _group_signs(B, Cout, 32, g)
    q = torch.zeros(B, Cout // 4, 2, device=cuda)
    if source.endswith('bias'):         # one offset per channel: both images share it
        bias = (ratio * std * signs[0]).to(cuda)
        x = U.conv3x3_f16(xin, wp, Cout, bias=bias, qstats=q)
    else:
        res = (ratio * std * signs)[:, None, None, :].expand(B, H, H, Cout).half().contiguous().to(cuda)
        x = U.conv3x3_f16(xin, wp, Cout, residual=res, qstats=q)
    return x, (True, q, None), 32


@pytest.mark.parametrize('ratio', RATIOS)
@pytest.mark.parametrize('source', SOURCES)
def test_groupnorm_at_group_offsets(cuda, source, ratio):
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(7 + ratio)
    x, st, G = _gn_source(source, ratio, cuda, g)
    B, H, W, C = x.shape
    gamma, beta = (1 + 0.2 * torch.randn(C, generator=g)).to(cuda), (0.2 * torch.randn(C, generator=g)).to(cuda)
    out = torch.empty_like(x)
    L, s = N.lib(), N.stream_ptr()
    quad, s1, _ = st
    fn = L.ssdnerf_gn_apply_q if quad else L.ssdnerf_gn_apply
    stats_args = (N.ptr(s1), None) if quad else (N.ptr(s1),)
    N.check(fn(N.ptr(x), N.c_u32(C), None, N.c_u32(0), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), *stats_args, N.ptr(gamma), N.ptr(beta),
               None, N.c_longlong(0), N.c_f32(1e-5), N.c_int(1), N.ptr(out), s))
    dy = torch.randn(B, H, W, C, generator=g).half().to(cuda)
    dx = torch.empty_like(x)
    U.gn_bwd(x, None, st, gamma, beta, dy, dx, silu=True, groups=G)
    xr = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.silu(F.group_norm(xr, G, gamma.double(), beta.double(), 1e-5))
    gref, = torch.autograd.grad(ref, xr, dy.double().permute(0, 3, 1, 2))
    ref, gref = ref.detach().permute(0, 2, 3, 1), gref.permute(0, 2, 3, 1)
    grp = xr.detach().reshape(B, G, -1)
    realized = float((grp.mean(-1).abs() / grp.std(-1)).max())
    fwd, bwd = _rel_l2(out, ref), _rel_l2(dx, gref)
    fwd_max, bwd_max = float((out.double() - ref).abs().max()), float((dx.double() - gref).abs().max())
    print(f'GroupNorm {source} |mean|/std {ratio} (max realized {realized:.1f}): forward rel l2 {fwd:.2e} max abs {fwd_max:.2e}, '
          f'backward rel l2 {bwd:.2e} max abs {bwd_max:.2e}')
    assert torch.isfinite(out).all() and torch.isfinite(dx).all()
    if ratio <= 30:
        assert fwd_max < 2e-2 and fwd < 2e-3
        assert bwd_max < 2e-3 * float(gref.abs().max()) + 2e-3 and bwd < 1.5e-3
    else:
        e_fwd, e_bwd = ENVELOPE[source, ratio]
        assert fwd <= 2 * e_fwd and bwd <= 2 * e_bwd


# ================================================================================================================ peaked attention
def _peaked_qkv(B, T, heads, ch, g, tile=64):
    """legacy head layout [B, T, 3c] in fp16 with a near one-hot softmax row per query: key j(t) dominates with a logit 30-50 units
    (after the 1/sqrt(ch) scale) above the row's typical logit.  Query t % 3 == 0 picks its key in the first K tile, t % 3 == 1 in
    the last, the rest anywhere; query 5 sees keys 0 and T-1 (first and last tile) with identical k: two tied maxima."""
    scale = 1.0 / math.sqrt(ch)
    qkv = torch.zeros(B, T, heads, 3, ch)
    n = torch.randn(B, heads, T, ch, generator=g)
    n = n / n.norm(dim=-1, keepdim=True)
    n[..., T - 1, :] = n[..., 0, :]                            # keys 0 and T-1 identical
    j = torch.randint(0, T, (T,), generator=g)
    j[0::3] = torch.randint(1, tile, (len(j[0::3]),), generator=g)
    j[1::3] = torch.randint(T - tile, T - 1, (len(j[1::3]),), generator=g)
    j[j == T - 1] = T - 2
    j[j == 0] = 1
    j[5] = 0
    beta = 6.0
    alpha = (30 + 20 * torch.rand(B, heads, T, generator=g)) / (scale * beta)      # dominant logit = scale * alpha * beta in [30, 50]
    qkv[:, :, :, 1] = (beta * n).permute(0, 2, 1, 3)
    qkv[:, :, :, 0] = (alpha[..., None] * n[:, :, j]).permute(0, 2, 1, 3)
    qkv[:, :, :, 2] = torch.randn(B, T, heads, ch, generator=g)
    return qkv.reshape(B, T, 3 * heads * ch).half(), j


def _attn_ref(qkv, heads, scale):
    B, T, c3 = qkv.shape
    ch = c3 // 3 // heads
    x = qkv.double().view(B, T, heads, 3, ch).requires_grad_(True)
    q, k, v = x[..., 0, :], x[..., 1, :], x[..., 2, :]
    logits = torch.einsum('bthc,bshc->bhts', q, k) * scale
    o = torch.einsum('bhts,bshc->bthc', torch.softmax(logits, dim=-1), v).reshape(B, T, heads * ch)
    return x, logits.detach(), o


def _check_peaks(logits, j, T):
    top2 = logits.topk(2, dim=-1)
    assert torch.equal(top2.indices[..., 0][..., torch.arange(T) != 5], j.expand_as(top2.indices[..., 0])[..., torch.arange(T) != 5])
    gap = logits.max(-1).values - logits.median(-1).values
    assert float(gap.min()) > 25 and float(gap.max()) < 60
    assert torch.equal(top2.values[..., 5, 0], top2.values[..., 5, 1])     # the tie is exact in fp16 and in float64


@pytest.mark.parametrize('T,ch', [(1024, 64), (256, 128), (2048, 64)])
def test_flash_attention_peaked_rows(cuda, T, ch):
    from ssdnerf_b200 import unet_ops as U
    B, heads = 2, 2
    g = torch.Generator().manual_seed(T + ch)
    qkv, j = _peaked_qkv(B, T, heads, ch, g)
    scale = 1.0 / math.sqrt(ch)
    x, logits, ref = _attn_ref(qkv, heads, scale)
    _check_peaks(logits, j, T)
    out = U.flash_attn(qkv.to(cuda), heads, scale).double().cpu()
    ref = ref.detach()
    err = float((out - ref).abs().max())
    print(f'flash attention T {T} ch {ch}, peaked rows: max abs {err:.2e} (output range {float(ref.abs().max()):.2f})')
    assert err < 2e-3 * float(ref.abs().max()) + 1e-3


@pytest.mark.parametrize('T,ch,narrow', [(1024, 64, False), (256, 128, False), (768, 40, True), (192, 80, True)])
def test_unfused_attention_and_backward_peaked_rows(cuda, T, ch, narrow):
    """the unfused composition (the narrow heads of the tiled config) and the recomputing backward (every head width)"""
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    B, heads = 2, 2
    g = torch.Generator().manual_seed(T * ch)
    qkv, j = _peaked_qkv(B, T, heads, ch, g)
    scale = 1.0 / math.sqrt(ch)
    x, logits, ref = _attn_ref(qkv, heads, scale)
    _check_peaks(logits, j, T)
    qd = qkv.to(cuda)
    if narrow:
        S = U.attn_scores(qd, heads, scale, narrow=True)
        P = torch.empty(B, heads, T, T, dtype=torch.float16, device=cuda)
        N.check(N.lib().ssdnerf_softmax_rows(N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(P), N.stream_ptr()))
        vt = torch.empty(B, heads, ch, T, dtype=torch.float16, device=cuda)
        N.check(N.lib().ssdnerf_transpose_v(N.ptr(qd), N.c_u32(B), N.c_u32(T), N.c_u32(heads), N.c_u32(ch), N.ptr(vt), N.stream_ptr()))
        out = U.attn_pv(P, vt, narrow=True).double().cpu()
        fwd = _rel_l2(out, ref.detach())
        print(f'unfused attention T {T} ch {ch}, peaked rows: rel l2 {fwd:.2e}')
        assert fwd < 3e-3
    d_o = torch.randn(B, T, heads * ch, generator=g).half()
    gref, = torch.autograd.grad(ref, x, d_o.double())
    gref = gref.reshape(B, T, -1)
    ws = {}
    got = U.attn_backward(qd, d_o.to(cuda), heads, scale, lambda name, shape, dtype: ws.setdefault(name, torch.empty(shape, dtype=dtype, device=cuda)),
                          narrow=narrow).double().cpu()
    err, mx = _rel_l2(got, gref), float((got - gref).abs().max())
    print(f'attention backward T {T} ch {ch}, peaked rows: rel l2 {err:.2e} max abs {mx:.2e} (range {float(gref.abs().max()):.2f})')
    assert torch.isfinite(got).all()
    assert mx < 4e-3 * float(gref.abs().max())
    assert err < (5e-3 if narrow else 3e-3)
