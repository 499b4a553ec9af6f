"""Weight-gradient pass of the UNet (C ABI section 4c, `unet_train.WeightGradPass`) vs torch / oracle autograd.

Bars: the pixel-axis GEMM multiplies fp16 operands exactly and accumulates in fp32 -> vs torch's fp32 convolution weight gradient on the SAME
fp16-rounded operands: relative L2 <= 1e-4.  Whole network: every parameter's gradient vs autograd of the fp32 oracle: relative L2 <=
2e-2 per parameter and <= 6e-3 over all parameters together (fp16 activations + fp16 loss-scaled gradient storage; the measured values are
printed and recorded in DESIGN.md)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import unet_port as up
from tests.test_unet_bwd_gpu import SMALL, _nhwc, _rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('mode,B,H,cin,cout', [('s1', 2, 16, 128, 64), ('s2', 2, 16, 64, 128), ('up', 1, 8, 64, 64), ('1x1', 3, 8, 192, 64),
                                               ('s1', 4, 8, 64, 64)])
def test_conv_wgrad_matches_torch(cuda, mode, B, H, cin, cout):
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(H + cin)
    W = H
    x = torch.randn(B, cin, H, W, generator=g).half().float()
    taps = 1 if mode == '1x1' else 9
    stride = 2 if mode == 's2' else 1
    xin = F.interpolate(x, scale_factor=2, mode='nearest') if mode == 'up' else x
    w = torch.zeros(cout, cin, 3 if taps == 9 else 1, 3 if taps == 9 else 1, requires_grad=True)
    y = F.conv2d(xin, w, None, stride=stride, padding=1 if taps == 9 else 0)
    gy = torch.randn(y.shape, generator=g).half().float()
    ref, = torch.autograd.grad((y * gy).sum(), w)
    gyd, xd = _nhwc(gy).half().to(cuda), _nhwc(x).half().to(cuda)
    if mode == '1x1':        # channel concat of two sources (shortcut over a skip connection): 128 + 64
        dw = torch.zeros(cout, 1, cin, dtype=torch.float32, device=cuda)
        U.conv_wgrad(gyd, xd[..., :128].contiguous(), dw, cout, 128, dw_c0=0)
        U.conv_wgrad(gyd, xd, dw, cout, 64, x_c0=128, dw_c0=128)
        got = dw.view(cout, cin, 1, 1)
    else:
        dw = torch.full((cout, 9, cin), 1.0, dtype=torch.float32, device=cuda)          # accumulated into
        U.conv_wgrad(gyd, xd, dw, cout, cin, taps=9, stride=stride, up=(mode == 'up'))
        got = (dw - 1.0).view(cout, 3, 3, cin).permute(0, 3, 1, 2)
    err = _rel_l2(got, ref)
    print(mode, 'wgrad rel l2', err)
    assert err < 1e-4
    # a forced split over the pixel axis gives the same sums
    if mode == 's1':
        dw2 = torch.zeros(cout, 9, cin, dtype=torch.float32, device=cuda)
        U.conv_wgrad(gyd, xd, dw2, cout, cin, taps=9, ksplit=B * H * W // 64)
        assert _rel_l2(dw2.view(cout, 3, 3, cin).permute(0, 3, 1, 2), ref) < 1e-4


def test_conv_wgrad_rejects_bad_shapes(cuda):
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    gy = torch.zeros(1, 8, 8, 64, dtype=torch.float16, device=cuda)
    x = torch.zeros(1, 8, 8, 64, dtype=torch.float16, device=cuda)
    with pytest.raises(N.SSDNeRFNativeError):
        U.conv_wgrad(gy, x, torch.zeros(64, 9, 64, device=cuda), 64, 32, taps=9)              # cin % 64
    with pytest.raises(N.SSDNeRFNativeError):
        U.conv_wgrad(gy, x, torch.zeros(64, 9, 64, device=cuda), 64, 64, taps=9, stride=2)    # sizes do not match the stride


def test_colsum_dropout_and_channel_sums(cuda):
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    g = torch.Generator().manual_seed(8)
    src = torch.randn(1000, 192, generator=g).half()
    out = torch.ones(128, device=cuda)
    U.colsum(src.to(cuda), 128, out, c0=64)
    torch.testing.assert_close(out.cpu() - 1, src.float()[:, 64:].sum(0), rtol=1e-5, atol=1e-3)
    # dropout: deterministic in (seed, index), keep fraction and scale
    x = torch.ones(1 << 20, dtype=torch.float16, device=cuda)
    a, b, c = x.clone(), x.clone(), x.clone()
    U.dropout_f16(a, 1234, 0.1); U.dropout_f16(b, 1234, 0.1); U.dropout_f16(c, 1235, 0.1)
    assert torch.equal(a, b) and not torch.equal(a, c)
    keep = float((a != 0).float().mean())
    assert abs(keep - 0.9) < 2e-3 and abs(float(a.max()) - 1 / 0.9) < 2e-3 and abs(float(a.float().mean()) - 1.0) < 3e-3
    # GroupNorm channel sums -> d gamma, d beta, d scale, d shift vs autograd
    B, H, W, C = 2, 8, 8, 256
    xx = (torch.randn(B, C, H, W, generator=g) * 1.3).half().float()
    gamma, beta = (1 + 0.2 * torch.randn(C, generator=g)).requires_grad_(True), (0.2 * torch.randn(C, generator=g)).requires_grad_(True)
    ss = (torch.randn(B, 2 * C, generator=g) * 0.3).requires_grad_(True)
    dy = torch.randn(B, C, H, W, generator=g).half().float()
    y = F.silu(F.group_norm(xx, 32, gamma, beta, 1e-5) * (1 + ss[:, :C, None, None]) + ss[:, C:, None, None])
    rg, rb, rss = torch.autograd.grad((y * dy).sum(), [gamma, beta, ss])
    x1 = _nhwc(xx).half().to(cuda)
    q = x1.float().view(B, H * W, C // 4, 4)
    stats = (True, torch.stack([q.sum(dim=(1, 3)), (q * q).sum(dim=(1, 3))], dim=-1).contiguous(), None)
    cs = torch.full((B, C, 2), 7.0, device=cuda)
    ssd = ss.detach().to(cuda).contiguous()
    U.gn_bwd(x1, None, stats, gamma.detach().to(cuda), beta.detach().to(cuda), _nhwc(dy).half().to(cuda),
             torch.empty(B, H, W, C, dtype=torch.float16, device=cuda), scale_shift_ptr=N.c_void_p(ssd.data_ptr()), ss_batch_stride=2 * C,
             silu=True, csum=cs)
    r1, r2 = cs[..., 0].cpu(), cs[..., 1].cpu()
    one_s = 1 + ss.detach()[:, :C]
    assert _rel_l2((one_s * r2).sum(0), rg) < 2e-3 and _rel_l2((one_s * r1).sum(0), rb) < 2e-3
    assert _rel_l2(torch.cat([gamma.detach() * r2 + beta.detach() * r1, r1], dim=1), rss) < 2e-3


def _weight_grad_case(cfg, spec, sd, B, res, cuda, oracle_device, bar_each, bar_all, r=None):
    from ssdnerf_b200.unet import DenoisingUnetMod
    g = torch.Generator().manual_seed(21)
    x = torch.randn(B, 18, res, res, generator=g)
    if r is None:
        r = torch.randn(B, 18, res, res, generator=g) * 1e-3
    t = torch.tensor([999, 400, 19][:B])
    m = DenoisingUnetMod(**cfg)
    m.load_state_dict(sd, strict=True)
    m = m.to(cuda).train()
    xg = x.to(cuda).requires_grad_(True)
    v = m(xg, t.to(cuda))
    (v * r.to(cuda)).sum().backward()
    sdo = {k: p.detach().clone().to(oracle_device).requires_grad_(True) for k, p in sd.items()}
    xo = x.to(oracle_device).requires_grad_(True)
    vo = up.unet_forward(sdo, spec, xo, t.to(oracle_device))
    names = list(sdo)
    grads = torch.autograd.grad((vo * r.to(oracle_device)).sum(), [xo] + [sdo[k] for k in names], allow_unused=True)
    assert _rel_l2(xg.grad, grads[0]) < 5e-3
    got = dict(m.named_parameters())
    assert set(got) == set(names)
    worst, num, den = [], 0.0, 0.0
    for k, gr in zip(names, grads[1:]):
        assert gr is not None and got[k].grad is not None, k
        assert got[k].grad.shape == gr.shape and torch.isfinite(got[k].grad).all(), k
        a, b = got[k].grad.double().cpu(), gr.double().cpu()
        num += float((a - b).square().sum()); den += float(b.square().sum())
        worst.append((_rel_l2(a, b), k))
    worst.sort(reverse=True)
    print('all-parameter rel l2 %.2e; worst parameters:' % (num / den) ** 0.5, [(f'{e:.1e}', k) for e, k in worst[:5]])
    assert (num / den) ** 0.5 < bar_all
    assert worst[0][0] < bar_each, worst[:5]
    return m


def test_small_unet_weight_gradients(cuda):
    spec = up.unet_spec(**{k: v for k, v in SMALL.items() if k != 'use_scale_shift_norm'})
    sd = up.random_state_dict(spec, seed=1, std=0.04)
    m = _weight_grad_case(SMALL, spec, sd, 3, 32, cuda, torch.device('cpu'), 2e-2, 6e-3)
    # the optimizer step changes the packed weights; the next forward must see them (engine re-pack keyed on parameter versions)
    opt = torch.optim.SGD(m.parameters(), lr=1e-2)
    x = torch.randn(3, 18, 32, 32, device=cuda)
    t = torch.tensor([5, 6, 7], device=cuda)
    with torch.no_grad():
        v0 = m(x, t).clone()
    opt.step()
    with torch.no_grad():
        v1 = m(x, t)
    assert float((v1 - v0).abs().max()) > 0


def test_full_size_unet_weight_gradients(cuda):
    """the 122.4 M-parameter UNet of the shipped configs, B=2, against the fp32 oracle on the same GPU (TF32 off)"""
    full = dict(image_size=128, in_channels=18, base_channels=128, channels_cfg=[1, 2, 2, 4, 4], resblocks_per_downsample=2,
                num_heads=4, attention_res=[32, 16, 8], use_scale_shift_norm=True, dropout=0.0)
    spec = up.unet_spec()
    sd = up.random_state_dict(spec, seed=7, std=0.02)
    up.fp32_reference_mode()
    _weight_grad_case(full, spec, sd, 2, 128, cuda, cuda, 3e-2, 8e-3)


def test_dropout_training_forward_backward_consistent(cuda):
    """ResBlock dropout (0.1 in the recons configs; 0.5 here so that a wrong mask would halve the correlation): the backward and the
    weight-gradient pass regenerate the forward's mask -- finite-difference check of d(v . r) along a random direction of the weight
    right behind the dropout, seed held fixed.  The bar (30 %) covers the fp16 run-to-run noise of two forwards (~10 % of the
    difference at this step size) plus the third-order term of the central difference; a mask mismatch shows up as ~50 %."""
    from ssdnerf_b200.unet import DenoisingUnetMod
    cfg = dict(SMALL, dropout=0.5)
    m = DenoisingUnetMod(**cfg)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for p_ in m.parameters():            # incl. the zero-initialised last convolution of every block
            if p_.dim() > 1:
                p_.copy_(torch.randn(p_.shape, generator=g) * 0.04)
    assert any(k.endswith('conv_2.2.weight') for k in m.state_dict())      # mmgen key layout with the Dropout module in the Sequential
    m = m.to(cuda).train()
    x, r = torch.randn(2, 18, 32, 32, generator=g).to(cuda), torch.randn(2, 18, 32, 32, generator=g).to(cuda)
    t = torch.tensor([100, 700], device=cuda)
    torch.manual_seed(11)
    v = m(x, t)
    (v * r).sum().backward()
    torch.manual_seed(11)
    v_same = m(x, t)
    assert _rel_l2(v_same.detach(), v.detach()) < 5e-3          # same seed -> same mask (run-to-run noise floor only)
    torch.manual_seed(12)
    assert _rel_l2(m(x, t).detach(), v.detach()) > 2e-2          # another mask
    m.eval()
    with torch.no_grad():
        assert _rel_l2(m(x, t), v.detach()) > 2e-2               # eval: no dropout
    m.train()
    p = dict(m.named_parameters())['mid_blocks.0.conv_2.2.weight']          # the convolution right behind the dropout
    d = torch.randn_like(p) * 0.01
    ana = float((p.grad * d).sum())
    vals = []
    for sgn in (1, -1):
        with torch.no_grad():
            p.add_(sgn * d)
        torch.manual_seed(11)
        vals.append(float((m(x, t).detach() * r).sum()))
        with torch.no_grad():
            p.sub_(sgn * d)
    num = (vals[0] - vals[1]) / 2
    print('dropout directional derivative: analytic', ana, 'finite difference', num)
    assert abs(ana - num) < 0.3 * abs(num) + 1e-3
