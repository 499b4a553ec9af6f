"""Inception-v3 features of FID / KID on the native kernels (csrc/inception.cu, ssdnerf_b200/inception.py) against torch and the oracle.

Bars, fixed on the CPU before any GPU run (tests/test_inception_cpu.py, DESIGN.md §6d):
  * each convolution form: relative L2 <= 1e-4 against F.conv2d in float64 on the same fp16-rounded operands, rounded to fp16 as the
    kernel stores (what is left is fp32 accumulation order and the rounding flips it causes);
  * pools: max exact, average within 1 fp16 ulp of float64 torch;
  * preprocessing: u8 bit-exact, normalised values within 1 fp16 ulp of the oracle;
  * the network: per-image feature relative L2 against the float32 oracle below BAR_128 (smooth 128 x 128 images, upsampled) and
    BAR_299 (a 299 x 299 image), twice what emulating the native fp16 storage in float64 moves the features on the fixture."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import inception_port as ip
from tests.test_inception_cpu import BAR_128, BAR_299, GOLDEN, _tf_module

pytestmark = pytest.mark.gpu

ASSET = os.path.join('work_dirs', 'cache', 'inception-2015-12-05.pt')


def _lib():
    from ssdnerf_b200 import _lib as N
    return N


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope='module')
def sd(golden):
    return ip.fixture_state_dict(golden)


@pytest.fixture(scope='module')
def net(sd):
    from ssdnerf_b200.inception import InceptionV3
    return InceptionV3.from_state_dict(sd)


def _rel_rows(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm(dim=1) / b.norm(dim=1)).numpy()


CONV_CASES = [
    # n, h, w, cin, cout, kh, kw, stride, pad_h, pad_w
    (2, 35, 35, 48, 64, 5, 5, 1, 2, 2),          # 5 x 5 pad 2
    (2, 17, 17, 128, 128, 1, 7, 1, 0, 3),        # 1 x 7
    (2, 17, 17, 160, 192, 7, 1, 1, 3, 0),        # 7 x 1
    (2, 8, 8, 384, 384, 1, 3, 1, 0, 1),          # 1 x 3
    (2, 8, 8, 448, 384, 3, 1, 1, 1, 0),          # 3 x 1 (K not a multiple of 64)
    (2, 299, 299, 16, 32, 3, 3, 2, 0, 0),        # valid stride 2, 299 -> 149
    (2, 149, 149, 32, 32, 3, 3, 1, 0, 0),        # valid, 149 -> 147
    (1, 147, 147, 32, 64, 3, 3, 1, 1, 1),        # same, 147
    (3, 73, 73, 64, 80, 1, 1, 1, 0, 0),          # 1 x 1 at 73
    (2, 73, 73, 80, 192, 3, 3, 1, 0, 0),         # valid, 73 -> 71
    (2, 35, 35, 288, 384, 3, 3, 2, 0, 0),        # valid stride 2, 35 -> 17
    (2, 17, 17, 192, 320, 3, 3, 2, 0, 0),        # valid stride 2, 17 -> 8
    (5, 8, 8, 2048, 192, 1, 1, 1, 0, 0),         # 1 x 1 at 8, K 2048
]


@pytest.mark.parametrize('relu', [1, 0])
@pytest.mark.parametrize('case', CONV_CASES, ids=lambda c: 'x'.join(map(str, c)))
def test_conv_forms_match_torch(cuda, case, relu):
    n, h, w, cin, cout, kh, kw, s, ph, pw = case
    if not relu and case != CONV_CASES[0] and case != CONV_CASES[5]:
        pytest.skip('relu off on two shapes only')
    N = _lib()
    g = torch.Generator().manual_seed(hash(case) % (1 << 31))
    # input and output live in channel slices of wider maps: 16 channels before, 8 after
    xs, ys = cin + 24, cout + 24
    xfull = torch.randn(n, h, w, xs, generator=g).half()
    x = xfull[..., 16:16 + cin]
    wt = (torch.randn(cout, kh, kw, cin, generator=g) / (cin * kh * kw) ** 0.5).half()
    b = torch.randn(cout, generator=g) * 0.1
    oh, ow = (h + 2 * ph - kh) // s + 1, (w + 2 * pw - kw) // s + 1
    sentinel = torch.full((n, oh, ow, ys), 7.0).half()
    xd, wd, bd, yd = xfull.to(cuda), wt.to(cuda), b.to(cuda), sentinel.to(cuda)
    N.check(N.lib().ssdnerf_incep_conv_f16(N.c_void_p(xd.data_ptr() + 32), N.c_u32(n), N.c_u32(h), N.c_u32(w), N.c_u32(cin),
                                           N.c_u32(xs), N.ptr(wd), N.ptr(bd), N.c_u32(cout), N.c_u32(kh), N.c_u32(kw), N.c_u32(s),
                                           N.c_u32(ph), N.c_u32(pw), N.c_int(relu), N.c_void_p(yd.data_ptr() + 32), N.c_u32(ys),
                                           N.stream_ptr()))
    y = yd.cpu()
    ref = F.conv2d(x.permute(0, 3, 1, 2).double().to(cuda), wt.permute(0, 3, 1, 2).double().to(cuda), b.double().to(cuda), stride=s,
                   padding=(ph, pw))
    if relu:
        ref = ref.relu()
    ref = ref.permute(0, 2, 3, 1).half().double().cpu()
    got = y[..., 16:16 + cout].double()
    rel = float((got - ref).norm() / ref.norm())
    assert rel <= 1e-4, rel
    assert torch.equal(y[..., :16], sentinel[..., :16]) and torch.equal(y[..., 16 + cout:], sentinel[..., 16 + cout:])


@pytest.mark.parametrize('mode,n,h,w,c', [(0, 2, 147, 147, 64), (0, 2, 71, 71, 192), (0, 2, 35, 35, 288), (0, 2, 17, 17, 768),
                                          (1, 2, 35, 35, 288), (1, 2, 17, 17, 768), (1, 3, 8, 8, 1280), (2, 3, 8, 8, 2048)])
def test_pools_match_torch(cuda, mode, n, h, w, c):
    N = _lib()
    g = torch.Generator().manual_seed(mode * 100 + h)
    x = torch.randn(n, h, w, c, generator=g).half()
    oh, ow = ((h - 3) // 2 + 1, (w - 3) // 2 + 1) if mode == 0 else (h, w)
    ys = c + 16                                                         # into a channel slice at offset 8
    yd = torch.full((n, oh, ow, ys), 3.0).half().to(cuda)
    xd = x.to(cuda)
    N.check(N.lib().ssdnerf_incep_pool_f16(N.ptr(xd), N.c_u32(n), N.c_u32(h), N.c_u32(w), N.c_u32(c), N.c_u32(c), N.c_int(mode),
                                           N.c_void_p(yd.data_ptr() + 16), N.c_u32(ys), N.stream_ptr()))
    y = yd.cpu()
    xt = x.permute(0, 3, 1, 2).double()
    if mode == 0:
        ref = F.max_pool2d(xt, 3, 2)
    elif mode == 1:
        ref = F.avg_pool2d(xt, 3, 1, 1, count_include_pad=False)
    else:
        ref = F.max_pool2d(xt, 3, 1, 1)
    ref = ref.permute(0, 2, 3, 1)
    got = y[..., 8:8 + c].double()
    if mode == 1:
        ulp = (ref.half().double().abs() * 2.0 ** -10).clamp_min(2.0 ** -24)
        assert ((got - ref).abs() <= ulp).all()
    else:
        assert torch.equal(got, ref)
    assert (y[..., :8] == 3).all() and (y[..., 8 + c:] == 3).all()


@pytest.mark.parametrize('h,w', [(128, 128), (299, 299), (64, 96), (300, 517)])
def test_prep_kernel(cuda, h, w):
    N = _lib()
    g = torch.Generator().manual_seed(h + w)
    n = 3
    x = torch.rand(n, 3, h, w, generator=g) * 2.2 - 1.1
    k = torch.arange(256, dtype=torch.float64)
    edge = ((k - 128) / 127.5).float()
    edge = torch.cat([edge, torch.nextafter(edge, edge + 1), torch.nextafter(edge, edge - 1), torch.tensor([-1.0, 1.0])])
    flat = x.view(-1)
    flat[:edge.numel()] = edge
    xd = x.to(cuda)
    out = torch.empty(n, 299, 299, 16, dtype=torch.float16, device=cuda)
    u8 = torch.empty(n, 3, h, w, dtype=torch.uint8, device=cuda)
    N.check(N.lib().ssdnerf_incep_prep_f16(N.ptr(xd), N.c_u32(n), N.c_u32(h), N.c_u32(w), N.ptr(out), N.ptr(u8), N.stream_ptr()))
    assert torch.equal(u8.cpu(), ip.quantize(x))
    assert torch.equal(u8.cpu(), (x * 127.5 + 128).clamp(0, 255).to(torch.uint8))
    o = out.cpu()
    assert (o[..., 3:] == 0).all()
    ref = ip.preprocess(x).permute(0, 2, 3, 1)
    got = o[..., :3].double()
    ulp = (ref.abs() * 2.0 ** -10).clamp_min(2.0 ** -24)
    assert ((got - ref).abs() <= ulp + 1e-6).all(), float((got - ref).abs().max())
    if (h, w) == (299, 299):
        assert torch.equal(got, ref.half().double())


@torch.no_grad()
def test_network_matches_oracle_on_fixture(cuda, golden, sd, net):
    P = {k: (w.float().to(cuda), b.float().to(cuda)) for k, (w, b) in ip.folded_params(sd).items()}
    for key, fkey, bar in (('u128', 'feat128', BAR_128), ('u299', 'feat299', BAR_299)):
        x = ip.fixture_images(golden, key).to(cuda)
        got = net(x)
        with torch.backends.cudnn.flags(allow_tf32=False):
            ref32 = ip.forward(P, ip.preprocess(x.cpu(), torch.float32).to(cuda))
        e32 = _rel_rows(got, ref32)
        e64 = _rel_rows(got, torch.from_numpy(golden[fkey]))
        print(key, 'rel vs fp32 oracle', e32, 'vs fixture', e64)
        assert (e32 < bar).all() and (e64 < bar).all()


def _smooth(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(n, 3, 8, 8, generator=g) * 2 - 1, size=(h, w), mode='bicubic', align_corners=False)
    return (base + 0.15 * torch.randn(n, 3, h, w, generator=g)).clamp(-1, 1)


@torch.no_grad()
def test_network_bench_batch(cuda, sd, net):
    """one bench val_cond batch (16 scenes x 251 views = 4016 images at 128 x 128) against the float32 oracle"""
    x = _smooth(4016, 128, 128, 11).to(cuda)
    got = net(x)
    P = {k: (w.float().to(cuda), b.float().to(cuda)) for k, (w, b) in ip.folded_params(sd).items()}
    ref = torch.empty_like(got)
    with torch.backends.cudnn.flags(allow_tf32=False):
        for j in range(0, 4016, 251):
            ref[j:j + 251] = ip.forward(P, ip.preprocess(x[j:j + 251].cpu(), torch.float32).to(cuda))
    e = _rel_rows(got, ref)
    print('bench batch rel L2: median', np.median(e), 'max', e.max())
    assert np.isfinite(got.cpu().numpy()).all()
    assert np.median(e) < BAR_128 / 2 and e.max() < BAR_128


@torch.no_grad()
def test_chunk_independence_and_run_to_run_identity(cuda, sd, net):
    from ssdnerf_b200.inception import InceptionV3, image_bytes
    x = _smooth(11, 128, 128, 5).to(cuda)
    a = net(x)
    assert torch.equal(a, net(x))
    small = InceptionV3.from_state_dict(sd, workspace_bytes=3 * image_bytes())
    assert small.chunk() == 3
    assert torch.equal(a, small(x))
    assert torch.equal(a[4:5], net(x[4:5]))


@torch.no_grad()
def test_fidkid_native_against_oracle_features(cuda, sd, net, tmp_path):
    from ssdnerf_b200.metrics import FIDKID
    real, fake = _smooth(48, 128, 128, 21).to(cuda), (_smooth(48, 128, 128, 22) * 0.8).to(cuda)
    P = {k: (w.float().to(cuda), b.float().to(cuda)) for k, (w, b) in ip.folded_params(sd).items()}

    def oracle_fn(b):
        with torch.backends.cudnn.flags(allow_tf32=False):
            return ip.forward(P, ip.preprocess(b.cpu(), torch.float32).to(cuda))

    path = str(tmp_path / 'inception-2015-12-05.pt')
    torch.jit.save(_tf_module(sd), path)
    results = []
    for kw in (dict(inception_args=dict(type='StyleGAN', inception_path=path)), dict(feature_fn=oracle_fn)):
        m = FIDKID(num_images=48, num_subsets=10, max_subset_size=32, **kw)
        for j in range(0, 48, 16):
            m.feed(real[j:j + 16], 'reals')
            m.feed(fake[j:j + 16], 'fakes')
        results.append(m.summary(generator=torch.Generator().manual_seed(0)))
    (fid_n, _, _, kid_n), (fid_o, _, _, kid_o) = results
    print('native fid / kid', fid_n, kid_n, 'oracle', fid_o, kid_o)
    assert abs(fid_n - fid_o) <= 0.05 * abs(fid_o)
    assert abs(kid_n - kid_o) <= 0.05 * abs(kid_o) + 1e-3


@pytest.mark.skipif(not os.path.isfile(ASSET), reason=f'{ASSET} (the StyleGAN Inception TorchScript) is not present')
@torch.no_grad()
def test_asset_torchscript_against_native(cuda):
    """the real asset: its own TorchScript on the GPU vs the native extractor loaded from it (name mapping and resize rule)"""
    from ssdnerf_b200.inception import InceptionV3
    from ssdnerf_b200.metrics import frechet_distance, feature_statistics
    ts = torch.jit.load(ASSET, map_location=cuda).eval()
    net = InceptionV3.load(ASSET)
    a, b = _smooth(64, 128, 128, 31).to(cuda), _smooth(64, 128, 128, 32).to(cuda)
    feats = []
    for x in (a, b):
        ref = ts(ip.quantize(x), return_features=True).float()
        got = net(x)
        e = _rel_rows(got, ref)
        print('asset rel L2 max', e.max())
        assert e.max() < 1e-2
        feats.append((got, ref))
    fid_n = frechet_distance(*feature_statistics(feats[0][0]), *feature_statistics(feats[1][0]))[0]
    fid_t = frechet_distance(*feature_statistics(feats[0][1]), *feature_statistics(feats[1][1]))[0]
    assert abs(fid_n - fid_t) <= 0.01 * abs(fid_t)
