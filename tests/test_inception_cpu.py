"""CPU checks of the Inception-v3 feature extractor of FID / KID: the oracle against the torchvision-executed fixture, the resize rule's
closed form against the affine_grid / grid_sample composition, the u8 quantisation, BatchNorm folding, the TorchScript loader's
order-and-shape mapping, the fp16 precision probe behind the GPU bars, and FIDKID's errors without the weight file."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import inception_port as ip
from ssdnerf_b200 import inception as I
from ssdnerf_b200.metrics import FIDKID

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'reference_inception_v1.npz')
# per-image relative L2 of the features, fp16 storage (native path) vs float64; DESIGN.md §6d.  Twice the probe's maximum below.
BAR_128 = 0.09
BAR_299 = 1.2e-2


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope='module')
def params(golden):
    return ip.folded_params(ip.fixture_state_dict(golden))


def _rel(a, b):
    return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


@torch.no_grad()
def test_oracle_matches_torchvision_fixture(golden, params):
    taps = {}
    x = ip.fixture_images(golden, 'u128')
    assert np.array_equal(ip.quantize(x).numpy(), golden['u128'])
    f = ip.features(params, x, taps=taps)
    assert _rel(f, torch.from_numpy(golden['feat128'])) < 1e-10
    m5d = taps['Mixed_5d'][0, :8].permute(1, 2, 0)
    assert torch.allclose(m5d, torch.from_numpy(golden['mixed_5d']).double(), rtol=1e-6, atol=1e-6)
    f = ip.features(params, ip.fixture_images(golden, 'u299'))
    assert _rel(f, torch.from_numpy(golden['feat299'])) < 1e-10


@torch.no_grad()
def test_fp16_probe_is_within_the_bars(golden, params):
    """the native path's storage precision emulated in float64: what the GPU bars are set from"""
    f = ip.features(params, ip.fixture_images(golden, 'u128'), fp16=True)
    assert _rel(f, torch.from_numpy(golden['feat128'])) < BAR_128 / 2
    f = ip.features(params, ip.fixture_images(golden, 'u299'), fp16=True)
    assert _rel(f, torch.from_numpy(golden['feat299'])) < BAR_299 / 2


@pytest.mark.parametrize('h,w', [(128, 128), (64, 96), (17, 23), (300, 512), (299, 150), (1, 1)])
def test_resize_closed_form_equals_affine_grid_composition(h, w):
    g = torch.Generator().manual_seed(h * 1000 + w)
    u = torch.randint(0, 256, (2, 3, h, w), generator=g).double()
    a = ip.resize_closed_form(u)
    b = ip.resize_affine_grid(u)
    assert a.shape == b.shape == (2, 3, 299, 299)
    assert (a - b).abs().max().item() < 1e-9


def test_quantization_matches_torch_uint8_on_edges():
    ks = torch.arange(0, 256, dtype=torch.float64)
    exact = ((ks - 128) / 127.5).float()                       # x * 127.5 + 128 lands on (or next to) an integer
    xs = torch.cat([torch.tensor([-1.0, 1.0, 0.0, -1.5, 1.5, 1e-8, -1e-8]), exact, torch.nextafter(exact, exact + 1),
                    torch.nextafter(exact, exact - 1)]).float()
    want = (xs * 127.5 + 128).clamp(0, 255).to(torch.uint8)
    assert torch.equal(ip.quantize(xs), want)
    # the same computation in numpy float32 (separately rounded multiply and add, truncation): what the kernel states
    v = np.float32(xs.numpy()) * np.float32(127.5)
    v = (v + np.float32(128)).astype(np.float32)
    assert np.array_equal(np.trunc(np.clip(v, 0, 255)).astype(np.uint8), want.numpy())
    assert int(ip.quantize(torch.tensor([-1.0]))) == 0 and int(ip.quantize(torch.tensor([1.0]))) == 255


def test_bn_folding_is_exact_in_fp64():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 9, 11, generator=g, dtype=torch.float64)
    w = torch.randn(24, 16, 3, 1, generator=g, dtype=torch.float64)
    gamma, beta, mean = (torch.randn(24, generator=g, dtype=torch.float64) for _ in range(3))
    var = torch.rand(24, generator=g, dtype=torch.float64) + 0.1
    ref = F.batch_norm(F.conv2d(x, w, padding=(1, 0)), mean, var, gamma, beta, training=False, eps=1e-3)
    for fold in (I.fold_bn, ip.fold_bn):
        wf, bf = fold(w, gamma, beta, mean, var)
        assert torch.allclose(F.conv2d(x, wf, bf, padding=(1, 0)), ref, rtol=1e-12, atol=1e-12)


def test_package_spec_matches_oracle():
    assert I.CONVS == tuple(ip.CONVS) and len(I.CONVS) == 94
    assert abs(ip.shape_gflop() - 11.42) < 0.01


class _Leaf(torch.nn.Module):
    def forward(self, x):
        return x


def _tf_module(sd, order=None):
    """a scripted module holding the canonical weights under TF-style names (`conv_k` submodules with weight / beta / mean / var)"""
    root = torch.nn.Module()
    names = [c[0] for c in I.CONVS]
    for i in (order if order is not None else range(len(names))):
        leaf = _Leaf()
        p = names[i]
        leaf.register_parameter('weight', torch.nn.Parameter(sd[f'{p}.conv.weight'].float()))
        w = sd[f'{p}.bn.weight'].float()
        # TF has no BatchNorm scale: put gamma into the weights so the folded network is unchanged
        leaf.weight.data *= w.reshape(-1, 1, 1, 1)
        leaf.register_buffer('beta', sd[f'{p}.bn.bias'].float())
        leaf.register_buffer('mean', sd[f'{p}.bn.running_mean'].float() * w)
        leaf.register_buffer('var', sd[f'{p}.bn.running_var'].float())
        root.add_module(f'layer_{len(root._modules)}_{p.lower().replace(".", "_")}', leaf)
    root.add_module('output', torch.nn.Linear(2048, 1008))

    class Net(torch.nn.Module):
        def __init__(self, r):
            super().__init__()
            self.layers = r

        def forward(self, x):
            return x
    return torch.jit.script(Net(root))


def test_torchscript_loader_maps_by_order_and_shape(golden, tmp_path):
    sd = ip.fixture_state_dict(golden)
    path = str(tmp_path / 'incep.pt')
    torch.jit.save(_tf_module(sd), path)
    net = I.InceptionV3.load(path)
    ref = I.InceptionV3.from_state_dict(sd)
    for name, *_ in I.CONVS:
        (w1, b1), (w2, b2) = net._host[name], ref._host[name]
        assert (w1.float() - w2.float()).abs().max() <= 1e-3 * w2.float().abs().max(), name
        assert torch.allclose(b1, b2, rtol=1e-4, atol=1e-4), name


def test_torchscript_loader_refuses_swapped_branches_and_changed_shapes(golden, tmp_path):
    sd = ip.fixture_state_dict(golden)
    order = list(range(94))
    i1 = [c[0] for c in I.CONVS].index('Mixed_5b.branch1x1')
    order[i1], order[i1 + 1] = order[i1 + 1], order[i1]        # Mixed_5b's 192->64 and 192->48 1x1s
    path = str(tmp_path / 'swapped.pt')
    torch.jit.save(_tf_module(sd, order), path)
    with pytest.raises(ValueError, match=r"mixed_5b_branch5x5_1.*\(48, 192, 1, 1\).*\(64, 192, 1, 1\)"):
        I.InceptionV3.load(path)
    sd2 = dict(sd)
    sd2['Mixed_6b.branch7x7_2.conv.weight'] = sd['Mixed_6b.branch7x7_2.conv.weight'].transpose(2, 3).contiguous()   # 1x7 -> 7x1
    path = str(tmp_path / 'shape.pt')
    torch.jit.save(_tf_module(sd2), path)
    with pytest.raises(ValueError, match=r"mixed_6b_branch7x7_2.*\(128, 128, 7, 1\).*\(128, 128, 1, 7\)"):
        I.InceptionV3.load(path)


def test_from_state_dict_names_missing_and_misshapen_keys(golden):
    sd = ip.fixture_state_dict(golden)
    bad = dict(sd)
    del bad['Mixed_7c.branch_pool.bn.running_var']
    with pytest.raises(ValueError, match='Mixed_7c.branch_pool.bn.running_var'):
        I.InceptionV3.from_state_dict(bad)
    bad = dict(sd)
    bad['Mixed_5d.branch5x5_2.conv.weight'] = torch.zeros(64, 48, 3, 3)
    with pytest.raises(ValueError, match=r'Mixed_5d.branch5x5_2.conv.weight.*\(64, 48, 3, 3\)'):
        I.InceptionV3.from_state_dict(bad)


def test_fidkid_without_the_torchscript_names_the_path(tmp_path):
    path = str(tmp_path / 'cache' / 'inception-2015-12-05.pt')
    m = FIDKID(num_images=4, inception_args=dict(type='StyleGAN', inception_path=path))
    with pytest.raises(RuntimeError, match='inception-2015-12-05.pt'):
        m.feed(torch.zeros(2, 3, 8, 8), 'fakes')
    m = FIDKID(num_images=4, inception_args=dict(type='PyTorch'))
    with pytest.raises(NotImplementedError, match='PyTorch'):
        m.feed(torch.zeros(2, 3, 8, 8), 'fakes')
    with pytest.raises(RuntimeError, match='feature_fn'):
        FIDKID(num_images=4).feed(torch.zeros(2, 3, 8, 8), 'fakes')
