"""Occupancy-grid builder (csrc/density.cu) the way training, inverse rendering and guided sampling run it: decayed updates of
live fp16 / fp32 grids with invalid cells, one threshold for the whole batch, fp16 and fp32 saturation, and grid sizes, bounds
and plane shapes the shipped configs never use.

Every case is checked in two layers, so that MLP round-off cannot hide a logic error:
  * decode (toleranced): one update of a zero fp32 grid with decay 1 leaves sigma in the grid; it is compared with the float64
    decode of `render_port.point_decode` at the same jittered voxel centres;
  * update, threshold and pack (exact): the update kernel has no atomics and its decode does not depend on the grid dtype, so
    the same planes, blob and jitter give that same fp32 sigma again.  From it the new grid is an exact function of the prior
    grid (base_nerf.py:349-350 and 379-380, `_expected_grid`), the threshold a function of the new grid (:382-386) and the
    bitfield `packbits(grid, threshold)` (:387)."""
import numpy as np
import pytest
import torch

import oracle as orc
from oracle import render_port as rp

pytestmark = pytest.mark.gpu

FLT_MAX = float(torch.finfo(torch.float32).max)
P_RTOL = 2e-4                     # variant P decodes in fp32 with __expf
S_MEDIAN, S_MAX = 2e-3, 3e-2      # variant S rounds features and weights to fp16 (bounds of test_density_gpu's S test)
SHAPES = dict(P=(6, 128, 128), S=(32, 128, 128))


# ----------------------------------------------------------------------------------------------------------- inputs
def _params(variant, seed, bias):
    """Decoder weights whose density logit is `bias` higher than the random draw's and gains 0.75 x code channel 0: hidden units
    0 and 1 read +0.5 and -0.5 x channel 0 of each plane and feed the density head with +0.5 and -0.5, and
    silu(x) - silu(-x) = x.  No other unit reads channel 0.  The decoder is shared by the batch, so channel 0 is how a case
    gives each scene its own density level."""
    p = rp.make_decoder_params(variant, seed)
    w = p['base_net.0.weight'].clone()          # features in the reference order c*3 + plane: channel 0 is 0, 1, 2
    w[:, :3] = 0
    w[:2] = 0
    w[0, :3], w[1, :3] = 0.5, -0.5
    p['base_net.0.weight'] = w
    b = p['base_net.0.bias'].clone()
    b[:2] = 0
    p['base_net.0.bias'] = b
    wd = p['density_net.0.weight'].clone()
    wd[0, 0], wd[0, 1] = 0.5, -0.5
    p['density_net.0.weight'] = wd
    p['density_net.0.bias'] = p['density_net.0.bias'] + bias
    return p


def _code(variant, levels, seed, hw=None):
    """random triplanes [B,3,C,H,W]; channel 0 of scene b is levels[b] plus a little noise (its density level, see `_params`)"""
    g = torch.Generator().manual_seed(seed)
    C, H, W = SHAPES[variant] if hw is None else (SHAPES[variant][0], *hw)
    code = torch.randn(len(levels), 3, C, H, W, generator=g).clamp(-2, 2)
    code[:, :, 0] = torch.tensor(levels, dtype=torch.float32)[:, None, None, None] + 0.5 * code[:, :, 0]
    return code


def _sigma64(params, code, rand, G, bound):
    """float64 density of every scene at the (jittered) voxel centres of base_nerf.py:328-344, morton order [B, G^3]"""
    _, idx, xyzs = rp.voxel_centres(G, bound)
    if rand is not None:
        half = bound / G
        xyzs = xyzs + (rand * (2 * half) - half)
    out = torch.empty(code.shape[0], G ** 3, dtype=torch.float64)
    for b in range(code.shape[0]):
        out[b, idx] = rp.point_decode(params, xyzs, None, code[b], density_only=True, dtype=torch.float64)[0]
    return out


def _expected_grid(old, sigma32, decay):
    """base_nerf.py:349-350, 379-380 in the grid's dtype: tmp = sigma clamped to the dtype's max and cast; cells of value -1
    are kept"""
    tmp = sigma32.clamp(max=torch.finfo(old.dtype).max).to(old.dtype)
    return torch.where((old >= 0) & (tmp >= 0), torch.maximum(old * decay, tmp), old)


def _prior(sig64, dtype, seed, invalid=0.1):
    """a live grid: sigma x exp(U(-1, 1)), so that old * 0.9 wins in ~45 % of the voxels and sigma in the rest, with a fraction
    `invalid` of cells at -1"""
    g = torch.Generator().manual_seed(seed)
    old = sig64 * torch.exp(torch.rand(sig64.shape, generator=g, dtype=torch.float64) * 2 - 1)
    old = old.clamp(max=torch.finfo(dtype).max).to(dtype)
    old[torch.rand(sig64.shape, generator=g) < invalid] = -1
    return old


# ----------------------------------------------------------------------------------------------------------- kernel calls
def _device_inputs(variant, params, code, cuda):
    from ssdnerf_b200 import renderer as R
    vid = {'P': R.DEC_P, 'S': R.DEC_S}[variant]
    return vid, R.pack_planes(code.to(cuda), vid), R.pack_decoder_blob(params, vid, device=cuda)


def _update(vid, planes, hw, blob, grid, jitter, density_thresh, decay, G, bound):
    """one full update in place: -> bitfield [B, G^3/8] (device), threshold used (the kernel's thresh_out)"""
    from ssdnerf_b200 import density as D
    bits = torch.zeros(grid.shape[0], G ** 3 // 8, dtype=torch.uint8, device=grid.device)
    th = torch.full((1,), float('nan'), device=grid.device)
    D.update_extra_state(vid, planes, hw, blob, grid, bits, jitter, density_thresh=density_thresh, decay=decay, grid_size=G,
                         bound=bound, thresh_out=th)
    return bits, float(th)


def _sigma32(vid, planes, hw, blob, B, jitter, G, bound, cuda):
    """the kernel's own fp32 sigma: a decay-1 update of a zero fp32 grid"""
    grid = torch.zeros(B, G ** 3, device=cuda)
    _update(vid, planes, hw, blob, grid, jitter, 0.01, 1.0, G, bound)
    return grid.cpu()


# ----------------------------------------------------------------------------------------------------------- checks
def _decode_error(variant, sigma32, sig64):
    """-> (median, max) relative error of the kernel's sigma against the float64 decode (clamped to FLT_MAX like the kernel);
    asserts the variant's tolerance"""
    ref = sig64.clamp(max=FLT_MAX)
    floor = 1e-3 if variant == 'S' else 1e-30
    rel = (sigma32.double() - ref).abs() / ref.clamp(min=floor)
    med, mx = float(rel.median()), float(rel.max())
    if variant == 'P':
        assert mx < P_RTOL, (med, mx)
    else:
        assert med < S_MEDIAN and mx < S_MAX, (med, mx)
    return med, mx


def _check_thresh(grid, th, density_thresh):
    """thresh_out = min(mean(clamp(grid, 0)) over the whole batch, density_thresh); an fp16 grid's mean is an fp16 value
    (torch.mean of a half tensor), which may round differently from the float64 mean by one fp16 ulp"""
    dt = float(np.float32(density_thresh))
    mean = float(grid.double().clamp(min=0).mean())
    if mean >= dt:
        assert th == dt, (th, mean, dt)
    elif grid.dtype == torch.float32:
        assert th == pytest.approx(mean, rel=1e-6, abs=0), (th, mean)
    else:
        assert float(np.float16(th)) == th, f'fp16 grid mean {th!r} is not an fp16 value'
        ref = float(np.float16(mean))
        assert abs(th - ref) <= float(np.spacing(np.float16(min(th, ref)))), (th, ref)
    return mean


def _check_bits(bits, grid, th):
    """bits (numpy) == packbits(grid, th)"""
    exp = orc.packbits(grid.float().numpy().reshape(-1), th).reshape(grid.shape[0], -1)
    assert np.array_equal(bits, exp), f'{int(np.unpackbits(bits ^ exp).sum())} bits differ from packbits(grid, {th})'


def _assert_grid_equal(got, exp):
    assert got.dtype == exp.dtype
    same = (got == exp) | (torch.isnan(got) & torch.isnan(exp))
    if not bool(same.all()):
        i = int((~same).flatten().nonzero()[0])
        raise AssertionError(f'{int((~same).sum())} of {same.numel()} voxels differ; first at {i}: got {got.flatten()[i].item()!r}, '
                             f'expected {exp.flatten()[i].item()!r}')


# ----------------------------------------------------------------------------------------------------------- cases
# levels: code channel 0 per scene (the scene's density level); branch: where the batch mean lies against density_thresh
CASES = {
    # B = 3: one almost empty scene, one in between, one dense; the scene means straddle the threshold, the batch mean is below
    'live_P': dict(variant='P', levels=[-6.0, -3.0, 0.3], bias=-2.0, G=64, bound=1.0, density_thresh=0.1, branch='below',
                   straddle=True),
    'live_S': dict(variant='S', levels=[-6.0, -3.0, 0.3], bias=-2.0, G=64, bound=1.0, density_thresh=0.1, branch='below',
                   straddle=True),
    'live_P_above': dict(variant='P', levels=[-4.0, 1.0, 3.0], bias=0.0, G=64, bound=1.0, density_thresh=0.1, branch='above',
                         straddle=True),
    # default threshold 0.01, both branches; G = 32 with B = 3 has 384 partial sums (not a multiple of 1024)
    'g32_b3_thresh001_below': dict(variant='P', levels=[-6.0, -3.0, 0.0], bias=-4.0, G=32, bound=1.0, density_thresh=0.01,
                                   branch='below', straddle=True),
    'g32_b3_thresh001_above': dict(variant='P', levels=[-2.0, 0.0, 2.0], bias=-2.0, G=32, bound=1.0, density_thresh=0.01,
                                   branch='above'),
    # 2M voxels: the threshold kernel's partial-sum loop runs 8 times
    'g128': dict(variant='P', levels=[0.0], bias=-2.0, G=128, bound=1.0, density_thresh=0.1, branch='above'),
    'bound05': dict(variant='P', levels=[-2.0, 1.0], bias=-2.0, G=64, bound=0.5, density_thresh=0.01, branch='above'),
    # voxel centres beyond the planes: the border clamp
    'bound15': dict(variant='P', levels=[-2.0, 1.0], bias=-2.0, G=64, bound=1.5, density_thresh=0.1, branch='above'),
    # non-square planes for the variant-S gather (96 rows, 160 columns)
    'S_96x160': dict(variant='S', levels=[-2.0, 1.0], bias=-2.0, G=32, bound=1.0, density_thresh=0.1, branch='above', hw=(96, 160)),
    'P_96x160': dict(variant='P', levels=[-2.0, 1.0], bias=-2.0, G=32, bound=1.2, density_thresh=0.1, branch='above', hw=(96, 160)),
}
# saturation: sigma beyond 65504 in an fp16 grid, exp overflowing float32 in an fp32 grid; the logits straddle the limit
SATURATION = {
    torch.float16: dict(variant='P', levels=[-1.0, 1.0], bias=11.0, G=32, bound=1.0, density_thresh=0.1, branch='above'),
    torch.float32: dict(variant='P', levels=[-1.0, 1.0], bias=88.7, G=32, bound=1.0, density_thresh=0.1, branch='above'),
}
_CACHE = {}


def _case_inputs(name, c):
    """CPU inputs and float64 sigma of a case (shared by its fp16 and fp32 runs)"""
    if name not in _CACHE:
        seed = sum(map(ord, name))
        params = _params(c['variant'], seed, c['bias'])
        code = _code(c['variant'], c['levels'], 100 + seed, c.get('hw'))
        rand = torch.rand(c['G'] ** 3, 3, generator=torch.Generator().manual_seed(200 + seed))
        _CACHE[name] = params, code, rand, _sigma64(params, code, rand, c['G'], c['bound'])
    return _CACHE[name]


def _run_case(name, c, grid_dtype, cuda):
    """both layers for one case: decode of a zero fp32 grid against float64, then a decay-0.9 update of a live prior grid
    checked exactly (grid, threshold, bits)"""
    params, code, rand, sig64 = _case_inputs(name, c)
    B, G, bound, hw = code.shape[0], c['G'], c['bound'], tuple(code.shape[-2:])
    vid, planes, blob = _device_inputs(c['variant'], params, code, cuda)
    jitter = rand.to(cuda)
    sigma32 = _sigma32(vid, planes, hw, blob, B, jitter, G, bound, cuda)
    med, mx = _decode_error(c['variant'], sigma32, sig64)

    old = _prior(sig64, grid_dtype, 300 + sum(map(ord, name)))
    grid = old.to(cuda, copy=True)
    bits, th = _update(vid, planes, hw, blob, grid, jitter, c['density_thresh'], 0.9, G, bound)
    grid, bits = grid.cpu(), bits.cpu().numpy()
    _assert_grid_equal(grid, _expected_grid(old, sigma32, 0.9))
    invalid = old == -1
    assert bool((grid[invalid] == -1).all())
    assert 0.05 < float(invalid.double().mean()) < 0.15
    mean = _check_thresh(grid, th, c['density_thresh'])
    _check_bits(bits, grid, th)
    assert (mean < c['density_thresh']) == (c['branch'] == 'below'), (mean, c['density_thresh'])
    occupied = float(np.unpackbits(bits).mean())
    print(f'{name} {str(grid_dtype)[6:]}: decode rel err median {med:.2e} max {mx:.2e}; mean {mean:.4g} thresh {th:.4g}; '
          f'occupied {occupied:.3f}')
    return dict(old=old, grid=grid, bits=bits, th=th, mean=mean, sigma32=sigma32, sig64=sig64, occupied=occupied)


@pytest.mark.parametrize('grid_dtype', [torch.float16, torch.float32], ids=['fp16', 'fp32'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_decayed_update_of_live_grid(cuda, name, grid_dtype):
    """decay 0.9 on a live grid with invalid cells: decode within tolerance of float64, then grid bit-exact against the update
    formula from the kernel's own sigma, threshold = min(batch mean, density_thresh), bits = packbits(grid, threshold)"""
    c = CASES[name]
    r = _run_case(name, c, grid_dtype, cuda)
    old, grid = r['old'], r['grid']
    # the case covers what it is meant to: both sides of the max, both threshold branches, a mixed bitfield
    tmp, valid = r['sigma32'].to(grid_dtype), old >= 0
    decayed = float((valid & (old * 0.9 > tmp)).double().mean())
    fresh = float((valid & (tmp > old * 0.9)).double().mean())
    assert decayed > 0.05 and fresh > 0.05, (decayed, fresh)
    assert abs(r['mean'] / c['density_thresh'] - 1) > 0.05, 'batch mean too close to the threshold to tell the branches apart'
    assert 0.01 < r['occupied'] < 0.99, r['occupied']
    if c.get('straddle'):
        # the scene means lie on both sides of the batch threshold, so a per-scene threshold would change the sparse scene's bits
        scene_means = grid.double().clamp(min=0).mean(dim=1)
        assert float(scene_means.min()) < r['th'] < float(scene_means.max()), (scene_means.tolist(), r['th'])
        sparse = int(scene_means.argmin())
        own = orc.packbits(grid[sparse].float().numpy(), float(scene_means[sparse]))
        assert not np.array_equal(own, r['bits'][sparse])


@pytest.mark.parametrize('grid_dtype', [torch.float16, torch.float32], ids=['fp16', 'fp32'])
def test_saturated_density(cuda, grid_dtype):
    """fp16 grid: sigma beyond 65504 is stored as exactly 65504 (not inf); fp32 grid: exp overflows to inf and the grid holds
    FLT_MAX, whose sum makes the mean inf, so the threshold is density_thresh (as torch.mean gives in the reference)"""
    c = SATURATION[grid_dtype]
    r = _run_case(f'saturation_{str(grid_dtype)[6:]}', c, grid_dtype, cuda)
    limit = float(torch.finfo(grid_dtype).max)
    grid, sig64, valid = r['grid'], r['sig64'], r['old'] >= 0
    over = sig64 > limit * (1 + 1e-3)
    assert 0.1 < float(over.double().mean()) < 0.9, float(over.double().mean())
    assert bool((grid[over & valid] == limit).all())
    assert bool(torch.isfinite(grid).all())
    assert r['th'] == float(np.float32(c['density_thresh']))


# ----------------------------------------------------------------------------------------------------------- jitter
def _update_raw(vid, planes, hw, blob, grid, jitter, decay, G, bound, workspace):
    """ssdnerf_density_update through the C ABI as is (NULL jitter, NULL workspace); raises SSDNeRFNativeError on refusal"""
    from ssdnerf_b200 import _lib as N
    N.check(N.lib().ssdnerf_density_update(N.c_int(vid), N.ptr(planes), N.c_u32(hw[0]), N.c_u32(hw[1]), N.ptr(blob),
                                           N.c_u32(grid.shape[0]), N.c_u32(G), N.c_f32(bound), N.ptr(jitter), N.c_f32(decay),
                                           N.ptr(grid), N.c_int(int(grid.dtype == torch.float16)), N.ptr(workspace), N.stream_ptr()))


def test_jitter_default_and_constant(cuda):
    """jitter=None draws torch.rand(G^3, 3) on the device; a constant jitter of 0.5 puts every sample exactly on the voxel
    centre (the NULL-jitter path) and decodes like float64 at `render_port.voxel_centres`"""
    from ssdnerf_b200 import density as D
    name = 'g32_b3_thresh001_above'
    c = CASES[name]
    params, code, _, _ = _case_inputs(name, c)
    B, G, bound, hw = code.shape[0], c['G'], c['bound'], tuple(code.shape[-2:])
    vid, planes, blob = _device_inputs(c['variant'], params, code, cuda)
    runs = []
    for seed, explicit in ((7, False), (7, True), (8, False)):
        torch.cuda.manual_seed(seed)
        jitter = torch.rand(G ** 3, 3, device=cuda) if explicit else None
        grid = torch.zeros(B, G ** 3, dtype=torch.float16, device=cuda)
        bits, _ = _update(vid, planes, hw, blob, grid, jitter, c['density_thresh'], 0.9, G, bound)
        runs.append((grid, bits))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert not torch.equal(runs[0][0], runs[2][0])          # the draw is used

    half = torch.full((G ** 3, 3), 0.5, device=cuda)
    grids = [torch.zeros(B, G ** 3, device=cuda) for _ in range(2)]
    ws = D._workspace(B, G, cuda)
    _update_raw(vid, planes, hw, blob, grids[0], half, 1.0, G, bound, ws)
    _update_raw(vid, planes, hw, blob, grids[1], None, 1.0, G, bound, ws)
    assert torch.equal(grids[0], grids[1])
    _decode_error('P', grids[0].cpu(), _sigma64(params, code, None, G, bound))
    _decode_error('P', grids[0].cpu(), _sigma64(params, code, torch.full((G ** 3, 3), 0.5), G, bound))


# ----------------------------------------------------------------------------------------------------------- chains
FP16_ULP = 2.0 ** -10      # relative spacing of fp16 at the bottom of a binade
FP16_TINY = 2.0 ** -24     # fp16 subnormal spacing


def _chain_tol(grid_dtype):
    """(rtol, atol) of a grid built by the kernel against one built from float64 sigma: the decode tolerance, and for fp16 two
    ulps: rounding sigma to fp16 may land on the other side of a tie (one ulp), and a voxel that keeps old * decay carries
    that ulp down into the next lower binade, where it is two"""
    return (P_RTOL, 1e-30) if grid_dtype == torch.float32 else (P_RTOL + 2 * FP16_ULP, 2 * FP16_TINY)


@pytest.mark.parametrize('grid_dtype', [torch.float16, torch.float32], ids=['fp16', 'fp32'])
def test_decayed_chain_tracks_oracle(cuda, grid_dtype):
    """ten decay-0.9 updates in a row (inverse_code / val_guide), the code moving a little between them like an optimizer
    step: the kernel's grid stays within round-off of a chain driven by the float64 decode, that divergence does not grow, and
    a bit differs only where the float64 density lies within round-off of the threshold"""
    from ssdnerf_b200 import renderer as R
    G, steps, dt = 64, 10, 0.1
    params = _params('P', 31, -2.0)
    code = _code('P', [-4.0, -1.0], 131)
    blob = R.pack_decoder_blob(params, R.DEC_P, device=cuda)
    g = torch.Generator().manual_seed(231)
    rtol, atol = _chain_tol(grid_dtype)
    grid = torch.zeros(code.shape[0], G ** 3, dtype=grid_dtype, device=cuda)
    ref = torch.zeros(code.shape[0], G ** 3, dtype=grid_dtype)
    div, flips = [], 0
    for step in range(steps):
        rand = torch.rand(G ** 3, 3, generator=g)
        bits, th = _update(R.DEC_P, R.pack_planes(code.to(cuda), R.DEC_P), (128, 128), blob, grid, rand.to(cuda), dt, 0.9, G, 1.0)
        ref = _expected_grid(ref, _sigma64(params, code, rand, G, 1.0), 0.9)
        th_ref = min(float(ref.clamp(min=0).mean()), dt)
        bits_ref = orc.packbits(ref.float().numpy().reshape(-1), th_ref).reshape(code.shape[0], -1)
        got, exp = grid.cpu().double(), ref.double()
        err = (got - exp).abs() / (rtol * exp.abs() + atol)
        div.append(float((got - exp).abs().div(exp.abs().clamp(min=atol)).max()))
        assert float(err.max()) <= 1, (step, div[-1])
        assert th == pytest.approx(th_ref, rel=rtol), (step, th, th_ref)
        diff = np.unpackbits(bits.cpu().numpy() ^ bits_ref, axis=-1, bitorder='little').astype(bool)
        # voxel n of the bitfield is grid element n (morton order)
        near = ((exp - th_ref).abs() <= rtol * exp.abs() + atol + abs(th - th_ref)).numpy()
        assert not (diff & ~near).any(), (step, int((diff & ~near).sum()))
        flips += int(diff.sum())
        code = code + 0.02 * torch.randn(code.shape, generator=g)
    occupied = float(np.unpackbits(bits_ref).mean())
    assert 0.05 < occupied < 0.95, occupied
    assert max(div[steps // 2:]) <= 2 * max(div[:steps // 2]), div
    print(f'chain {str(grid_dtype)[6:]}: per-step max rel divergence {["%.2e" % d for d in div]}; {flips} bits flipped near '
          f'the threshold over {steps} steps')


# ----------------------------------------------------------------------------------------------------------- model
def test_model_update_after_decoder_step(cuda):
    """BaseNeRF.update_extra_state as train_step calls it (fp16 grid, decay 0.9, iter_density 0), an in-place optimizer step on
    the decoder, then again: the second update decodes with the updated weights (the packed blob follows Parameter._version)"""
    from ssdnerf_b200.nerf import BaseNeRF
    G, B = 64, 2
    params = _params('P', 32, -2.0)
    code = _code('P', [-2.0, 1.0], 132)
    model = BaseNeRF(code_size=(3, 6, 128, 128), grid_size=G, use_lpips_metric=False,
                     decoder=dict(type='TriPlaneDecoder', base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3],
                                  use_dir_enc=True, dir_layers=[16, 64]))
    sd = model.decoder.state_dict()
    sd.update(params)
    model.decoder.load_state_dict(sd)
    model = model.to(cuda)
    dec = model.decoder
    grid, bits = model.get_init_density_grid(B, cuda), model.get_init_density_bitfield(B, cuda)
    assert grid.dtype == torch.float16
    g = torch.Generator().manual_seed(232)
    opt = torch.optim.SGD(dec.parameters(), lr=1.0)
    rtol, atol = _chain_tol(torch.float16)
    for step in range(2):
        rand = torch.rand(G ** 3, 3, generator=g)
        old = grid.cpu()
        model.update_extra_state(dec, code.to(cuda), grid, bits, 0, density_thresh=0.1, jitter=rand.to(cuda))
        weights = {k: v.detach().cpu() for k, v in dec.decoder_params().items()}
        sig = _sigma64(weights, code, rand, G, 1.0)
        exp = _expected_grid(old, sig, 0.9).double()
        got = grid.cpu().double()
        assert float(((got - exp).abs() / (rtol * exp.abs() + atol)).max()) <= 1, step
        if step == 0:
            # a training step: raise the density bias by 0.7 and nudge every weight, in place
            for p in dec.parameters():
                p.grad = 0.01 * torch.randn(p.shape, generator=g).to(cuda)
            dec.density_net[0].bias.grad.fill_(-0.7)
            opt.step()
    # the step moved the densities far beyond the tolerance, so the weights before it could not have passed
    assert float((sig / _sigma64(params, code, rand, G, 1.0)).median()) > 1.5
    with pytest.raises(NotImplementedError):
        model.update_extra_state(dec, code.to(cuda), grid, bits, 16)


# ----------------------------------------------------------------------------------------------------------- refusals
def test_refusals_and_empty_batch(cuda):
    """a grid size that is not a power of two, an unknown decoder variant and a NULL workspace are refused; an empty batch is a
    no-op"""
    from ssdnerf_b200 import _lib as N, density as D
    name = 'g32_b3_thresh001_above'
    c = CASES[name]
    params, code, rand, _ = _case_inputs(name, c)
    G, hw = c['G'], tuple(code.shape[-2:])
    vid, planes, blob = _device_inputs(c['variant'], params, code, cuda)
    grid = torch.zeros(1, 48 ** 3, device=cuda)
    with pytest.raises(N.SSDNeRFNativeError, match='power of two'):
        D.update_extra_state(vid, planes, hw, blob, grid, torch.zeros(1, 48 ** 3 // 8, dtype=torch.uint8, device=cuda), grid_size=48)
    grid = torch.zeros(1, G ** 3, device=cuda)
    bits = torch.zeros(1, G ** 3 // 8, dtype=torch.uint8, device=cuda)
    with pytest.raises(N.SSDNeRFNativeError, match='unknown decoder variant'):
        D.update_extra_state(7, planes, hw, blob, grid, bits, grid_size=G)
    with pytest.raises(N.SSDNeRFNativeError, match='NULL'):
        _update_raw(vid, planes, hw, blob, grid, rand.to(cuda), 0.9, G, 1.0, None)
    with pytest.raises(N.SSDNeRFNativeError, match='NULL'):
        N.check(N.lib().ssdnerf_density_pack(N.ptr(grid), N.c_int(0), N.c_u32(1), N.c_u32(G), N.c_f32(0.1), N.ptr(bits), None, None,
                                             N.stream_ptr()))
    assert not bool(grid.any()) and not bool(bits.any())
    # an empty batch (whose tensors have no storage) does nothing
    th = torch.full((1,), 123.0, device=cuda)
    empty = torch.zeros(0, G ** 3, dtype=torch.float16, device=cuda)
    D.update_extra_state(vid, planes, hw, blob, empty, torch.zeros(0, G ** 3 // 8, dtype=torch.uint8, device=cuda),
                         rand.to(cuda), density_thresh=0.1, grid_size=G, thresh_out=th)
    assert float(th) == 123.0
