"""Fused renderer (C-ABI ssdnerf_render_fwd) vs the CPU oracle of the reference's eval loop.

Bit-exact: per-ray sample count and the occupancy-bit index of every composited sample.
Floats (image / depth / weights_sum): tolerance stated per variant below."""
import numpy as np
import pytest
import torch

from oracle import render_port as rp
from tests.common import config1, spiral_poses

pytestmark = pytest.mark.gpu

# split-precision tensor-core MLP with fp32 accumulation (variant P): only round-off / fast-intrinsic differences vs the fp32 oracle
TOL_P = dict(rtol=2e-4, atol=2e-5)
# fp16 tensor-core MLP + fp16 planes (variant S): BASELINE.json north_star "1e-3 relative fp16 tolerance" on rendered RGB, taken on the
# image range [0, 1]; the bar is half the stated tolerance.
TOL_S = dict(rtol=0, atol=5e-4)


def _bitfields():
    ones = np.full(64 ** 3 // 8, 255, np.uint8)
    sphere = rp.sphere_bitfield()
    rand = np.random.default_rng(0).integers(0, 256, 64 ** 3 // 8, dtype=np.uint8)   # ~half the cells: many empty / occupied switches
    return {'ones': ones, 'sphere': sphere, 'random': rand}


def _run_gpu(variant, vid, params, code, bf, poses, intr, res, cuda, max_steps, explicit, trace_cap):
    from ssdnerf_b200 import renderer as R
    blob = R.pack_decoder_blob(params, vid, device=cuda)
    planes = R.pack_planes(code.to(cuda), vid)
    bft = torch.from_numpy(bf)[None].to(cuda)
    kw = dict(grid_size=64, max_steps=max_steps, trace_cap=trace_cap)
    if explicit:
        ro, rd = rp.get_cam_rays(poses[0], intr[0], res, res)
        out = R.render_fwd(vid, planes, (128, 128), bft, blob, rays_o=ro.reshape(1, -1, 3).to(cuda),
                           rays_d=rd.reshape(1, -1, 3).to(cuda), **kw)
    else:
        out = R.render_fwd(vid, planes, (128, 128), bft, blob, poses=poses.to(cuda), intrinsics=intr.to(cuda),
                           img_hw=(res, res), **kw)
    torch.cuda.synchronize()
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}


@pytest.mark.parametrize('variant', ['P', 'S'])
@pytest.mark.parametrize('grid', ['ones', 'sphere', 'random'])
@pytest.mark.parametrize('max_steps', [32, 256])
def test_config1_explicit_rays(cuda, variant, grid, max_steps):
    """SURVEY §8d config 1: 64x64 render, max_steps=32 (fixed step dt_max), bit-exact integer trace; also at the shipped
    max_steps=256, where the emulated sample budget and the ray's exit from the box end the march instead."""
    from ssdnerf_b200 import renderer as R
    vid = {'P': R.DEC_P, 'S': R.DEC_S}[variant]
    code, poses, intr = config1(variant[0])
    params = rp.make_decoder_params(variant[0], 0)
    bf = _bitfields()[grid]
    res = 64
    ro, rd = rp.get_cam_rays(poses[0], intr[0], res, res)
    ref = rp.render_eval_scene(params, ro.reshape(-1, 3).numpy(), rd.reshape(-1, 3).numpy(), code[0], bf, max_steps=max_steps,
                               return_trace=True)
    cap = ref['total_budget']
    out = _run_gpu(variant, vid, params, code, bf, poses, intr, res, cuda, max_steps, True, max(cap, 1))
    counts_ref = np.array([len(t) for t in ref['trace']], np.int32)
    counts = out['num_samples'][0]
    tr = out['trace'][0]
    if variant[0] != 'S':
        assert np.array_equal(counts, counts_ref)
    else:
        # The occupancy-hit SEQUENCE is integer work and bit-exact for every ray.  Where a ray STOPS depends on a float comparison
        # (T < 1e-4 on the accumulated transmittance): the fp16 MLP can cross that threshold one sample earlier or later than the fp32
        # oracle on a handful of rays -- then one trace is a prefix of the other and the extra sample carries a weight < 1e-4.
        differ = np.nonzero(counts != counts_ref)[0]
        assert len(differ) <= max(2, int(2e-3 * len(counts))), len(differ)
        assert np.abs(counts - counts_ref).max() <= 1
    for i in range(len(counts)):
        n = min(counts[i], counts_ref[i])
        assert list(tr[i, :n]) == ref['trace'][i][:n], f'ray {i}'
    tol = TOL_S if variant[0] == 'S' else TOL_P
    err = np.abs(out['image'][0] - ref['image'])
    print(f'{variant}/{grid}: image max abs err {err.max():.2e} mean {err.mean():.2e}; rays with a different sample count: {(counts != counts_ref).sum()}')
    np.testing.assert_allclose(out['image'][0], ref['image'], **tol)                 # every ray, including the ones that stopped one sample apart
    np.testing.assert_allclose(out['weights_sum'][0], ref['weights_sum'], **tol)
    np.testing.assert_allclose(out['depth'][0], ref['depth'], rtol=tol['rtol'], atol=tol['atol'] * 4)
    blend = ref['image'] + 1.0 * (1 - ref['weights_sum'][:, None])
    np.testing.assert_allclose(out['rgb'][0], blend, **tol)


def test_multi_scene_multi_view_P(cuda):
    """B=2 scenes x V=3 views at 32x32, density-pruned bitfields from the oracle's get_density, max_steps=256."""
    from ssdnerf_b200 import renderer as R
    g = torch.Generator().manual_seed(7)
    code = torch.randn(2, 3, 6, 128, 128, generator=g).clamp(-2, 2)
    params = rp.make_decoder_params('P', 2)
    rands = [torch.rand(64 ** 3, 3, generator=g) for _ in range(2)]
    _, bf = rp.get_density(params, code, rands, density_thresh=0.1)
    poses = torch.from_numpy(spiral_poses(3))[None].repeat(2, 1, 1, 1)
    intr = torch.tensor([32 * 131.25 / 128, 32 * 131.25 / 128, 16, 16]).expand(2, 3, 4).contiguous()
    blob = R.pack_decoder_blob(params, R.DEC_P, device=cuda)
    planes = R.pack_planes(code.to(cuda), R.DEC_P)
    ro, rd = rp.get_cam_rays(poses, intr, 32, 32)
    out = R.render_fwd(R.DEC_P, planes, (128, 128), torch.from_numpy(bf).to(cuda), blob,
                       rays_o=ro.reshape(2, -1, 3).to(cuda), rays_d=rd.reshape(2, -1, 3).to(cuda), max_steps=256)
    for b in range(2):
        ref = rp.render_eval_scene(params, ro[b].reshape(-1, 3).numpy(), rd[b].reshape(-1, 3).numpy(), code[b], bf[b], max_steps=256)
        np.testing.assert_allclose(out['image'][b].cpu().numpy(), ref['image'], **TOL_P)
        np.testing.assert_allclose(out['weights_sum'][b].cpu().numpy(), ref['weights_sum'], **TOL_P)


def test_schedule_emulation_budget(cuda):
    """all-ones grid, max_steps=32: rays crossing the cube want ~64 samples, so the reference host loop's budget
    (n_step = clamp(N // n_alive, 1, 8) quanta) binds; the fused kernel must truncate at exactly the same count."""
    from ssdnerf_b200 import renderer as R
    code, poses, intr = config1('P', seed=3)
    params = rp.make_decoder_params('P', 3)
    # make the medium thin so transmittance never terminates rays before the budget does
    params['density_net.0.bias'] = params['density_net.0.bias'] - 6.0
    bf = _bitfields()['ones']
    ro, rd = rp.get_cam_rays(poses[0], intr[0], 64, 64)
    ref = rp.render_eval_scene(params, ro.reshape(-1, 3).numpy(), rd.reshape(-1, 3).numpy(), code[0], bf, max_steps=32, return_trace=True)
    out = _run_gpu('P', R.DEC_P, params, code, bf, poses, intr, 64, cuda, 32, True, 0)
    counts_ref = np.array([len(t) for t in ref['trace']], np.int32)
    assert counts_ref.max() == ref['total_budget'] > 32
    assert np.array_equal(out['num_samples'][0], counts_ref)
    np.testing.assert_allclose(out['image'][0], ref['image'], **TOL_P)
