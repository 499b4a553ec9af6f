"""The fused inference renderer (ssdnerf_render_fwd: k_render_p3 for variant P, k_render_s2 for variant S) in the settings the shipped
configs call it with, against the CPU oracle of the reference's eval loop (oracle/render_port.py):

  * per-scene dt_gamma (DiffusionNeRF.render passes dt_gamma_scale * 2 / (fx + fy) for every scene);
  * camera mode with several views per scene, rectangular images, anisotropic off-centre intrinsics, on both the 8x4 patch-tile and
    the flat-tile path -- bit for bit against explicit rays made on the host with the kernel's own float32 operations;
  * per-scene sample budgets of the schedule-emulation fix-up pass, one binding and one not;
  * non-square, odd plane sizes;
  * base / colour pre-activations of +-100 and density logits beyond exp's float32 range (variant P).

Integer results (per-ray sample count, occupancy-bit trace) are bit-exact against the float32-MLP oracle for P and follow the prefix rule of
tests/test_render_gpu.py for S.  P's floats are compared with the float64-MLP oracle, S's with the float32 one, at the bars of
tests/test_render_gpu.py.  The preconditions that make each case meaningful need only the oracle and run without a GPU."""
import functools
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import render_port as rp
from tests.common import config1, spiral_poses
from tests.test_render_gpu import TOL_P, TOL_S

F32 = np.float32


def _bitfield(name):
    if name == 'ones':
        return np.full(64 ** 3 // 8, 255, np.uint8)
    if name.startswith('sphere'):
        return rp.sphere_bitfield(radius=float(name[6:] or 0.6))     # 'sphereR': voxel centres within radius R
    return np.random.default_rng(int(name[6:])).integers(0, 256, 64 ** 3 // 8, dtype=np.uint8)   # 'randomN': about half the cells


def _code(variant, seed, hw=(128, 128)):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, 3, 6 if variant == 'P' else 32, *hw, generator=g).clamp(-2, 2)


def _cam_rays(res=64):
    _, poses, intr = config1('P', res=res)
    ro, rd = rp.get_cam_rays(poses[0, 0], intr[0, 0], res, res)
    return ro.reshape(-1, 3).numpy(), rd.reshape(-1, 3).numpy()


def _counts(ref):
    return np.array([len(t) for t in ref['trace']], np.int32)


def _oracle(variant, params, ro, rd, code1, bf, **kw):
    """float32-MLP oracle (integer trace) and, for P, the float64-MLP oracle (floats)"""
    r32 = rp.render_eval_scene(params, ro, rd, code1, bf, return_trace=True, **kw)
    r64 = rp.render_eval_scene(params, ro, rd, code1, bf, dtype=torch.float64, **kw) if variant == 'P' else None
    return r32, r64


def _render(cuda, variant, params, code, bitfields, rays=None, cams=None, **kw):
    """one render_fwd of B scenes: rays = (rays_o, rays_d) [B,N,3] numpy, or cams = (poses [B,V,4,4], intrinsics [B,V,4], (h, w))"""
    from ssdnerf_b200 import renderer as R
    vid = R.DEC_P if variant == 'P' else R.DEC_S
    blob = R.pack_decoder_blob(params, vid, device=cuda)
    planes = R.pack_planes(code.to(cuda), vid)
    bft = torch.from_numpy(np.stack(bitfields)).to(cuda)
    hw = tuple(code.shape[-2:])
    if rays is not None:
        out = R.render_fwd(vid, planes, hw, bft, blob, rays_o=torch.from_numpy(rays[0]).to(cuda), rays_d=torch.from_numpy(rays[1]).to(cuda), **kw)
    else:
        out = R.render_fwd(vid, planes, hw, bft, blob, poses=torch.from_numpy(cams[0]).to(cuda), intrinsics=torch.from_numpy(cams[1]).to(cuda),
                           img_hw=cams[2], **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}


def _check(variant, out, b, r32, r64, bg_color=1.0):
    """scene b of a render against its oracle runs"""
    counts_ref = _counts(r32)
    counts, tr = out['num_samples'][b], out['trace'][b]
    if variant == 'P':
        assert np.array_equal(counts, counts_ref), f'scene {b}: {(counts != counts_ref).sum()} rays with a different sample count'
    else:
        # fp16 MLP: where a ray stops (T < T_thresh) may move by one sample on a handful of rays (see tests/test_render_gpu.py)
        differ = np.nonzero(counts != counts_ref)[0]
        assert len(differ) <= max(2, int(2e-3 * len(counts))), (b, len(differ))
        assert np.abs(counts - counts_ref).max() <= 1
    for i in range(len(counts)):
        n = min(counts[i], counts_ref[i])
        assert list(tr[i, :n]) == r32['trace'][i][:n], f'scene {b} ray {i}'
    ref, tol = (r64, TOL_P) if variant == 'P' else (r32, TOL_S)
    np.testing.assert_allclose(out['image'][b], ref['image'], **tol)
    np.testing.assert_allclose(out['weights_sum'][b], ref['weights_sum'], **tol)
    np.testing.assert_allclose(out['depth'][b], ref['depth'], rtol=tol['rtol'], atol=tol['atol'] * 4)
    np.testing.assert_allclose(out['rgb'][b], ref['image'] + bg_color * (1 - ref['weights_sum'][:, None]), **tol)


# ============================================================================================ 1. per-scene dt_gamma
DT_GAMMA = [0.0, 0.0076, 0.03]      # off; the shipped dt_gamma_scale 0.5 at the 64x64 focal length (0.5 * 2 / (2 * 65.625)); most steps at dt_max
DTG_GRIDS = ['sphere0.45', 'sphere', 'random3']


@functools.lru_cache(maxsize=None)
def _dtg_case(variant):
    params = rp.make_decoder_params(variant, 0)
    code = torch.cat([_code(variant, 10 + b) for b in range(3)])
    bfs = [_bitfield(g) for g in DTG_GRIDS]
    ro, rd = _cam_rays()
    refs = [_oracle(variant, params, ro, rd, code[b], bfs[b], max_steps=256, dt_gamma=DT_GAMMA[b]) for b in range(3)]
    return params, code, bfs, (ro, rd), refs


def test_dt_gamma_changes_the_traces():
    """precondition: each non-zero dt_gamma moves the samples of at least 10 % of its scene's rays"""
    params, code, bfs, (ro, rd), refs = _dtg_case('P')
    for b in (1, 2):
        r0 = rp.render_eval_scene(params, ro, rd, code[b], bfs[b], max_steps=256, return_trace=True)
        moved = np.mean([a != c for a, c in zip(refs[b][0]['trace'], r0['trace'])])
        assert moved >= 0.1, (DT_GAMMA[b], moved)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['P', 'S'])
def test_per_scene_dt_gamma(cuda, variant):
    """B = 3 scenes with their own code, grid and dt_gamma in one launch; each scene matches its own oracle run"""
    params, code, bfs, (ro, rd), refs = _dtg_case(variant)
    cap = max(_counts(r32).max() for r32, _ in refs) + 1
    out = _render(cuda, variant, params, code, bfs, rays=(np.stack([ro] * 3), np.stack([rd] * 3)), max_steps=256,
                  dt_gamma=torch.tensor(DT_GAMMA), trace_cap=int(cap))
    for b in range(3):
        _check(variant, out, b, *refs[b])


# ============================================================================================ 2. camera mode
def _fma(a, b, c):
    """IEEE float32 fma(a, b, c).  The float64 product is exact, and rounding the float64 sum to float32 is correct unless that sum
    lies on a float32 rounding midpoint without being exact (double rounding): those elements are rounded from the exact rational."""
    a, b, c = np.broadcast_arrays(a, b, c)
    r = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
    f = r.astype(F32)
    g = np.nextafter(f, np.where(r > f, np.inf, -np.inf).astype(F32))
    mid = (f.astype(np.float64) + g.astype(np.float64)) / 2
    for i in zip(*np.nonzero((r != f) & (r == mid))):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        if exact != Fraction(float(mid[i])):
            f[i] = max(f[i], g[i]) if exact > Fraction(float(mid[i])) else min(f[i], g[i])
    return f


def host_make_ray(poses, intr, h, w):
    """csrc/render_common.cuh make_ray on the host, operation for operation in float32 -> rays_o, rays_d [B, V*h*w, 3]"""
    B, V = poses.shape[:2]
    py, px = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing='ij')
    K = intr[:, :, None, None, :]
    c2w = poses[:, :, None, None]
    dcx = ((px + F32(0.5)) - K[..., 2]) / K[..., 0]
    dcy = ((py + F32(0.5)) - K[..., 3]) / K[..., 1]
    wv = [_fma(dcx, c2w[..., i, 0], _fma(dcy, c2w[..., i, 1], c2w[..., i, 2])) for i in range(3)]
    nrm = np.maximum(np.sqrt(_fma(wv[2], wv[2], _fma(wv[1], wv[1], wv[0] * wv[0]))), F32(1e-12))
    rd = np.stack([v / nrm for v in wv], axis=-1)
    ro = np.broadcast_to(c2w[..., :3, 3], rd.shape)
    assert rd.dtype == F32 and ro.dtype == F32
    return np.ascontiguousarray(ro.reshape(B, -1, 3)), np.ascontiguousarray(rd.reshape(B, -1, 3))


def _cameras(h, w):
    """B = 2 scenes x V = 3 views: different spiral poses per scene, fx != fy, principal point off centre and different per view"""
    poses = spiral_poses(6).reshape(3, 2, 4, 4).transpose(1, 0, 2, 3).copy()
    f = 131.25 * w / 128
    intr = np.array([[[f * (1.1 + 0.03 * v), f * (0.93 - 0.02 * b), w / 2 + 1.5 - v - 0.25 * b, h / 2 - 2.25 + 0.75 * v]
                      for v in range(3)] for b in range(2)], F32)
    return poses, intr


CAM_SIZES = [(24, 32, True), (18, 30, False), (20, 36, False)]     # (h, w, takes the 8x4 patch-tile path)


@functools.lru_cache(maxsize=None)
def _cam_case(variant, h, w):
    params = rp.make_decoder_params(variant, 1)
    code = torch.cat([_code(variant, 20 + b) for b in range(2)])
    bfs = [_bitfield('sphere'), _bitfield('sphere0.8')]
    poses, intr = _cameras(h, w)
    ro, rd = host_make_ray(poses, intr, h, w)
    refs = [_oracle(variant, params, ro[b], rd[b], code[b], bfs[b], max_steps=256) for b in range(2)]
    return params, code, bfs, poses, intr, (ro, rd), refs


def test_host_rays_match_the_oracle_rays():
    """the host restatement of make_ray agrees with the oracle's get_cam_rays (nerf_utils.py) to float32 round-off"""
    poses, intr = _cameras(20, 36)
    ro, rd = host_make_ray(poses, intr, 20, 36)
    ro_ref, rd_ref = rp.get_cam_rays(torch.from_numpy(poses), torch.from_numpy(intr), 20, 36)
    np.testing.assert_array_equal(ro, ro_ref.reshape(2, -1, 3).numpy())
    np.testing.assert_allclose(rd, rd_ref.reshape(2, -1, 3).numpy(), rtol=0, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['P', 'S'])
@pytest.mark.parametrize('h,w,patch', CAM_SIZES)
def test_camera_mode_bitwise(cuda, variant, h, w, patch):
    """camera mode (rays made in the kernel, 8x4 patch tiles or flat tiles) == explicit mode with the host's rays, every output bit for
    bit: each ray's arithmetic is per lane and each MMA output row depends only on its own A row, so which rays share a warp cannot
    matter.  The host rays also reproduce the oracle's trace; bg_color 0.25 blends as image + bg (1 - weights_sum)."""
    assert ((w % 8 == 0) and (h % 4 == 0)) == patch          # render.cu: patch tiles only when the image splits into 8x4 patches
    params, code, bfs, poses, intr, rays, refs = _cam_case(variant, h, w)
    cap = int(max(_counts(r32).max() for r32, _ in refs) + 1)
    kw = dict(max_steps=256, trace_cap=cap, bg_color=0.25)
    cam = _render(cuda, variant, params, code, bfs, cams=(poses, intr, (h, w)), **kw)
    exp = _render(cuda, variant, params, code, bfs, rays=rays, **kw)
    for k in ('image', 'rgb', 'depth', 'weights_sum', 'num_samples', 'trace'):
        assert cam[k].shape == exp[k].shape and np.array_equal(cam[k].view(np.uint32), exp[k].view(np.uint32)), k
    blend = cam['image'] + F32(0.25) * (F32(1) - cam['weights_sum'][..., None])
    assert np.array_equal(cam['rgb'], blend)
    for b in range(2):
        _check(variant, cam, b, *refs[b], bg_color=0.25)


# ============================================================================================ 3. per-scene budgets of the fix-up pass
@functools.lru_cache(maxsize=None)
def _budget_case(variant, binding_scene):
    """max_steps 32, a thin medium (density bias -6) so transmittance never ends a ray: the all-ones grid makes the emulated budget
    of the reference's host loop bind, the radius-0.6 sphere leaves it slack"""
    params = rp.make_decoder_params(variant, 3)
    params['density_net.0.bias'] = params['density_net.0.bias'] - 6.0
    code = torch.cat([_code(variant, 3 + b) for b in range(2)])
    grids = ['sphere', 'sphere']
    grids[binding_scene] = 'ones'
    bfs = [_bitfield(g) for g in grids]
    ro, rd = _cam_rays()
    refs = [_oracle(variant, params, ro, rd, code[b], bfs[b], max_steps=32) for b in range(2)]
    return params, code, bfs, (ro, rd), refs


@pytest.mark.parametrize('variant', ['P', 'S'])
def test_budget_binds_in_one_scene_only(variant):
    """precondition: the oracle's sample budget truncates rays in the all-ones scene and in no other"""
    for binding in (0, 1):
        *_, refs = _budget_case(variant, binding)
        for b, (r32, _) in enumerate(refs):
            c = _counts(r32)
            if b == binding:
                assert c.max() == r32['total_budget'] > 32, (c.max(), r32['total_budget'])
            else:
                assert c.max() < r32['total_budget'], (c.max(), r32['total_budget'])


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['P', 'S'])
@pytest.mark.parametrize('binding_scene', [0, 1])
def test_per_scene_budget(cuda, variant, binding_scene):
    """B = 2: the fix-up pass truncates each scene at its own emulated budget (both scene orders, so a budget read from the wrong
    scene shows either way)"""
    params, code, bfs, rays, refs = _budget_case(variant, binding_scene)
    cap = int(max(_counts(r32).max() for r32, _ in refs) + 1)
    out = _render(cuda, variant, params, code, bfs, rays=tuple(np.stack([a] * 2) for a in rays), max_steps=32, trace_cap=cap)
    for b in range(2):
        _check(variant, out, b, *refs[b])


# ============================================================================================ 4. non-square planes
PLANE_HW = [(96, 160), (97, 131)]


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['P', 'S'])
@pytest.mark.parametrize('plane_hw', PLANE_HW)
def test_non_square_planes(cuda, variant, plane_hw):
    """pack_planes + render_fwd with plane_h != plane_w (odd sizes too), B = 2, against grid_sample on the same code"""
    params = rp.make_decoder_params(variant, 2)
    code = torch.cat([_code(variant, 30 + b, plane_hw) for b in range(2)])
    bfs = [_bitfield('sphere'), _bitfield('sphere0.8')]
    ro, rd = _cam_rays(48)
    refs = [_oracle(variant, params, ro, rd, code[b], bfs[b], max_steps=256) for b in range(2)]
    cap = int(max(_counts(r32).max() for r32, _ in refs) + 1)
    out = _render(cuda, variant, params, code, bfs, rays=(np.stack([ro] * 2), np.stack([rd] * 2)), max_steps=256, trace_cap=cap)
    for b in range(2):
        _check(variant, out, b, *refs[b])


@pytest.mark.gpu
def test_get_density_non_square_planes(cuda):
    """occupancy-grid builder on 96 x 160 planes (assertions of test_density_gpu.test_get_density_matches_oracle)"""
    from ssdnerf_b200 import renderer as R, density as D
    g = torch.Generator().manual_seed(23)
    B = 2
    code = torch.randn(B, 3, 6, 96, 160, generator=g).clamp(-2, 2)
    params = rp.make_decoder_params('P', 4)
    params['density_net.0.bias'] = params['density_net.0.bias'] - 2.5
    rands = [torch.rand(64 ** 3, 3, generator=g) for _ in range(3)]
    grid_ref, bf_ref = rp.get_density(params, code, rands, density_thresh=0.1)
    blob = R.pack_decoder_blob(params, R.DEC_P, device=cuda)
    planes = R.pack_planes(code.to(cuda), R.DEC_P)
    grid, bf = D.get_density(R.DEC_P, planes, (96, 160), blob, B, density_thresh=0.1, density_step=3, jitters=[r.to(cuda) for r in rands])
    np.testing.assert_allclose(grid.float().cpu().numpy(), grid_ref.float().numpy(), rtol=2e-3, atol=1e-6)
    diff = np.unpackbits(bf.cpu().numpy() ^ bf_ref, axis=-1).sum()
    assert diff <= 1e-4 * B * 64 ** 3, diff
    assert 0.02 < np.unpackbits(bf_ref).mean() < 0.98


# ============================================================================================ 5. large pre-activations (variant P)
def big_preact_params():
    """A shipped-shape decoder whose pre-activations span the whole range the P kernel's SiLU-in-fours has to handle.

    base_net and dir_net are scaled x50 (pre-activations of about +-100).  Three columns are set by hand:
      * column 0: base -120, colour -320 whatever the sample (both far below the exponent clamp at -20.8);
      * column 1: base in about [-9, -6], colour about -250: with column 0 that is a quad of SiLU inputs whose four denominators
        1 + e^-x multiply to more than 2^128 unless the exponents are clamped near 30 -- the kernel must still return column 1's
        small negative SiLU, which its density weight (20) makes visible;
      * column 2: density weight 2, so that the density logit exceeds 89 (exp overflows float32, alpha must be 1) where its base is
        large.
    The other density weights are scaled x0.1 and the colour head x0.025, which keeps the density and colour logits O(1) to O(100)
    sums that float32 arithmetic resolves to within the float bars (with the colour head unscaled, float32 round-off of the +-100
    pre-activations alone moves the composited colour by more than 2e-4)."""
    p = rp.make_decoder_params('P', 5)
    for k in ('base_net.0.weight', 'base_net.0.bias', 'dir_net.0.weight', 'dir_net.0.bias'):
        p[k] = p[k] * 50.0
    p['color_net.0.weight'] = p['color_net.0.weight'] * 0.025
    p['density_net.0.weight'] = p['density_net.0.weight'] * 0.1
    p['base_net.0.weight'][0] = 0.0
    p['base_net.0.bias'][0] = -120.0
    p['base_net.0.weight'][1] = p['base_net.0.weight'][1] * (0.75 / 50.0)
    p['base_net.0.bias'][1] = -7.5
    p['dir_net.0.weight'][:2] = 0.0
    p['dir_net.0.bias'][:2] = torch.tensor([-200.0, -243.0])
    p['density_net.0.weight'][0, 1] = 20.0
    p['density_net.0.weight'][0, 2] = 2.0
    return p


def random_rays(n, seed):
    """rays from random points 2.6 from the origin towards random points of the inner box: every lane of a tile has its own direction"""
    rng = np.random.default_rng(seed)
    o = rng.normal(size=(n, 3))
    o = o / np.linalg.norm(o, axis=1, keepdims=True) * 2.6
    d = rng.uniform(-0.6, 0.6, size=(n, 3)) - o
    return o.astype(F32), (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)


@functools.lru_cache(maxsize=None)
def _big_case():
    params = big_preact_params()
    code = _code('P', 5)
    bf = _bitfield('sphere')
    ro, rd = random_rays(2048, 1)
    r32 = rp.render_eval_scene(params, ro, rd, code[0], bf, max_steps=256, return_samples=True)
    r64 = rp.render_eval_scene(params, ro, rd, code[0], bf, max_steps=256, dtype=torch.float64)
    return params, code, bf, (ro, rd), (r32, r64)


def test_large_preactivations_reach_the_clamp():
    """precondition: at the samples the oracle composites, base and colour pre-activations span at least [-100, 100], >= 1 % lie below
    the kernel's exponent clamp (-20.8) and some below -89; some density logits exceed 89"""
    params, code, _, _, (r32, _) = _big_case()
    xs, ds = r32['samples']
    base, colour, logit = (a.numpy() for a in rp.point_preacts(params, torch.from_numpy(xs), torch.from_numpy(ds), code[0], dtype=torch.float64))
    for a in (base, colour):
        assert a.min() <= -100 and a.max() >= 100, (a.min(), a.max())
        assert (a < -20.8).mean() >= 0.01 and (a < -89).any()
    assert (logit > 89).any(), logit.max()
    assert ((base[:, 1] > -9.5) & (base[:, 1] < -5.6)).mean() > 0.99


@pytest.mark.gpu
def test_large_preactivations(cuda):
    """no NaN / Inf anywhere, trace and counts bit-exact, floats within TOL_P of the float64-MLP oracle"""
    params, code, bf, (ro, rd), (r32, r64) = _big_case()
    cap = int(_counts(r32).max() + 1)
    out = _render(cuda, 'P', params, code, [bf], rays=(ro[None], rd[None]), max_steps=256, trace_cap=cap)
    for k in ('image', 'rgb', 'depth', 'weights_sum'):
        assert np.isfinite(out[k]).all(), k
    _check('P', out, 0, r32, r64)
