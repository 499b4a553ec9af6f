"""Marching cubes on the device (csrc/mesh.cu) against the CPU oracle (oracle/mesh_port.py): identical triangle arrays and bit-identical
vertex arrays on every case, and the mesh paths of the model (`extract_geometry`, `save_mesh`, `val_step` with save_mesh=True)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import mesh_port as mp
from oracle import render_port as rp
from tests.common import GOLDEN

pytestmark = pytest.mark.gpu


def _run(u_np, thr, cuda):
    from ssdnerf_b200 import mesh
    v, t = mesh.marching_cubes(torch.from_numpy(np.ascontiguousarray(u_np, np.float32)).to(cuda), thr)
    assert v.dtype == torch.float64 and t.dtype == torch.int64 and v.is_cuda and t.is_cuda
    return v.cpu().numpy(), t.cpu().numpy()


def _assert_same(u_np, thr, cuda):
    v, t = _run(u_np, thr, cuda)
    ov, ot = mp.marching_cubes(u_np, thr)
    assert v.shape == ov.shape and t.shape == ot.shape, (v.shape, ov.shape, t.shape, ot.shape)
    assert np.array_equal(t, ot)
    assert np.array_equal(v.view(np.uint64), ov.view(np.uint64))            # bit-identical
    return v, t


def _smooth(shape, seed):
    g = np.random.default_rng(seed)
    x, y, z = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing='ij')
    u = np.zeros(shape)
    for _ in range(6):
        k = g.normal(0, 0.35, 3)
        u += np.cos(k[0] * x + k[1] * y + k[2] * z + g.uniform(0, 2 * np.pi))
    return u.astype(np.float32)


def test_all_single_cube_cases(cuda):
    g = np.random.default_rng(0)
    for case in range(256):
        low = np.array([(case >> i) & 1 for i in range(8)], bool)
        vals = np.where(low, g.uniform(-1.0, 0.25, 8), g.uniform(0.3, 2.0, 8)).astype(np.float32)
        u = np.zeros((2, 2, 2), np.float32)
        for i in range(8):
            u[i & 1, (i >> 1) & 1, (i >> 2) & 1] = vals[i]
        v, t = _assert_same(u, 0.25, cuda)
        assert len(t) == mp.case_table()[0][case]


@pytest.mark.parametrize('shape', [(32, 32, 32), (17, 40, 9), (2, 3, 257)])
def test_smooth_fields(cuda, shape):
    u = _smooth(shape, sum(shape))
    v, t = _assert_same(u, 0.3, cuda)
    assert len(t) > 0


def test_ties_at_lattice_values(cuda):
    g = np.random.default_rng(3)
    u = g.integers(0, 4, (19, 23, 21)).astype(np.float32)
    for thr in (0.0, 1.0, 2.0, 3.0):
        _assert_same(u, thr, cuda)


def test_empty_meshes(cuda):
    for u, thr in [(np.zeros((8, 9, 10), np.float32), 0.5), (np.full((8, 9, 10), 3, np.float32), 0.5),
                   (np.zeros((8, 9, 10), np.float32), 0.0), (_smooth((1, 20, 20), 1), 0.0), (_smooth((20, 1, 20), 2), 0.0),
                   (_smooth((20, 20, 1), 3), 0.0), (np.zeros((0, 4, 4), np.float32), 0.0)]:
        v, t = _run(u, thr, cuda)
        assert v.shape == (0, 3) and t.shape == (0, 3)


def _decoder(cuda):
    import ssdnerf_b200 as S
    params = rp.make_decoder_params('P', 7)
    dec = S.build_module(dict(type='TriPlaneDecoder', base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3], use_dir_enc=True,
                              dir_layers=[16, 64], max_steps=256))
    sd = dec.state_dict(); sd.update(params); dec.load_state_dict(sd)
    return dec.to(cuda).eval()


def _code(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(3, 6, 128, 128, generator=g) * 0.7).clamp(-2, 2)


def test_extract_fields_lattice_256_and_determinism(cuda):
    from ssdnerf_b200 import mesh
    from ssdnerf_b200.nerf import extract_fields
    dec = _decoder(cuda)
    with torch.no_grad():
        u = extract_fields(dec, _code(9).to(cuda), resolution=256)
    un = u.cpu().numpy()
    thr = float(np.quantile(un[un > 0], 0.6))
    v, t = _assert_same(un, thr, cuda)
    assert len(t) > 10000
    v2, t2 = mesh.marching_cubes(u, thr)
    assert v2.cpu().numpy().tobytes() == v.tobytes() and t2.cpu().numpy().tobytes() == t.tobytes()


def test_extract_geometry_world_mapping(cuda):
    from ssdnerf_b200.nerf import extract_fields, extract_geometry
    dec = _decoder(cuda)
    code = _code(4).to(cuda)
    R = 96
    with torch.no_grad():
        un = extract_fields(dec, code, resolution=R).cpu().numpy()
    thr = float(np.quantile(un[un > 0], 0.6))
    verts, tris = extract_geometry(dec, code, resolution=R, threshold=thr)
    assert isinstance(verts, np.ndarray) and verts.dtype == np.float64 and tris.dtype == np.int64
    ov, ot = mp.marching_cubes(un, thr)
    lo, hi = (dec.aabb[:3] - 0.1).cpu().numpy(), (dec.aabb[3:] + 0.1).cpu().numpy()
    assert len(ot) > 0 and np.array_equal(tris, ot)
    assert np.array_equal(verts, mp.to_world(ov, R, lo, hi))


def _stl_matches_oracle(path, un, thr, R, lo, hi):
    header, normals, v, attr = mp.read_stl(path)
    assert not header.startswith(b'solid') and (attr == 0).all()
    ov, ot = mp.marching_cubes(un, thr)
    assert len(ot) > 0
    np.testing.assert_array_equal(v, mp.to_world(ov, R, lo, hi)[ot].astype(np.float32))


def test_save_mesh_and_val_step_write_stl(cuda, tmp_path):
    import ssdnerf_b200 as S
    from ssdnerf_b200.nerf import extract_fields
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_recons1v.py']
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg']).to(cuda).eval()
    decoder = model._modules_for_eval()[1]
    B, R = 2, 64
    g = torch.Generator().manual_seed(1)
    code = (torch.randn(B, 3, 6, 128, 128, generator=g) * 0.5).to(cuda)
    with torch.no_grad():
        fields = [extract_fields(decoder, code[i], resolution=R).cpu().numpy() for i in range(B)]
    thr = float(np.quantile(np.concatenate([f[f > 0] for f in fields]), 0.6))
    lo, hi = (decoder.aabb[:3] - 0.1).cpu().numpy(), (decoder.aabb[3:] + 0.1).cpu().numpy()
    # save_mesh on its own
    model.save_mesh(str(tmp_path / 'direct'), decoder, code, ['s0', 's1'], R, thr)
    for i in range(B):
        _stl_matches_oracle(str(tmp_path / 'direct' / f's{i}.stl'), fields[i], thr, R, lo, hi)
    # val_step with stored scenes and save_mesh in test_cfg (diffusion_nerf.py:455-461)
    stored = [dict(param=dict(code=code[i].cpu(), density_grid=torch.zeros(64 ** 3).half(),
                              density_bitfield=torch.zeros(64 ** 3 // 8, dtype=torch.uint8))) for i in range(B)]
    out_dir = tmp_path / 'val'
    model.test_cfg.update(save_dir=str(out_dir), save_mesh=True, mesh_resolution=R, mesh_threshold=thr)
    out = model.val_step(dict(scene_id=[0, 1], scene_name=['a', 'b'], code=stored))
    assert out['num_samples'] == B
    for i, name in enumerate(['a', 'b']):
        assert (out_dir / f'{name}.pth').is_file()
        _stl_matches_oracle(str(out_dir / f'{name}.stl'), fields[i], thr, R, lo, hi)


def test_bad_arguments_raise(cuda):
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import mesh
    L = N.lib()
    u = torch.rand(8, 8, 8, device=cuda)
    work = torch.empty(L.ssdnerf_mc_workspace_bytes(8, 8, 8), dtype=torch.uint8, device=cuda)
    counts = torch.empty(2, dtype=torch.int64, device=cuda)
    with pytest.raises(N.SSDNeRFNativeError, match='2\\^32'):
        N.check(L.ssdnerf_mc_count(N.ptr(u), 1 << 11, 1 << 11, 1 << 9, 0.5, N.ptr(work), N.ptr(counts), N.stream_ptr()))
    with pytest.raises(N.SSDNeRFNativeError, match='NULL'):
        N.check(L.ssdnerf_mc_count(N.ptr(u), 8, 8, 8, 0.5, None, N.ptr(counts), N.stream_ptr()))
    with pytest.raises(N.SSDNeRFNativeError):
        N.check(L.ssdnerf_mc_emit(N.ptr(u), 8, 8, 8, 0.5, N.ptr(work), None, None, N.stream_ptr()))
    with pytest.raises(N.SSDNeRFNativeError, match='aligned'):
        N.check(L.ssdnerf_mc_count(ctypes.c_void_p(u.data_ptr() + 2), 8, 8, 8, 0.5, N.ptr(work), N.ptr(counts), N.stream_ptr()))
    with pytest.raises(ValueError):
        mesh.marching_cubes(u.double(), 0.5)
    with pytest.raises(N.SSDNeRFNativeError):
        mesh.marching_cubes(u.cpu(), 0.5)
    # the library still works after the refusals
    v, t = mesh.marching_cubes(u, 0.5)
    ov, ot = mp.marching_cubes(u.cpu().numpy(), 0.5)
    assert np.array_equal(t.cpu().numpy(), ot) and np.array_equal(v.cpu().numpy(), ov)
