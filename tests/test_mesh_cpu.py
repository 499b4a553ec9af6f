"""Marching cubes without a GPU: the generated case table (the library's host copy and the oracle's), the oracle's meshes on smooth
fields (closed, consistently oriented, outward normals), ambiguous faces shared by two cubes, the binary STL writer, and argument checks
that fail before any device work."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mesh_port as mp


def _gaussians(shape, k, seed):
    """sum of k Gaussians with centres well inside the lattice: below 0.05 on the border, so the threshold 0.5 surface is closed"""
    g = np.random.default_rng(seed)
    n = np.array(shape, np.float64)
    centres = g.uniform(0.35, 0.65, (k, 3)) * (n - 1)
    sigma = g.uniform(0.07, 0.11, k) * n.min()
    amp = g.uniform(1.0, 2.0, k)
    pts = np.stack(np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing='ij'), axis=-1)
    u = sum(a * np.exp(-((pts - c) ** 2).sum(-1) / (2 * s * s)) for c, s, a in zip(centres, sigma, amp))
    border = np.concatenate([u[[0, -1]].ravel(), u[:, [0, -1]].ravel(), u[:, :, [0, -1]].ravel()])
    assert border.max() < 0.05
    return u.astype(np.float32), (centres, sigma, amp)


def _grad(p, params):
    centres, sigma, amp = params
    g = np.zeros_like(p)
    for c, s, a in zip(centres, sigma, amp):
        d = p - c
        g += (a * np.exp(-(d ** 2).sum(-1) / (2 * s * s)))[:, None] * (-d / (s * s))
    return g


def _directed(tris):
    return np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])


def _edge_counts(tris):
    d = _directed(tris)
    und, n_und = np.unique(np.sort(d, axis=1), axis=0, return_counts=True)
    dirs, n_dir = np.unique(d, axis=0, return_counts=True)
    return und, n_und, dirs, n_dir


def _assert_closed_oriented(tris):
    und, n_und, dirs, n_dir = _edge_counts(tris)
    assert (n_und == 2).all(), np.bincount(n_und)
    assert (n_dir == 1).all()
    return und


def _assert_balanced(tris):
    """watertight and consistently oriented even where an edge is shared by more than two triangles: every directed edge is used as
    often as its reverse"""
    d = _directed(tris)
    key = lambda e: e[:, 0] * (int(tris.max()) + 1) + e[:, 1]
    fwd = np.unique(key(d), return_counts=True)
    rev = np.unique(key(d[:, ::-1]), return_counts=True)
    assert np.array_equal(fwd[0], rev[0]) and np.array_equal(fwd[1], rev[1])


# ------------------------------------------------------------------------------------------------------------------ case table
def test_library_table_equals_oracle_table():
    from ssdnerf_b200 import mesh
    count, tri = mesh.case_table()
    ocount, otri = mp.case_table()
    assert np.array_equal(count, ocount) and np.array_equal(tri, otri)


def _face_ambiguous(case):
    low = [(case >> i) & 1 for i in range(8)]
    for a in range(3):
        for s in (0, 1):
            c = [i for i in range(8) if (i >> a) & 1 == s]        # face corners in bit order: diagonals are (c0, c3) and (c1, c2)
            if low[c[0]] == low[c[3]] and low[c[1]] == low[c[2]] and low[c[0]] != low[c[1]]:
                return True
    return False


def test_case_table_loops_closed_and_complete():
    count, tri = mp.case_table()
    assert count.max() <= mp.MAX_TRIS
    assert count[0] == 0 and count[255] == 0
    for case in range(256):
        crossed = {e for e in range(12) if ((case >> mp.edge_corners(e)[0]) & 1) != ((case >> mp.edge_corners(e)[1]) & 1)}
        t = tri[case, :count[case]]
        assert set(t.ravel().tolist()) == crossed, case
        # boundary of the cube's triangles: directed edges whose reverse is not there (fan diagonals come in both directions)
        d = {tuple(e) for e in _directed(t).tolist()}
        bnd = [e for e in d if (e[1], e[0]) not in d]
        outs = sorted(p for p, _ in bnd)
        ins = sorted(q for _, q in bnd)
        assert outs == sorted(crossed) and ins == sorted(crossed), case          # closed loops through every crossed edge
        for p, q in bnd:                                                          # every loop segment lies on one cube face
            cp, cq = set(mp.edge_corners(p)), set(mp.edge_corners(q))
            assert any(all(((c >> a) & 1) == s for c in cp | cq) for a in range(3) for s in (0, 1)), (case, p, q)
        assert count[case] == len(crossed) - 2 * len(mp.case_loops(case))


def test_complement_reverses_winding_without_ambiguous_faces():
    count, tri = mp.case_table()
    canon = lambda t: {tuple(np.roll(x, -int(np.argmin(x))).tolist()) for x in t}
    n = 0
    for case in range(256):
        if _face_ambiguous(case):
            continue
        n += 1
        a = canon(tri[case, :count[case]])
        b = canon(tri[255 - case, :count[255 - case]][:, ::-1])
        assert a == b, case
    assert n > 100


def test_single_low_corner_normal_points_at_it():
    v = np.ones((2, 2, 2), np.float32)
    v[0, 0, 0] = 0.0
    verts, tris = mp.marching_cubes(v, 0.5)
    assert len(verts) == 3 and len(tris) == 1
    a, b, c = verts[tris[0]]
    n = np.cross(b - a, c - a)
    assert (n < 0).all()
    np.testing.assert_array_equal(np.sort(verts.sum(1)), [0.5, 0.5, 0.5])


# ------------------------------------------------------------------------------------------------------------------ oracle meshes
@pytest.mark.parametrize('shape,k,seed', [((24, 24, 24), 1, 0), ((17, 20, 23), 1, 1), ((24, 24, 24), 3, 2), ((17, 20, 23), 4, 3),
                                          ((32, 32, 32), 5, 4)])
def test_oracle_mesh_on_smooth_fields(shape, k, seed):
    u, params = _gaussians(shape, k, seed)
    verts, tris = mp.marching_cubes(u, 0.5)
    assert len(tris) > 50
    assert np.unique(tris).size == len(verts)                 # every vertex is used
    und = _assert_closed_oriented(tris)
    if k == 1:
        assert len(verts) - len(und) + len(tris) == 2           # a sphere
    p0, p1, p2 = (verts[tris[:, i]] for i in range(3))
    volume = np.einsum('ij,ij->i', p0, np.cross(p1, p2)).sum() / 6
    assert volume > 0
    # volume of {u > 0.5} counted on the lattice, within the surface's sub-cell accuracy
    assert abs(volume - (u > 0.5).sum()) < 0.1 * (u > 0.5).sum()
    n = np.cross(p1 - p0, p2 - p0)
    area = np.linalg.norm(n, axis=1)
    ok = area > 1e-9
    cos = np.einsum('ij,ij->i', n[ok] / area[ok, None], -_grad((p0 + p1 + p2)[ok] / 3, params))
    assert (cos > 0).mean() > 0.999, (cos <= 0).sum()


def test_oracle_sphere_radii():
    n, c, r0 = 40, np.array([19.3, 20.1, 18.7]), 12.0
    pts = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing='ij'), axis=-1)
    u = (r0 - np.linalg.norm(pts - c, axis=-1)).astype(np.float32)
    verts, tris = mp.marching_cubes(u, 0.0)
    r = np.linalg.norm(verts - c, axis=1)
    assert np.abs(r - r0).max() < 0.05, np.abs(r - r0).max()
    und = _assert_closed_oriented(tris)
    assert len(verts) - len(und) + len(tris) == 2


@pytest.mark.parametrize('flip', [False, True])
def test_adjacent_ambiguous_cubes_close_up(flip):
    """two cubes sharing a face whose diagonal corners are alike: both pair its crossed edges around the low corners"""
    u = np.zeros((5, 4, 4), np.float32)                       # low border
    u[1:4, 1:3, 1:3] = 1.0                                    # dense 3 x 2 x 2 block: cubes [1, 2] and [2, 3] along x
    lo = [(1, 2), (2, 1)] if not flip else [(1, 1), (2, 2)]
    for y, z in lo:
        u[2, y, z] = 0.0                                      # face x = 2: low corners on one diagonal, dense on the other
    low = u <= 0.5
    assert low[2, 1, 1] == low[2, 2, 2] and low[2, 1, 2] == low[2, 2, 1] and low[2, 1, 1] != low[2, 1, 2]
    verts, tris = mp.marching_cubes(u, 0.5)
    _assert_closed_oriented(tris)
    # the same mesh for the shifted / mirrored copy: ambiguous faces do not depend on which cube sees them first
    verts2, tris2 = mp.marching_cubes(u[::-1].copy(), 0.5)
    _assert_closed_oriented(tris2)
    assert len(tris2) == len(tris) and len(verts2) == len(verts)


@pytest.mark.parametrize('seed', range(4))
def test_random_binary_fields_are_watertight(seed):
    """every ambiguous configuration at once: random 0 / 1 interiors with a low border"""
    g = np.random.default_rng(seed)
    u = np.zeros((9, 8, 7), np.float32)
    u[1:-1, 1:-1, 1:-1] = g.integers(0, 2, (7, 6, 5))
    verts, tris = mp.marching_cubes(u, 0.5)
    assert len(tris) > 0
    _assert_balanced(tris)


def test_oracle_ties_and_empty():
    g = np.random.default_rng(5)
    u = g.integers(0, 4, (6, 7, 8)).astype(np.float32)
    verts, tris = mp.marching_cubes(u, 2.0)                   # u == threshold is low
    low = u <= 2.0
    assert len(verts) == sum((np.diff(low, axis=a) != 0).sum() for a in range(3))
    for shape in [(1, 5, 5), (5, 0, 5)]:
        v, t = mp.marching_cubes(np.zeros(shape, np.float32), 0.5)
        assert v.shape == (0, 3) and t.shape == (0, 3)
    v, t = mp.marching_cubes(np.full((4, 4, 4), 7, np.float32), 0.5)
    assert len(v) == 0 and len(t) == 0


def test_pymcubes_vertices_agree():
    mcubes = pytest.importorskip('mcubes')
    u, _ = _gaussians((24, 24, 24), 3, 7)
    verts, _ = mp.marching_cubes(u, 0.5)
    ref, _ = mcubes.marching_cubes(u, 0.5)
    a = verts[np.lexsort(verts.T[::-1])]
    b = np.asarray(ref, np.float64)[np.lexsort(np.asarray(ref).T[::-1])]
    assert a.shape == b.shape
    np.testing.assert_allclose(a, b, rtol=0, atol=1e-9)


# ------------------------------------------------------------------------------------------------------------------ STL writer
def test_write_stl_round_trip(tmp_path):
    from ssdnerf_b200.mesh import write_stl
    u, _ = _gaussians((20, 20, 20), 2, 8)
    verts, tris = mp.marching_cubes(u, 0.5)
    verts = verts * 0.1 - 1.0
    tris = np.concatenate([tris, [[0, 0, 1]]])                # a zero-area face
    path = tmp_path / 'm.stl'
    write_stl(str(path), verts, tris)
    header, normals, v, attr = mp.read_stl(str(path))
    assert len(header) == 80 and not header.startswith(b'solid')
    assert path.stat().st_size == 84 + 50 * len(tris)
    np.testing.assert_array_equal(v, verts[tris].astype(np.float32))
    assert (attr == 0).all()
    norm = np.linalg.norm(normals.astype(np.float64), axis=1)
    np.testing.assert_allclose(norm[:-1], 1.0, atol=1e-6)
    assert norm[-1] == 0
    ref = np.cross(verts[tris[:-1, 1]] - verts[tris[:-1, 0]], verts[tris[:-1, 2]] - verts[tris[:-1, 0]])
    ref /= np.linalg.norm(ref, axis=1, keepdims=True)
    np.testing.assert_allclose(normals[:-1], ref, atol=1e-6)
    # tensors are accepted as they are, and an empty mesh is a valid file
    write_stl(str(tmp_path / 't.stl'), torch.from_numpy(verts), torch.from_numpy(tris))
    assert (tmp_path / 't.stl').read_bytes() == path.read_bytes()
    write_stl(str(tmp_path / 'e.stl'), np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    assert mp.read_stl(str(tmp_path / 'e.stl'))[2].shape == (0, 3, 3)


# ------------------------------------------------------------------------------------------------------------------ arguments
def test_mc_arguments_rejected_before_device_work():
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    fake = ctypes.c_void_p(1 << 20)                           # never dereferenced: validation fails first
    assert L.ssdnerf_mc_workspace_bytes(256, 256, 256) <= 4 * 256 ** 3
    assert L.ssdnerf_mc_workspace_bytes(1, 256, 256) == 0
    assert L.ssdnerf_mc_workspace_bytes(1 << 11, 1 << 11, 1 << 9) == 0
    assert L.ssdnerf_mc_count(fake, 1 << 11, 1 << 11, 1 << 9, 0.5, fake, fake, None) == -2
    assert b'2^32' in L.ssdnerf_last_error()
    assert L.ssdnerf_mc_count(None, 8, 8, 8, 0.5, fake, fake, None) == -2
    assert b'NULL' in L.ssdnerf_last_error()
    assert L.ssdnerf_mc_count(fake, 8, 8, 8, 0.5, None, fake, None) == -2
    assert L.ssdnerf_mc_count(fake, 8, 8, 8, 0.5, fake, None, None) == -2
    assert L.ssdnerf_mc_count(ctypes.c_void_p((1 << 20) + 2), 8, 8, 8, 0.5, fake, fake, None) == -2
    assert b'aligned' in L.ssdnerf_last_error()
    assert L.ssdnerf_mc_emit(fake, 8, 8, 8, 0.5, fake, None, fake, None) == -2
    assert L.ssdnerf_mc_emit(fake, 1 << 11, 1 << 11, 1 << 9, 0.5, fake, fake, fake, None) == -2
    assert L.ssdnerf_mc_case_table(None, None) == -2


def test_marching_cubes_refuses_cpu_tensors():
    from ssdnerf_b200 import mesh
    from ssdnerf_b200._lib import SSDNeRFNativeError
    with pytest.raises(SSDNeRFNativeError):
        mesh.marching_cubes(torch.zeros(4, 4, 4), 0.5)
