"""CPU restatement of the package's marching cubes (TEST INFRASTRUCTURE): the contract of csrc/mesh.cu, which stands in for
PyMCubes' `marching_cubes(u, threshold)` in lib/core/utils/nerf_utils.py:84-112.

Definitions (the same ones the kernel and include/ssdnerf_b200.h state):
  * a lattice point is low when u <= threshold (float64 compare); a lattice edge is crossed when its ends differ and carries exactly
    one vertex, shared by all cubes around it;
  * on the edge from point a to a + e_axis, with f1 = u[a], f2 = u[a + e], the axis coordinate is (x2 - x1) * (thr - f1) / (f2 - f1) + x1
    in float64 in this operation order; the other two coordinates are the lattice point's (PyMCubes' linear interpolation);
  * vertices are ordered by edge id 3 * ((x * ny + y) * nz + z) + axis, triangles by the cube's lower-corner linear index, then by the
    case table's order;
  * the case table is generated from a rule (`case_loops`), not typed in: on each cube face the crossed edges are paired into segments
    (on an ambiguous face each segment cuts off one of the two low corners), segments are oriented so that every triangle normal
    (v1 - v0) x (v2 - v0) points to the low side, chained into loops, and each loop is fan-triangulated from its smallest cube-edge number.
Cube corner i sits at (i & 1, (i >> 1) & 1, (i >> 2) & 1) in (x, y, z); cube edge 4 a + k runs along axis a from the corner whose other
two axes b < c take the bits k & 1 and k >> 1.  Everything is vectorised over cubes, so it runs at 256^3."""
import struct

import numpy as np

MAX_TRIS = 10
OTHER_AXES = ((1, 2), (0, 2), (0, 1))


def edge_corners(e):
    a, k = divmod(e, 4)
    b, c = OTHER_AXES[a]
    base = ((k & 1) << b) | ((k >> 1) << c)
    return base, base | (1 << a)


def corner_pos(i):
    return np.array([i & 1, (i >> 1) & 1, (i >> 2) & 1], np.float64)


def edge_mid(e):
    c0, c1 = edge_corners(e)
    return (corner_pos(c0) + corner_pos(c1)) / 2


def face_segments(case):
    """oriented segments (p, q) between crossed cube edges on the six faces: next[p] = q.  Each segment is directed along
    L x n_face, L pointing to the face's low side, so the loop runs counter-clockwise seen from the low side"""
    low = [(case >> i) & 1 for i in range(8)]
    nxt = {}
    for a in range(3):
        for s in (0, 1):
            n = np.zeros(3)
            n[a] = 1.0 if s else -1.0
            corners = [c for c in range(8) if (c >> a) & 1 == s]
            crossed = [e for e in range(12) if e // 4 != a and (edge_corners(e)[0] >> a) & 1 == s
                       and low[edge_corners(e)[0]] != low[edge_corners(e)[1]]]
            segs = []
            if len(crossed) == 2:
                lo = np.mean([corner_pos(c) for c in corners if low[c]], axis=0)
                hi = np.mean([corner_pos(c) for c in corners if not low[c]], axis=0)
                segs.append((crossed[0], crossed[1], lo - hi))
            elif len(crossed) == 4:                    # ambiguous: one segment around each low corner, the dense corners stay connected
                centre = np.mean([corner_pos(c) for c in corners], axis=0)
                for c in corners:
                    if low[c]:
                        p, q = [e for e in crossed if c in edge_corners(e)]
                        segs.append((p, q, corner_pos(c) - centre))
            else:
                assert not crossed
            for p, q, L in segs:
                dot = float(np.dot(edge_mid(q) - edge_mid(p), np.cross(L, n)))
                assert dot != 0
                p, q = (p, q) if dot > 0 else (q, p)
                assert p not in nxt
                nxt[p] = q
    return nxt


def case_loops(case):
    """closed loops of cube-edge numbers, each starting at its smallest edge, in ascending order of that edge"""
    nxt = face_segments(case)
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop, f = [], e
        while f not in seen:
            seen.add(f)
            loop.append(f)
            f = nxt[f]
        assert f == e, 'open loop'
        loops.append(loop)
    return loops


def case_table():
    """triangle counts int64 [256] and cube-edge triples int64 [256, 10, 3] (zero past the count): the fan of every loop"""
    count = np.zeros(256, np.int64)
    tri = np.zeros((256, MAX_TRIS, 3), np.int64)
    for case in range(256):
        tris = [(loop[0], loop[i], loop[i + 1]) for loop in case_loops(case) for i in range(1, len(loop) - 1)]
        count[case] = len(tris)
        tri[case, :len(tris)] = np.array(tris, np.int64).reshape(-1, 3)
    return count, tri


_TABLE = None


def _table():
    global _TABLE
    if _TABLE is None:
        _TABLE = case_table()
    return _TABLE


def marching_cubes(u, threshold):
    """vertices float64 [V, 3] (lattice-index units) and triangles int64 [T, 3] of the float32 lattice u [nx, ny, nz]"""
    u = np.ascontiguousarray(u, np.float32)
    nx, ny, nz = u.shape
    if min(u.shape) < 2:
        return np.zeros((0, 3)), np.zeros((0, 3), np.int64)
    thr = float(threshold)
    ud = u.astype(np.float64).ravel()
    low = (ud <= thr).reshape(u.shape)
    lin = np.arange(u.size, dtype=np.int64).reshape(u.shape)
    strides = np.array([ny * nz, nz, 1], np.int64)
    ids = []
    for a in range(3):
        s0, s1 = [slice(None)] * 3, [slice(None)] * 3
        s0[a], s1[a] = slice(0, -1), slice(1, None)
        ids.append(3 * lin[tuple(s0)][low[tuple(s0)] != low[tuple(s1)]] + a)
    ids = np.sort(np.concatenate(ids))
    p, a = ids // 3, ids % 3
    xyz = np.stack([p // (ny * nz), (p // nz) % ny, p % nz], axis=1).astype(np.float64)
    rows = np.arange(len(ids))
    f1, f2 = ud[p], ud[p + strides[a]]
    x1 = xyz[rows, a]
    x2 = x1 + 1.0
    xyz[rows, a] = ((x2 - x1) * (thr - f1)) / (f2 - f1) + x1
    # cube cases: bit i set when corner i is low
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.uint8)
    for i in range(8):
        dx, dy, dz = i & 1, (i >> 1) & 1, (i >> 2) & 1
        case |= low[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.uint8) << i
    count, tri = _table()
    hit = count[case] > 0
    cube = lin[:-1, :-1, :-1][hit]                    # C order = ascending lower-corner index
    cs = case[hit]
    edges = tri[cs]                                   # [m, 10, 3]
    corner_off = np.array([(c & 1) * strides[0] + ((c >> 1) & 1) * strides[1] + (c >> 2) * strides[2] for c in range(8)], np.int64)
    edge_off = corner_off[[edge_corners(e)[0] for e in range(12)]]
    gid = 3 * (cube[:, None, None] + edge_off[edges]) + edges // 4
    gid = gid[np.arange(MAX_TRIS)[None, :] < count[cs][:, None]]
    return xyz, np.searchsorted(ids, gid).astype(np.int64)


def to_world(vertices, resolution, lo, hi):
    """nerf_utils.py:94-98: lattice-index units -> world coordinates over [lo, hi]"""
    return vertices / (resolution - 1.0) * (hi - lo)[None, :] + lo[None, :]


def read_stl(path):
    """binary STL -> (header bytes, normals float32 [T, 3], vertices float32 [T, 3, 3], attribute uint16 [T])"""
    data = open(path, 'rb').read()
    header = data[:80]
    n, = struct.unpack('<I', data[80:84])
    assert len(data) == 84 + 50 * n, (len(data), n)
    rec = np.frombuffer(data[84:], np.dtype([('normal', '<f4', (3,)), ('vertices', '<f4', (3, 3)), ('attr', '<u2')]), count=n)
    return header, rec['normal'].copy(), rec['vertices'].copy(), rec['attr'].copy()
