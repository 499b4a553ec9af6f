"""Mesh export: marching cubes on the device (csrc/mesh.cu) and a binary STL writer -- the surface and file steps of the reference's
`save_mesh` (lib/core/utils/nerf_utils.py:84-112 with PyMCubes, base_nerf.py:172-182 with trimesh), neither package needed."""
import ctypes

import numpy as np
import torch

from . import _lib as N


def case_table():
    """the generated marching-cubes case table the kernel uses: triangle counts uint8 [256] and cube-edge numbers uint8 [256, 10, 3]
    (layout in include/ssdnerf_b200.h, ssdnerf_mc_case_table)"""
    count, tri = np.zeros(256, np.uint8), np.zeros((256, 10, 3), np.uint8)
    N.check(N.lib().ssdnerf_mc_case_table(count.ctypes.data_as(ctypes.c_void_p), tri.ctypes.data_as(ctypes.c_void_p)))
    return count, tri


def marching_cubes(u, threshold):
    """PyMCubes' `marching_cubes(u, threshold)` on a CUDA float32 lattice u [nx, ny, nz] (indexed [x, y, z]) on the current device:
    vertices float64 [V, 3] in lattice-index units and triangles int64 [T, 3], both CUDA tensors.  One vertex per crossed lattice edge
    (a point is low when u <= threshold), ordered by edge id; triangle normals (v1 - v0) x (v2 - v0) point toward lower u.  A count
    pass, one host read of the totals, an emit pass; the result is deterministic."""
    N.require_cuda(u)
    if u.dim() != 3 or u.dtype != torch.float32:
        raise ValueError(f'marching_cubes: u must be a float32 [nx, ny, nz] tensor, got {u.dtype} {tuple(u.shape)}')
    u = u.contiguous()
    nx, ny, nz = u.shape
    L, dev, stream = N.lib(), u.device, N.stream_ptr()
    thr = float(threshold)
    work = torch.empty(L.ssdnerf_mc_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    N.check(L.ssdnerf_mc_count(N.ptr(u), nx, ny, nz, thr, N.ptr(work), N.ptr(counts), stream))
    nv, nt = counts.tolist()
    vertices = torch.empty(nv, 3, dtype=torch.float64, device=dev)
    triangles = torch.empty(nt, 3, dtype=torch.int64, device=dev)
    if nv or nt:
        N.check(L.ssdnerf_mc_emit(N.ptr(u), nx, ny, nz, thr, N.ptr(work), N.ptr(vertices), N.ptr(triangles), stream))
    return vertices, triangles


STL_HEADER = b'binary STL, ssdnerf_b200 marching cubes'.ljust(80, b' ')
STL_FACE = np.dtype([('normal', '<f4', (3,)), ('vertices', '<f4', (3, 3)), ('attr', '<u2')])     # 50 bytes, packed


def write_stl(path, vertices, triangles):
    """binary STL of an indexed mesh (numpy arrays or tensors): 80-byte header (not starting with `solid`), uint32 face count, and per
    face the float32 unit normal of (v1 - v0) x (v2 - v0) (zero for a zero-area face), the three float32 vertices and a uint16 0"""
    v = vertices.detach().cpu().numpy() if torch.is_tensor(vertices) else np.asarray(vertices)
    t = triangles.detach().cpu().numpy() if torch.is_tensor(triangles) else np.asarray(triangles)
    corners = v.astype(np.float64)[t.reshape(-1, 3)]                    # [T, 3, 3]
    n = np.cross(corners[:, 1] - corners[:, 0], corners[:, 2] - corners[:, 0])
    norm = np.linalg.norm(n, axis=1, keepdims=True)
    faces = np.zeros(len(corners), STL_FACE)
    faces['normal'] = np.divide(n, norm, out=np.zeros_like(n), where=norm > 0)
    faces['vertices'] = corners
    with open(path, 'wb') as f:
        f.write(STL_HEADER)
        f.write(np.uint32(len(faces)).tobytes())
        faces.tofile(f)
