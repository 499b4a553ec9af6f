"""The C-ABI shared library builds for sm_90a, loads without a GPU and exports every symbol include/ssdnerf_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'ssdnerf_b200.h')).read()
    return sorted(set(re.findall(r'SSDNERF_API\s+[\w\s\*]+?\b(ssdnerf_\w+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from ssdnerf_b200.build import build_lib
    lib = ctypes.CDLL(build_lib())
    names = _declared()
    assert len(names) >= 20
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    lib.ssdnerf_last_error.restype = ctypes.c_char_p
    assert lib.ssdnerf_compiled_arch() == 90
    assert isinstance(lib.ssdnerf_last_error(), bytes)


def test_argument_errors_without_gpu():
    """size queries and argument validation are host-only and must work (and fail loudly) without a device"""
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    assert L.ssdnerf_decoder_blob_floats(ctypes.c_int(0)) == 2572
    assert L.ssdnerf_decoder_blob_floats(ctypes.c_int(1)) == 31500
    assert L.ssdnerf_planes_bytes(ctypes.c_int(0), ctypes.c_uint32(1), ctypes.c_uint32(128), ctypes.c_uint32(128)) == 3 * 128 * 128 * 8 * 4
    assert L.ssdnerf_render_fwd(None, None) == -2
    assert b'NULL' in L.ssdnerf_last_error()


def test_unknown_decoder_variant_is_rejected_before_any_launch():
    """only SSDNERF_DEC_P (0) and SSDNERF_DEC_S (1) exist; render_fwd rejects any other id before it enqueues work on the stream"""
    from ssdnerf_b200 import _lib as N
    L = N.lib()
    u32 = ctypes.c_uint32
    n, max_steps = 64 * 64, 256
    ws_bytes = L.ssdnerf_render_workspace_bytes(u32(1), u32(n), u32(max_steps))
    fake = ctypes.c_void_p(1 << 20)                  # never dereferenced: validation fails first
    for v in (2, 4, 5, 7, -1):
        assert L.ssdnerf_decoder_blob_floats(ctypes.c_int(v)) == 0
        assert L.ssdnerf_planes_bytes(ctypes.c_int(v), u32(1), u32(128), u32(128)) == 0
        assert L.ssdnerf_pack_planes(ctypes.c_int(v), None, u32(1), u32(6), u32(128), u32(128), None, None) == -2
        a = N.RenderArgs()
        a.variant, a.num_scenes, a.rays_per_scene = v, 1, n
        a.rays_o = a.rays_d = a.planes = a.bitfield = a.decoder_blob = a.weights_sum = a.image = fake
        a.plane_h = a.plane_w = 128
        a.grid_size, a.bound, a.min_near, a.T_thresh, a.max_steps = 64, 1.0, 0.2, 1e-4, max_steps
        a.workspace, a.workspace_bytes = fake, ws_bytes
        assert L.ssdnerf_render_fwd(ctypes.byref(a), None) == -2, v
        assert b'variant' in L.ssdnerf_last_error()


def test_ctypes_arg_structs_match_header(tmp_path):
    """every ctypes argument struct mirrors its header struct field by field: the host compiler's sizeof and offsetof for the header
    equal ctypes' layout"""
    import subprocess
    from ssdnerf_b200 import _lib as N
    from ssdnerf_b200 import unet_ops as U
    mirrors = {'ssdnerf_render_args': N.RenderArgs, 'ssdnerf_render_train_args': N.RenderTrainArgs, 'ssdnerf_gemm_args': U.GemmArgs,
               'ssdnerf_gn_bwd_args': U.GnBwdArgs, 'ssdnerf_wgrad_args': U.WgradArgs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ssdnerf_b200.h"', 'int main(void) {']
    expect = []
    for cname, mirror in mirrors.items():
        lines.append(f'    printf("%zu\\n", sizeof({cname}));')
        expect.append(ctypes.sizeof(mirror))
        for name, _ in mirror._fields_:
            lines.append(f'    printf("%zu\\n", offsetof({cname}, {name}));')
            expect.append(getattr(mirror, name).offset)
    lines += ['    return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines) + '\n')
    subprocess.run(['cc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == expect


def test_python_frontend_refuses_cpu_tensors():
    import pytest
    import torch
    from ssdnerf_b200 import raymarching as rm
    from ssdnerf_b200._lib import SSDNeRFNativeError
    with pytest.raises(SSDNeRFNativeError):
        rm.near_far_from_aabb(torch.zeros(4, 3), torch.ones(4, 3), torch.tensor([-1., -1, -1, 1, 1, 1]))
