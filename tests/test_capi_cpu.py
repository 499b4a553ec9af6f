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


def test_python_frontend_refuses_cpu_tensors():
    import pytest
    import torch
    from ssdnerf_b200 import raymarching as rm
    from ssdnerf_b200._lib import SSDNeRFNativeError
    with pytest.raises(SSDNeRFNativeError):
        rm.near_far_from_aabb(torch.zeros(4, 3), torch.ones(4, 3), torch.tensor([-1., -1, -1, 1, 1, 1]))
