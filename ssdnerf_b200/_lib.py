"""ctypes binding of libssdnerf_b200.so (C ABI: include/ssdnerf_b200.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes
import os

import torch  # noqa: F401  (loads libcudart before our library)

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, 'libssdnerf_b200.so')
_lib = None

c_void_p = ctypes.c_void_p
c_u32 = ctypes.c_uint32
c_f32 = ctypes.c_float
c_double = ctypes.c_double
c_int = ctypes.c_int
c_size_t = ctypes.c_size_t
c_longlong = ctypes.c_longlong


class SSDNeRFNativeError(RuntimeError):
    pass


class RenderArgs(ctypes.Structure):
    """mirror of `ssdnerf_render_args` (include/ssdnerf_b200.h)"""
    _fields_ = [
        ('variant', c_int), ('num_scenes', c_u32), ('rays_per_scene', c_u32),
        ('rays_o', c_void_p), ('rays_d', c_void_p),
        ('poses', c_void_p), ('intrinsics', c_void_p),
        ('num_views', c_u32), ('img_h', c_u32), ('img_w', c_u32),
        ('planes', c_void_p), ('plane_h', c_u32), ('plane_w', c_u32),
        ('bitfield', c_void_p), ('grid_size', c_u32),
        ('decoder_blob', c_void_p), ('dt_gamma', c_void_p),
        ('bound', c_f32), ('min_near', c_f32), ('T_thresh', c_f32), ('bg_color', c_f32),
        ('max_steps', c_u32), ('emulate_schedule', c_int),
        ('weights_sum', c_void_p), ('depth', c_void_p), ('image', c_void_p), ('rgb_blend', c_void_p),
        ('num_samples', c_void_p), ('voxel_trace', c_void_p), ('trace_cap', c_u32),
        ('workspace', c_void_p), ('workspace_bytes', c_size_t),
    ]


class RenderTrainArgs(ctypes.Structure):
    """mirror of `ssdnerf_render_train_args` (include/ssdnerf_b200.h)"""
    _fields_ = [
        ('variant', c_int), ('num_scenes', c_u32), ('rays_per_scene', c_u32),
        ('rays_o', c_void_p), ('rays_d', c_void_p), ('noises', c_void_p),
        ('planes', c_void_p), ('plane_h', c_u32), ('plane_w', c_u32),
        ('bitfield', c_void_p), ('grid_size', c_u32),
        ('decoder_blob', c_void_p), ('dt_gamma', c_void_p),
        ('bound', c_f32), ('min_near', c_f32), ('T_thresh', c_f32),
        ('max_steps', c_u32),
        ('weights_sum', c_void_p), ('depth', c_void_p), ('image', c_void_p), ('num_samples', c_void_p),
        ('grad_ws', c_void_p), ('grad_image', c_void_p), ('grad_planes', c_void_p),
        ('counter', c_void_p), ('grad_decoder_blob', c_void_p),
    ]


class EmaTensor(ctypes.Structure):
    """mirror of `ssdnerf_ema_tensor` (include/ssdnerf_b200.h)"""
    _fields_ = [('ema', c_void_p), ('src', c_void_p), ('n', ctypes.c_uint64), ('trainable', c_u32)]


def lib():
    """Load the native library; raises if it has not been built (python -m ssdnerf_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise SSDNeRFNativeError(
                f'{_PATH} not found: build it with `python -m ssdnerf_b200.build` '
                '(there is no CPU / PyTorch fallback for the hot path)')
        L = ctypes.CDLL(_PATH)
        L.ssdnerf_last_error.restype = ctypes.c_char_p
        for name in ('ssdnerf_decoder_blob_floats', 'ssdnerf_planes_bytes', 'ssdnerf_render_workspace_bytes',
                     'ssdnerf_density_workspace_bytes', 'ssdnerf_unet_workspace_bytes'):
            if hasattr(L, name):
                getattr(L, name).restype = c_size_t
        # mesh extraction (header section 6)
        L.ssdnerf_mc_workspace_bytes.argtypes = [c_u32, c_u32, c_u32]
        L.ssdnerf_mc_workspace_bytes.restype = c_size_t
        L.ssdnerf_mc_count.argtypes = [c_void_p, c_u32, c_u32, c_u32, c_double, c_void_p, c_void_p, c_void_p]
        L.ssdnerf_mc_emit.argtypes = [c_void_p, c_u32, c_u32, c_u32, c_double, c_void_p, c_void_p, c_void_p, c_void_p]
        L.ssdnerf_mc_case_table.argtypes = [c_void_p, c_void_p]
        # PNG encoding (header section 8)
        for name in ('ssdnerf_png_workspace_bytes', 'ssdnerf_png_output_bound'):
            getattr(L, name).argtypes = [c_u32, c_u32, c_u32]
            getattr(L, name).restype = c_size_t
        L.ssdnerf_png_encode_views.argtypes = [c_void_p, c_void_p, c_u32, c_u32, c_u32, c_void_p, c_size_t, c_void_p, c_size_t,
                                               c_void_p, c_void_p]
        L.ssdnerf_png_encode_maps.argtypes = [c_void_p, c_u32, c_u32, c_u32, c_f32, c_f32, c_void_p, c_size_t, c_void_p, c_size_t,
                                              c_void_p, c_void_p]
        L.ssdnerf_png_viridis.argtypes = [c_void_p]
        # PNG decoding (header section 9)
        L.ssdnerf_png_decode_workspace_bytes.argtypes = [c_u32, c_u32, c_int]
        L.ssdnerf_png_decode_workspace_bytes.restype = c_size_t
        L.ssdnerf_png_decode.argtypes = [c_void_p, c_size_t, c_void_p, c_u32, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p]
        L.ssdnerf_png_decode_host.argtypes = [ctypes.c_char_p, c_size_t, c_u32, c_u32, c_int, ctypes.c_char_p, c_void_p, c_void_p]
        # KITTI instance crops (header section 10)
        L.ssdnerf_png_decode_raw_workspace_bytes.argtypes = [c_u32, c_u32, c_int, c_int]
        L.ssdnerf_png_decode_raw_workspace_bytes.restype = c_size_t
        L.ssdnerf_png_decode_raw.argtypes = [c_void_p, c_size_t, c_void_p, c_u32, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p,
                                             c_void_p]
        L.ssdnerf_png_decode_raw_host.argtypes = [ctypes.c_char_p, c_size_t, c_u32, c_u32, c_int, c_int, c_void_p, c_void_p]
        L.ssdnerf_kitti_boxes.argtypes = [c_void_p, c_void_p, c_u32, c_void_p, c_u32, c_void_p]
        L.ssdnerf_kitti_crops.argtypes = [c_void_p, c_void_p, c_void_p, c_u32, c_void_p, c_u32, c_u32, c_void_p, c_void_p, c_void_p]
        L.ssdnerf_kitti_resize_host.argtypes = [c_void_p, c_u32, c_u32, c_u32, c_u32, c_void_p]
        L.ssdnerf_png_bgr_layout.argtypes = [c_void_p, c_u32, c_void_p, c_void_p]
        L.ssdnerf_png_encode_bgr.argtypes = [c_void_p, c_void_p, c_void_p, c_u32, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p]
        # exponential moving average (header section 11)
        L.ssdnerf_ema_lerp_f32.argtypes = [ctypes.POINTER(EmaTensor), c_u32, c_f32, c_f32, c_void_p]
        # JPEG encoding (header section 12)
        for name in ('ssdnerf_jpeg_workspace_bytes', 'ssdnerf_jpeg_output_bound'):
            getattr(L, name).argtypes = [c_u32, c_u32, c_u32]
            getattr(L, name).restype = c_size_t
        for name in ('ssdnerf_jpeg_encode_u8', 'ssdnerf_jpeg_encode_f32'):
            getattr(L, name).argtypes = [c_void_p, c_u32, c_u32, c_u32, c_int, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p]
        # H.264 encoding (header section 13)
        for name in ('ssdnerf_h264_workspace_bytes', 'ssdnerf_h264_output_bound'):
            getattr(L, name).argtypes = [c_u32, c_u32, c_u32]
            getattr(L, name).restype = c_size_t
        for name in ('ssdnerf_h264_encode_u8', 'ssdnerf_h264_encode_f32'):
            getattr(L, name).argtypes = [c_void_p, c_u32, c_u32, c_u32, c_int, c_u32, c_u32, c_u32, c_void_p, c_size_t, c_void_p, c_size_t,
                                         c_void_p, c_void_p]
        _lib = L
    return _lib


def check(code):
    if code != 0:
        raise SSDNeRFNativeError(f'libssdnerf_b200 error {code}: {lib().ssdnerf_last_error().decode()}')


def ptr(t):
    """device pointer of a contiguous tensor (None -> NULL)"""
    if t is None:
        return None
    assert t.is_contiguous(), 'native ops need contiguous tensors'
    return c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(*tensors):
    """Every native op launches on the CURRENT device's current stream (`stream_ptr`), so its tensors must live on that device:
    a model on cuda:1 needs `torch.cuda.set_device(1)` (or a `torch.cuda.device(1)` block) around its calls -- enforced here
    instead of launching device-0 kernels on device-1 pointers."""
    cur = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise SSDNeRFNativeError('ssdnerf_b200 ops run on CUDA tensors only (no CPU fallback)')
        if cur is None:
            cur = torch.cuda.current_device()
        if t.device.index != cur:
            raise SSDNeRFNativeError(f'tensor on cuda:{t.device.index} but the current device is cuda:{cur}: the library launches on the '
                                     'current device (one GPU per process, or wrap the call in torch.cuda.device(...))')
