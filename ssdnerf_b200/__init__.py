"""ssdnerf_b200 -- H100-native (sm_90a) implementation of SSDNeRF's two data-parallel hot paths.

    renderer / decoders : fused occupancy-grid triplane renderer  (csrc/render.cu, csrc/render_p3.cu, csrc/render_s2.cu)
    density             : occupancy-grid builder                   (csrc/density.cu)
    unet / diffusion    : DDIM loop over triplane latents          (csrc/gemm_tc.cu, csrc/unet_glue.cu)
    raymarching / shencoder / activation : one-to-one mirrors of the reference's lib.ops (csrc/legacy_ops.cu)
    mesh                : marching cubes + binary STL of save_mesh  (csrc/mesh.cu)

Everything computes through libssdnerf_b200.so (C ABI: include/ssdnerf_b200.h); there is no CPU or PyTorch fallback.
"""
from .registry import MODELS, MODULES, build_model, build_module  # noqa: F401
from .config import Config  # noqa: F401
from . import activation, decoders, density, diffusion, mesh, nerf, raymarching, renderer, scene_cache, shencoder, unet  # noqa: F401
from .decoders import TriPlaneDecoder  # noqa: F401
from .diffusion import GaussianDiffusion  # noqa: F401
from .nerf import DiffusionNeRF, MultiSceneNeRF  # noqa: F401
from .unet import DenoisingUnetMod  # noqa: F401

__version__ = '0.1.0'
