"""ssdnerf_b200 -- H100-native (sm_90a) implementation of SSDNeRF's two data-parallel hot paths.

    renderer / decoders : fused occupancy-grid triplane renderer  (csrc/render.cu, csrc/render_p3.cu, csrc/render_s2.cu)
    density             : occupancy-grid builder                   (csrc/density.cu)
    unet / diffusion    : DDIM loop over triplane latents          (csrc/gemm_tc.cu, csrc/unet_glue.cu)
    raymarching / shencoder / activation : one-to-one mirrors of the reference's lib.ops (csrc/legacy_ops.cu)
    mesh                : marching cubes + binary STL of save_mesh  (csrc/mesh.cu)
    viz                 : PNG files under viz_dir, interpolation demo (csrc/png.cu)
    datasets            : ShapeNet SRN scenes, GPU PNG decoding of their views (csrc/png_decode.cu)
    evaluation          : the evaluation loop of tools/test.py (`evaluate_3d`, `SceneBatches`); `python -m ssdnerf_b200.test` runs it
    runner / ema        : the training runner of tools/train.py and its hooks, the fused EMA update (csrc/ema.cu);
                          `python -m ssdnerf_b200.train` runs it
    video / orbit       : orbit videos of the GUI's export: baseline JPEG frames on the device (csrc/jpeg.cu) in a Motion-JPEG AVI,
                          or all-intra H.264 (csrc/h264.cu) in an MP4; `python -m ssdnerf_b200.orbit` renders them

Everything computes through libssdnerf_b200.so (C ABI: include/ssdnerf_b200.h); there is no CPU or PyTorch fallback.
"""
from .registry import DATASETS, MODELS, MODULES, build_dataset, build_model, build_module  # noqa: F401
from .config import Config  # noqa: F401
from . import activation, datasets, decoders, density, diffusion, ema, evaluation, mesh, nerf, raymarching, renderer, runner, scene_cache, shencoder, unet, video, viz  # noqa: F401
from .datasets import ShapeNetSRN, collate, decode_png  # noqa: F401
from .decoders import TriPlaneDecoder  # noqa: F401
from .evaluation import SceneBatches, evaluate_3d  # noqa: F401
from .diffusion import GaussianDiffusion  # noqa: F401
from .nerf import DiffusionNeRF, MultiSceneNeRF  # noqa: F401
from .unet import DenoisingUnetMod  # noqa: F401
from .viz import interp_diffusion_nerf_ddim  # noqa: F401

__version__ = '0.1.0'
