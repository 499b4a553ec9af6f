"""`python -m ssdnerf_b200.orbit CONFIG CHECKPOINT --cameras DIR (--seed S [S ...] | --scene FILE.pth [...])`: the reference GUI's
Generate, Load scene, Export video and Export mesh (lib/core/ssdnerf_gui.py, demo/ssdnerf_gui.py) without a window.

Each scene becomes `<out-dir>/<scene>.avi`, a Motion-JPEG orbit of round(fps * sec) frames on the path of `video.surround_views`
around the GUI's initial camera (pose `--camera-id` of DIR/pose, DIR/intrinsics.txt: any ShapeNet SRN scene directory or the
reference's demo/camera_spiral_cars), rendered at `--res` rows by `BaseNeRF.render` on a white background with dt_gamma 0, as the GUI
exports it.  Frames go from the renderer to the JPEG encoder on the device; only the compressed files reach the host.

  * --seed S: set_random_seed(S, deterministic=True), noise torch.randn((1,) + code_size) on the CPU, then val_uncond with
    `num_timesteps = --steps`; the scene is `seed_S`.  Seeds are sampled --batch-scenes at a time (each noise drawn after its own
    seeding, so the noise is the GUI's; a batch of one reproduces the GUI's sampling exactly, larger batches differ only where the
    sampler draws device noise, which DDIM does not).
  * --scene FILE.pth: `param.code`, or code_activation(param.code_) when only the pre-activation code is saved (files of test.py's
    save_dir and of the GUI's Save scene load); the occupancy grid is rebuilt with density_thresh 0.1, density_step 16; the scene is
    the file's stem.
  * --mesh: `<scene>.stl` as save_mesh writes it (--mesh-resolution, --mesh-threshold); --save-scene: `<scene>.pth` in the GUI's
    format, param = dict(code, density_bitfield).
"""
import argparse
import os
import time

import torch

from . import video
from .config import Config
from .registry import build_model
from .test import DictAction, load_checkpoint, set_random_seed

EMA_HOOKS = ('ExponentialMovingAverageHookMod', 'ExponentialMovingAverageHook')


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Render orbit videos (and meshes) of sampled or saved scenes')
    p.add_argument('config', help='config file')
    p.add_argument('checkpoint', help='checkpoint file')
    p.add_argument('--cameras', required=True, help='directory with pose/*.txt and intrinsics.txt (a ShapeNet SRN scene directory)')
    p.add_argument('--camera-id', type=int, default=64, help='index of the initial pose in the sorted pose/ listing')
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument('--seed', type=int, nargs='+', help='sample one scene per seed')
    src.add_argument('--scene', nargs='+', help='saved scene files (.pth)')
    p.add_argument('--steps', type=int, default=20, help='diffusion sampling steps (num_timesteps)')
    p.add_argument('--batch-scenes', type=int, default=4, help='seeds sampled per batch')
    p.add_argument('--out-dir', default='orbits', help='where <scene>.avi (and .stl / .pth) go')
    p.add_argument('--fps', type=int, default=30)
    p.add_argument('--sec', type=float, default=4.0, help='video length in seconds')
    p.add_argument('--res', type=int, default=256, help='video height in pixels (the width keeps the cameras\' aspect ratio)')
    p.add_argument('--batch-frames', type=int, default=30, help='frames rendered and encoded per batch')
    p.add_argument('--quality', type=int, default=95, help='JPEG quality 1-100')
    p.add_argument('--mesh', action='store_true', help='also write <scene>.stl')
    p.add_argument('--mesh-resolution', type=int, default=256)
    p.add_argument('--mesh-threshold', type=float, default=10)
    p.add_argument('--save-scene', action='store_true', help='also write <scene>.pth (code and density bitfield)')
    p.add_argument('--gpu-id', type=int, default=0)
    p.add_argument('--cfg-options', nargs='+', action=DictAction, help='override config entries, key=value')
    args = p.parse_args(argv)
    for name in ('steps', 'batch_scenes', 'fps', 'res', 'batch_frames', 'mesh_resolution'):
        if getattr(args, name) < 1:
            p.error(f'--{name.replace("_", "-")} must be >= 1')
    if not 1 <= args.quality <= 100:
        p.error('--quality must be in [1, 100]')
    if not round(args.fps * args.sec) >= 1:
        p.error('--fps * --sec must give at least one frame')
    return args


def init_model(cfg, checkpoint, device, ema_only=True, logger=None):
    """lib/apis/inference.py init_model: build, load the checkpoint (test.py's load_checkpoint), and with ema_only delete the source
    modules of the config's EMA hooks (`diffusion` for `diffusion_ema`), so only the averaged copies remain; eval mode on `device`"""
    model = build_model(cfg['model'], train_cfg=cfg.get('train_cfg'), test_cfg=cfg.get('test_cfg'))
    load_checkpoint(model, checkpoint, logger)
    if ema_only:
        keys = []
        for hook in cfg.get('custom_hooks', None) or []:
            if hook.get('type') in EMA_HOOKS:
                mk = hook['module_keys']
                keys.extend([mk] if isinstance(mk, str) else mk)
        for key in keys:
            head, _, rest = key.partition('.')
            del model._modules['.'.join([head[:-4]] + ([rest] if rest else []))]
    return model.to(device).eval()


def seed_noise(seed, code_size):
    """the GUI's draw: set_random_seed(seed, deterministic=True), then torch.randn((1,) + code_size) on the CPU"""
    set_random_seed(seed, deterministic=True)
    return torch.randn((1,) + tuple(code_size))


def sample_seeds(model, seeds, steps):
    """codes [n, *code_size] and density bitfields of val_uncond for `seeds`, sampled with num_timesteps = steps"""
    diffusion, _ = model._modules_for_eval()
    diffusion.test_cfg['num_timesteps'] = steps
    device = next(model.parameters()).device
    noise = torch.cat([seed_noise(s, model.code_size) for s in seeds], dim=0)
    data = dict(noise=noise.to(device), scene_id=list(range(len(seeds))), scene_name=[f'seed_{s}' for s in seeds])
    with torch.no_grad():
        code, _, bitfield = model.val_uncond(data, show_pbar=False, save_intermediates=False)
    return code, bitfield


def load_scene(model, path):
    """the GUI's Load scene: (code [*code_size] on the model's device, density bitfield), the bitfield rebuilt from the code"""
    try:
        scene = torch.load(path, map_location='cpu', weights_only=True)
    except Exception as e:
        raise RuntimeError(f'{path}: cannot be loaded with torch.load(weights_only=True): {e}') from e
    param = scene.get('param') if isinstance(scene, dict) else None
    if not isinstance(param, dict) or not ('code' in param or 'code_' in param):
        raise ValueError(f'{path}: not a scene file (expected param.code or param.code_)')
    device = next(model.parameters()).device
    code = param['code'] if 'code' in param else model.code_activation(param['code_'].float())
    code = code.to(device=device, dtype=torch.float32)
    if tuple(code.shape) != tuple(model.code_size):
        raise ValueError(f'{path}: code of shape {tuple(code.shape)}, the model takes {tuple(model.code_size)}')
    _, decoder = model._modules_for_eval()
    with torch.no_grad():
        _, bitfield = model.get_density(decoder, code[None], cfg=dict(density_thresh=0.1, density_step=16))
    return code, bitfield[0]


def orbit_geometry(cameras, camera_id, res, fps, sec):
    """(poses [F, 4, 4], intrinsics [4] scaled to the video, (h, w)) of the GUI's export: F = round(fps * sec), scale res / h"""
    pose, intrinsics, (h, w) = video.gui_camera(cameras, camera_id)
    scale = res / h
    poses = video.surround_views(pose, num_frames=int(round(fps * sec)))
    return poses, intrinsics * scale, (int(round(h * scale)), int(round(w * scale)))


def render_frames(model, code, bitfield, poses, intrinsics, hw):
    """renders [F, h, w, 3] fp32 of one scene from poses [F, 4, 4] on a white background, dt_gamma 0 (the GUI's export)"""
    _, decoder = model._modules_for_eval()
    device = code.device
    bg = model.bg_color
    model.bg_color = 1.0
    try:
        with torch.no_grad():
            image, _ = model.render(decoder, code[None], bitfield[None], hw[0], hw[1],
                                    intrinsics.to(device)[None, None].expand(1, poses.size(0), 4).contiguous(),
                                    poses.to(device)[None], cfg=dict())
    finally:
        model.bg_color = bg
    return image[0]


def orbit_jpegs(model, code, bitfield, poses, intrinsics, hw, batch_frames, quality):
    """the orbit's JPEG files, rendered and encoded batch_frames at a time"""
    files = []
    for lo in range(0, poses.size(0), batch_frames):
        files += video.encode_jpeg(render_frames(model, code, bitfield, poses[lo:lo + batch_frames], intrinsics, hw), quality)
    return files


def export_scene(model, name, code, bitfield, geometry, args):
    """writes <out_dir>/<name>.avi (and .stl / .pth); returns the written paths"""
    poses, intrinsics, hw = geometry
    out = {}
    jpegs = orbit_jpegs(model, code, bitfield, poses, intrinsics, hw, args.batch_frames, args.quality)
    out['avi'] = os.path.join(args.out_dir, name + '.avi')
    video.write_avi(out['avi'], jpegs, hw[1], hw[0], args.fps)
    if args.mesh:
        _, decoder = model._modules_for_eval()
        model.save_mesh(args.out_dir, decoder, code[None], [name], args.mesh_resolution, args.mesh_threshold)
        out['stl'] = os.path.join(args.out_dir, name + '.stl')
    if args.save_scene:
        out['pth'] = os.path.join(args.out_dir, name + '.pth')
        torch.save(dict(param=dict(code=code.cpu(), density_bitfield=bitfield.cpu())), out['pth'])
    return out


def main(argv=None):
    """renders every scene; returns {scene name: {'avi': path, 'stl': path, 'pth': path}} in order"""
    args = parse_args(argv)
    cfg = Config.fromfile(args.config)
    if args.cfg_options is not None:
        Config.merge_options(cfg, args.cfg_options)
    torch.cuda.set_device(args.gpu_id)
    device = torch.device('cuda', torch.cuda.current_device())
    model = init_model(cfg, args.checkpoint, device)
    geometry = orbit_geometry(args.cameras, args.camera_id, args.res, args.fps, args.sec)
    os.makedirs(args.out_dir, exist_ok=True)
    written = {}

    def done(name, code, bitfield, t0):
        written[name] = export_scene(model, name, code, bitfield, geometry, args)
        print(f'{name}: {", ".join(written[name].values())} ({time.perf_counter() - t0:.1f} s)', flush=True)

    if args.seed is not None:
        for lo in range(0, len(args.seed), args.batch_scenes):
            t0 = time.perf_counter()
            seeds = args.seed[lo:lo + args.batch_scenes]
            codes, bitfields = sample_seeds(model, seeds, args.steps)
            for s, code, bitfield in zip(seeds, codes, bitfields):
                done(f'seed_{s}', code, bitfield, t0)
    else:
        for path in args.scene:
            t0 = time.perf_counter()
            code, bitfield = load_scene(model, path)
            done(os.path.splitext(os.path.basename(path))[0], code, bitfield, t0)
    return written


if __name__ == '__main__':
    main()
