"""Image files under `viz_dir`: the plt.imsave calls of the reference's `eval_and_viz` (base_nerf.py:574-608), `TriPlaneDecoder.visualize`
(triplane_decoder.py:186-194) and the interpolation demo (lib/apis/inference.py:55-100), encoded as PNG on the device (csrc/png.cu).

The pixels follow the reference's formulas; the compressed bytes are the encoder's own (decoded pixels are the contract).  Only the
compressed files are copied to the host, once per call, and then written."""
import ctypes
import glob
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as N


def viridis():
    """the viridis table of the colormap mode, uint8 [256, 3] RGB"""
    t = np.zeros((256, 3), np.uint8)
    N.check(N.lib().ssdnerf_png_viridis(t.ctypes.data_as(ctypes.c_void_p)))
    return t


def code_maps(code, flip_z=False):
    """the 2-D map `visualize` draws of triplane codes [n, 3, C, h, w]: rows flipped unless flip_z, laid out as [n, 3 h, C w]"""
    n, _, c, h, w = code.shape
    if not flip_z:
        code = code.flip(-2)
    return code.permute(0, 1, 3, 2, 4).reshape(n, 3 * h, c * w)


def encode_png(pred=None, real=None, maps=None, vmin=0.0, vmax=1.0):
    """PNG files (list of bytes), 8-bit RGBA, from CUDA fp32 images in one of two modes:
      * views: pred [n, h, w, 3] channels-last renders, bytes round(round(clamp(x, 0, 1) * 255) / 255 * 255); with real [n, h, w, 3]
        (bytes (t * 255) truncated) each file is real | pred side by side, 2 w wide;
      * maps: maps [n, h, w] through viridis with matplotlib's Normalize(vmin, vmax) index rule.
    Rows of 4 w + 1 bytes must fit SSDNERF_PNG_SEGMENT_BYTES (w <= 4095)."""
    if (pred is None) == (maps is None):
        raise ValueError('encode_png: give exactly one of pred (views) and maps')
    src = pred if maps is None else maps
    N.require_cuda(src, real)
    if maps is None:
        if pred.dim() != 4 or pred.shape[-1] != 3 or pred.dtype != torch.float32:
            raise ValueError(f'encode_png: pred must be float32 [n, h, w, 3], got {pred.dtype} {tuple(pred.shape)}')
        if real is not None and (real.shape != pred.shape or real.dtype != torch.float32):
            raise ValueError(f'encode_png: real must match pred, got {real.dtype} {tuple(real.shape)}')
        n, h, wv, _ = pred.shape
        w = 2 * wv if real is not None else wv
    else:
        if maps.dim() != 3 or maps.dtype != torch.float32:
            raise ValueError(f'encode_png: maps must be float32 [n, h, w], got {maps.dtype} {tuple(maps.shape)}')
        if real is not None:
            raise ValueError('encode_png: real goes with pred, not maps')
        if float(vmin) > float(vmax):
            raise ValueError(f'encode_png: vmin {vmin} > vmax {vmax}')
        n, h, w = maps.shape
    if n == 0:
        return []
    L, dev, stream = N.lib(), src.device, N.stream_ptr()
    ws_bytes, out_bytes = L.ssdnerf_png_workspace_bytes(n, h, w), L.ssdnerf_png_output_bound(n, h, w)
    if ws_bytes == 0:
        raise ValueError(f'encode_png: unsupported size n={n} h={h} w={w} (a row of 4 w + 1 bytes must fit 16384)')
    work = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    if maps is None:
        pred = pred.contiguous()
        real = real.contiguous() if real is not None else None
        N.check(L.ssdnerf_png_encode_views(N.ptr(pred), N.ptr(real), n, h, wv, N.ptr(work), ws_bytes, N.ptr(out), out_bytes,
                                           N.ptr(offsets), stream))
    else:
        maps = maps.contiguous()
        vrange = float(np.float32(float(vmax) - float(vmin)))
        N.check(L.ssdnerf_png_encode_maps(N.ptr(maps), n, h, w, float(vmin), vrange, N.ptr(work), ws_bytes, N.ptr(out), out_bytes,
                                          N.ptr(offsets), stream))
    off = offsets.cpu().tolist()
    data = out[:off[-1]].cpu().numpy().tobytes()
    return [data[off[i]:off[i + 1]] for i in range(n)]


def write_pngs(paths, **kw):
    """encode_png(**kw) and write file i to paths[i]"""
    files = encode_png(**kw)
    if len(files) != len(paths):
        raise ValueError(f'write_pngs: {len(paths)} paths for {len(files)} images')
    for path, data in zip(paths, files):
        with open(path, 'wb') as f:
            f.write(data)


def write_view_files(viz_dir, names, bases, files):
    """write files[i] to viz_dir/names[i] in order; with bases, first delete viz_dir/<bases[i]>*.png, as the reference does just before each
    view's imsave (base_nerf.py:594-603) -- so a view whose base name is a prefix of a later view's (stems '1' and '10') is deleted too"""
    for i, (name, data) in enumerate(zip(names, files)):
        if bases is not None:
            for f in glob.glob(os.path.join(viz_dir, bases[i] + '*.png')):
                os.remove(f)
        with open(os.path.join(viz_dir, name), 'wb') as f:
            f.write(data)


def view_file_names(scene_names, num_imgs, test_img_paths=None, psnr=None, ssim=None, lpips=None):
    """file names of eval_and_viz's view images, scene-major (base_nerf.py:588-600), and the base names whose `<base>*.png` files are
    deleted first (None without test images).  With test_img_paths: scene_<name>_<image stem>_psnr{:02.1f}_ssim{:.2f}_lpips{:.3f}.png
    from the per-image metrics (lpips None -> nan); without: scene_<name>_{:03d}.png."""
    names, bases = [], []
    for s, scene in enumerate(scene_names):
        for v in range(num_imgs):
            if test_img_paths is None:
                names.append('scene_' + scene + '_{:03d}.png'.format(v))
                continue
            k = s * num_imgs + v
            base = 'scene_' + scene + '_' + os.path.splitext(os.path.basename(test_img_paths[s][v]))[0]
            lp = float('nan') if lpips is None else float(lpips[k])
            names.append(base + '_psnr{:02.1f}_ssim{:.2f}_lpips{:.3f}.png'.format(float(psnr[k]), float(ssim[k]), lp))
            bases.append(base)
    return names, (bases if test_img_paths is not None else None)


def interp_noise(code_size, num_samples, type='linear'):
    """the interpolated noise batch of interp_diffusion_nerf_ddim [num_samples, *code_size] (CPU): two torch.randn draws a, b, then
    (1 - alpha) a + alpha b or the spherical form with theta = acos of the normalised dot product (inference.py:70-84)"""
    alpha = torch.linspace(0, 1, steps=num_samples)
    alpha = alpha.reshape([-1] + [1] * len(code_size))
    noise_ab = torch.randn((2,) + tuple(code_size))
    if type == 'spherical_linear':
        noise_ab_norm = F.normalize(noise_ab.flatten(1), dim=1)
        theta = torch.acos(noise_ab_norm.prod(dim=0).sum())
        return (torch.sin((1 - alpha) * theta) * noise_ab[0] + torch.sin(alpha * theta) * noise_ab[1]) / torch.sin(theta)
    if type == 'linear':
        return (1 - alpha) * noise_ab[0] + alpha * noise_ab[1]
    raise AttributeError(f'unknown interpolation type {type!r} (linear or spherical_linear)')


@torch.no_grad()
def interp_diffusion_nerf_ddim(model, test_poses, test_intrinsics, viz_dir=None, num_samples=10, batchsize=10, type='linear', **kwargs):
    """lib/apis/inference.py:55-100: sample `num_samples` scenes from noise interpolated between two draws, in batches of `batchsize`
    named interp_XX, through model.val_step; with viz_dir, every view of test_poses [V, 4, 4] and each triplane map is written there."""
    device = next(model.parameters()).device
    noise = interp_noise(model.code_size, num_samples, type)
    scene_id_cur = 0
    for noise_batch in noise.split(batchsize, dim=0):
        bs = noise_batch.size(0)
        scene_id = range(scene_id_cur, scene_id_cur + bs)
        data = dict(noise=noise_batch.to(device), scene_id=scene_id,
                    scene_name=['interp_{:02d}'.format(i) for i in scene_id],
                    test_intrinsics=test_intrinsics[None].expand(bs, -1, -1).to(device),
                    test_poses=test_poses[None].expand(bs, -1, -1, -1).to(device))
        model.val_step(data, viz_dir=viz_dir, show_pbar=True, **kwargs)
        scene_id_cur += bs
