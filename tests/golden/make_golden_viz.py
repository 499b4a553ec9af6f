"""Pins for the viz_dir outputs: the reference's OWN `BaseNeRF.eval_and_viz` (with and without test images),
`TriPlaneDecoder.visualize` and `lib/apis/inference.py:interp_diffusion_nerf_ddim`, executed from /root/reference on CPU.  As in
make_golden_joint_step.py the volume renderer is tests/common.py:ToyDecoder and mmgen / mmcv are stubbed; `eval_ssim_skimage` is
oracle/metrics_port.py; `plt.imsave` is a recorder that keeps (file name, array, vmin, vmax) and creates an empty file, so the
reference's glob-and-delete of stale files acts on a real directory.  The interpolation's `model.val_step` records its `data` dicts.
-> tests/golden/reference_viz_v1.npz, replayed by tests/test_viz_cpu.py and tests/test_viz_gpu.py.

    python tests/golden/make_golden_viz.py          (needs /root/reference)
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import metrics_port  # noqa: E402
from tests.golden import make_golden_ref as G  # noqa: E402
from tests.golden.make_golden_joint_step import MODEL1, load_all, views  # noqa: E402

STALE = ['scene_a_v0_psnr1.0_ssim0.00_lpipsnan.png', 'scene_a_v0.png', 'scene_a_v00_keep.png', 'scene_b_1_old.png', 'other.png']
PATHS = [['/d/a/v0.png', '/d/a/v1.jpg', '/d/a/v2.png'], ['/d/b/10.png', '/d/b/1.png', '/d/b/2.png']]   # stem '1' is a prefix of '10'


class Recorder:
    def __init__(self):
        self.calls = []

    def imsave(self, fname, arr, vmin=None, vmax=None, **kw):
        self.calls.append((os.path.basename(fname), np.array(arr), vmin, vmax))
        open(fname, 'wb').close()


def load_visualize(plt):
    """TriPlaneDecoder.visualize of triplane_decoder.py, loaded with its heavy imports stubbed"""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m
    mod('reflib.models.decoders').__path__ = []
    mod('reflib.models.decoders.base_volume_renderer', VolumeRenderer=nn.Module)
    sys.modules['mmcv.cnn'].xavier_init = sys.modules['mmcv.cnn'].constant_init = None
    sys.modules['lib.ops'].SHEncoder = sys.modules['lib.ops'].TruncExp = None
    tri = G._load('lib/models/decoders/triplane_decoder.py', 'reflib.models.decoders.triplane_decoder')
    tri.plt = plt
    return tri.TriPlaneDecoder.visualize


def run_reference():
    msn, dn, den = load_all()
    base = sys.modules['reflib.models.autodecoders.base_nerf']
    plt = Recorder()
    base.plt = plt
    base.eval_ssim_skimage = lambda p, t, data_range=1: torch.from_numpy(       # [n, 3, h, w] -> per-image SSIM
        metrics_port.ssim_skimage(p.permute(0, 2, 3, 1), t.permute(0, 2, 3, 1)))
    visualize = load_visualize(plt)
    out = {}
    torch.manual_seed(0)
    m = msn.MultiSceneNeRF(**dict(MODEL1, code_size=(3, 6, 8, 8), use_lpips_metric=False), train_cfg=dict(), test_cfg=dict())
    m.eval()
    dec = m.decoder
    dec.flip_z = False
    toy_forward = dec.forward

    def eval_forward(*a, **k):                 # the reference's eval-mode renderer returns per-scene lists
        return {key: list(v) if torch.is_tensor(v) else v for key, v in toy_forward(*a, **k).items()}
    dec.forward = eval_forward
    dec.visualize = types.MethodType(visualize, dec)
    g = torch.Generator().manual_seed(3)
    code = torch.randn(2, 3, 6, 8, 8, generator=g) * 0.8
    with torch.no_grad():
        m.init_code.copy_(torch.randn(3, 6, 8, 8, generator=g) * 0.5)
    bits = torch.zeros(2, 8 ** 3 // 8, dtype=torch.uint8)
    imgs, poses, intr = views(2, 3, 16, 42)
    out.update(code=code.numpy(), init_code=m.init_code.numpy().copy(), test_imgs=imgs.numpy(), poses=poses.numpy(), intr=intr.numpy(),
               paths=np.array(PATHS), stale=np.array(STALE))
    cfg = dict(img_size=(16, 16), clip_range=[-1.5, 1.5], dt_gamma_scale=0.5)
    for tag, data in (('eval', dict(scene_name=['a', 'b'], test_poses=poses, test_intrinsics=intr, test_imgs=imgs, test_img_paths=PATHS)),
                      ('noimg', dict(scene_name=['a', 'b'], test_poses=poses, test_intrinsics=intr))):
        plt.calls.clear()
        with tempfile.TemporaryDirectory() as d, torch.no_grad():
            for f in STALE:
                open(os.path.join(d, f), 'wb').close()
            image, _ = m.render(dec, code, bits, 16, 16, intr, poses, cfg=cfg)
            log_vars, _ = m.eval_and_viz(data, dec, code, bits, viz_dir=d, cfg=cfg)
            out[f'{tag}_files'] = np.array(sorted(os.listdir(d)))
        out[f'{tag}_image'] = image.numpy()
        out[f'{tag}_names'] = np.array([c[0] for c in plt.calls])
        views_ = [c for c in plt.calls if c[2] is None]
        maps = [c for c in plt.calls if c[2] is not None]
        out[f'{tag}_u8'] = np.stack([c[1] for c in views_])
        out[f'{tag}_maps'] = np.stack([c[1].astype(np.float32) for c in maps[:2]])
        out[f'{tag}_mean_map'] = maps[2][1].astype(np.float32)
        out[f'{tag}_vrange'] = np.array([[c[2], c[3]] for c in maps], np.float64)
    # interpolation: the reference's own function with a recording val_step
    inf = load_inference()
    rec = []
    model = types.SimpleNamespace(code_size=(3, 6, 8, 8), val_step=lambda data, **kw: rec.append((data, kw)))
    model.parameters = lambda: iter([torch.zeros(1)])
    for typ in ('linear', 'spherical_linear'):
        rec.clear()
        torch.manual_seed(17)
        inf.interp_diffusion_nerf_ddim(model, poses[0], intr[0], viz_dir='/v', num_samples=5, batchsize=2, type=typ)
        out[f'interp_{typ}_noise'] = torch.cat([r[0]['noise'] for r in rec]).numpy()
        out[f'interp_{typ}_names'] = np.array(sum([r[0]['scene_name'] for r in rec], []))
        out[f'interp_{typ}_ids'] = np.array(sum([list(r[0]['scene_id']) for r in rec], []))
        out[f'interp_{typ}_batch'] = np.array([len(r[0]['scene_name']) for r in rec])
        assert all(r[0]['test_poses'].shape == (len(r[0]['scene_name']), 3, 4, 4) for r in rec)
        assert all(r[1] == dict(viz_dir='/v', show_pbar=True) for r in rec)
    return out


def load_inference():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m
    sys.modules['mmgen.models'].build_model = None
    sys.modules['mmgen.models.architectures.common'].get_module_device = lambda m: torch.device('cpu')
    mod('lib.runner'); mod('lib.runner.hooks'); mod('lib.runner.hooks.ema_hook', get_ori_key=None)
    return G._load('lib/apis/inference.py', 'ref_inference')


def main():
    out = run_reference()
    path = os.path.join(HERE, 'reference_viz_v1.npz')
    np.savez_compressed(path, **out)
    print(path, sorted(out))


if __name__ == '__main__':
    main()
