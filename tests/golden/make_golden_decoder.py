"""Pins for the RENDERER oracle's Python layer: the reference's OWN `TriPlaneDecoder` (`point_decode`, `forward` eval branch = the host-driven
march / decode / composite loop of base_volume_renderer.py:79-123, `forward` train branch :59-77) together with its OWN op wrappers
`lib/ops/raymarching/raymarching.py` and `lib/ops/shencoder/sphere_harmonics.py`, executed from /root/reference on CPU.  The only thing
replaced is the compiled extension underneath the wrappers (`_raymarching`, `_shencoder`): a fake `_backend` forwards every call, argument
for argument, to the C oracle (oracle/*.c), which the GPU tests hold BIT-EXACT to the reference's CUDA kernels (tests/test_ref_gpu.py).
So: reference Python + kernel-exact C  ->  tests/golden/reference_decoder_v1.npz, against which tests/test_reference_pin_cpu.py checks the
oracle's restatements `render_port.point_decode / render_eval_scene` and `train_port.render_train_scene` (the functions every GPU parity
test of the fused renderers is measured against).

    python tests/golden/make_golden_decoder.py          (needs /root/reference)

A second entry point runs the same train branch in the regimes where its edge rules act -- TruncExp's gradient floor, the plane borders,
non-square planes, a binding sample budget -- into tests/golden/reference_train_edges_v1.npz:

    python tests/golden/make_golden_decoder.py --train-edges
"""
import ctypes
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import oracle as orc  # noqa: E402
from oracle import render_port as rp  # noqa: E402
from tests.common import spiral_poses  # noqa: E402
from tests.golden import make_golden_ref as G  # noqa: E402

u32, f32 = ctypes.c_uint32, ctypes.c_float


def P(t):
    if t is None:
        return None
    assert t.is_contiguous()
    return ctypes.c_void_p(t.data_ptr())


def fake_backends():
    L = orc.lib()
    rm = types.ModuleType('_raymarching')
    rm.near_far_from_aabb = lambda ro, rd, aabb, N, min_near, nears, fars: L.orc_near_far_from_aabb(P(ro), P(rd), P(aabb), u32(N), f32(min_near), P(nears), P(fars))
    rm.march_rays_train = lambda ro, rd, bits, bound, dtg, max_steps, N, C, H, M, nears, fars, xyzs, dirs, deltas, rays, counter, noises: \
        L.orc_march_rays_train(P(ro), P(rd), P(bits), f32(bound), f32(dtg), u32(max_steps), u32(N), u32(C), u32(H), u32(M), P(nears), P(fars),
                               P(xyzs), P(dirs), P(deltas), P(rays), P(counter), P(noises), None)
    rm.composite_rays_train_forward = lambda s, c, d, rays, M, N, T, ws, dep, img: \
        L.orc_composite_rays_train_forward(P(s), P(c), P(d), P(rays), u32(M), u32(N), f32(T), P(ws), P(dep), P(img))
    rm.composite_rays_train_backward = lambda gws, gimg, s, c, d, rays, ws, img, M, N, T, gs, gc: \
        L.orc_composite_rays_train_backward(P(gws), P(gimg), P(s), P(c), P(d), P(rays), P(ws), P(img), u32(M), u32(N), f32(T), P(gs), P(gc))
    rm.march_rays = lambda na, ns, alive, t, ro, rd, bound, dtg, max_steps, C, H, bits, near, far, xyzs, dirs, deltas, noises: \
        L.orc_march_rays(u32(na), u32(ns), P(alive), P(t), P(ro), P(rd), f32(bound), f32(dtg), u32(max_steps), u32(C), u32(H), P(bits), P(near),
                         P(far), P(xyzs), P(dirs), P(deltas), P(noises), None)
    rm.composite_rays = lambda na, ns, T, alive, t, s, c, d, ws, dep, img: \
        L.orc_composite_rays(u32(na), u32(ns), f32(T), P(alive), P(t), P(s.contiguous()), P(c.contiguous()), P(d), P(ws), P(dep), P(img))
    sh = types.ModuleType('_shencoder')

    def sh_fwd(inputs, outputs, B, D, degree, calc_grad, dy_dx):
        assert D == 3 and not calc_grad
        L.orc_sh_encode(P(inputs), u32(B), u32(degree), P(outputs))
    sh.sh_encode_forward = sh_fwd
    sys.modules['_raymarching'], sys.modules['_shencoder'] = rm, sh


def load_reference_decoder():
    G._install_stubs()
    fake_backends()

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m
    ray = G._load('lib/ops/raymarching/raymarching.py', 'ref_raymarching')
    shm = G._load('lib/ops/shencoder/sphere_harmonics.py', 'ref_sphere_harmonics')
    act = G._load('lib/ops/activation.py', 'ref_activation2')
    mod('lib')
    mod('lib.ops', SHEncoder=shm.SHEncoder, TruncExp=act.TruncExp, **{k: getattr(ray, k) for k in (
        'batch_near_far_from_aabb', 'march_rays_train', 'batch_composite_rays_train', 'march_rays', 'composite_rays')})

    def xavier_init(m, gain=1, bias=0, distribution='normal'):          # mmcv.cnn.xavier_init [mmcv-memory]
        (torch.nn.init.xavier_uniform_ if distribution == 'uniform' else torch.nn.init.xavier_normal_)(m.weight, gain=gain)
        torch.nn.init.constant_(m.bias, bias)
    sys.modules['mmcv.cnn'].xavier_init = xavier_init
    sys.modules['mmcv.cnn'].constant_init = G.constant_init
    mod('matplotlib'); mod('matplotlib.pyplot')
    sys.modules['matplotlib'].pyplot = sys.modules['matplotlib.pyplot']
    for name in ('reflib.models.decoders',):
        pkg = mod(name)
        pkg.__path__ = []
    G._load('lib/models/decoders/base_volume_renderer.py', 'reflib.models.decoders.base_volume_renderer')
    return G._load('lib/models/decoders/triplane_decoder.py', 'reflib.models.decoders.triplane_decoder')


CFG = dict(P=dict(base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3], use_dir_enc=True, dir_layers=[16, 64], max_steps=256),
           S=dict(max_steps=256))


def run_reference():
    tri = load_reference_decoder()
    torch.Tensor.cuda = lambda self, *a, **k: self                  # the op wrappers move host tensors to the GPU; there is none here
    out = {}
    res = 24
    f = 131.25 * res / 128
    poses = torch.from_numpy(spiral_poses(2)).float()
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(2, 4).contiguous()
    for variant in ('P', 'S'):
        C = 6 if variant == 'P' else 32
        g = torch.Generator().manual_seed(11 if variant == 'P' else 12)
        code = (torch.randn(2, 3, C, 128, 128, generator=g) * 0.7).clamp(-2, 2)
        params = rp.make_decoder_params(variant, 4)
        params['density_net.0.bias'] = params['density_net.0.bias'] + 1.0
        dec = tri.TriPlaneDecoder(**CFG[variant])
        missing = dec.load_state_dict({k: torch.as_tensor(v) for k, v in params.items()}, strict=False)
        assert set(missing.missing_keys) <= {'aabb'} and not missing.unexpected_keys, missing
        out[f'{variant}_state_keys'] = np.array(list(dec.state_dict().keys()))
        ro, rd = rp.get_cam_rays(poses, intr, res, res)
        ro, rd = ro.reshape(2, -1, 3).contiguous(), rd.reshape(2, -1, 3).contiguous()
        bits = torch.from_numpy(np.stack([rp.sphere_bitfield(radius=0.7), rp.sphere_bitfield(radius=0.5)]))
        dt_gamma = torch.tensor([0.0, 0.004])
        out[f'{variant}_code_seed'] = np.array(11 if variant == 'P' else 12)
        # ---- point_decode on explicit points (ragged per-scene lists, as the renderer calls it)
        xyz = [(torch.rand(37, 3, generator=g) * 2 - 1), (torch.rand(50, 3, generator=g) * 2 - 1)]
        dirs = [torch.nn.functional.normalize(torch.randn(n.shape[0], 3, generator=g), dim=-1) for n in xyz]
        with torch.no_grad():
            sig, rgb, npts = dec.point_decode(xyz, dirs, code)
        out[f'{variant}_pd_xyz'], out[f'{variant}_pd_dirs'] = torch.cat(xyz).numpy(), torch.cat(dirs).numpy()
        out[f'{variant}_pd_sigma'], out[f'{variant}_pd_rgb'], out[f'{variant}_pd_counts'] = sig.numpy(), rgb.numpy(), np.array(npts)
        # ---- eval branch: the host-driven loop
        dec.eval()
        with torch.no_grad():
            r = dec(ro, rd, code, bits, 64, dt_gamma=dt_gamma, perturb=False)
        for k in ('weights_sum', 'depth', 'image'):
            out[f'{variant}_eval_{k}'] = torch.stack(r[k]).numpy()
        if variant == 'S':
            continue
        # ---- train branch + gradient w.r.t. code and decoder weights (perturb=False: start offsets 0, as guidance tests inject)
        dec.train()
        sel = torch.stack([torch.randperm(res * res, generator=g)[:200] for _ in range(2)])
        ro_t = torch.stack([ro[b][sel[b]] for b in range(2)])
        rd_t = torch.stack([rd[b][sel[b]] for b in range(2)])
        code_t = code.clone().requires_grad_(True)
        r = dec(ro_t, rd_t, code_t, bits, 64, dt_gamma=dt_gamma, perturb=False, return_loss=True)
        gi, gw = torch.randn(2, 200, 3, generator=g), torch.randn(2, 200, generator=g)
        loss = (r['image'] * gi).sum() + (r['weights_sum'] * gw).sum()
        loss.backward()
        out['P_train_sel'], out['P_train_gi'], out['P_train_gw'] = sel.numpy(), gi.numpy(), gw.numpy()
        for k in ('weights_sum', 'depth', 'image'):
            out[f'P_train_{k}'] = r[k].detach().numpy()
        out['P_train_decoder_reg_loss_is_none'] = np.array(r['decoder_reg_loss'] is None)
        out['P_train_grad_code'] = code_t.grad.numpy()
        for k, p in dec.named_parameters():
            out[f'P_train_grad_{k}'] = p.grad.numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# Train branch in the regimes where the fused differentiable renderer's edge rules act (-> reference_train_edges_v1.npz):
#   floor       density bias -22: every density logit far below ln 1e-6, so K8's gradient reaches the code only through TruncExp's floor
#   ones        all-ones occupancy grid: samples fill the whole box and reach the plane borders (grid_sample padding_mode='border')
#   plane96x160 non-square planes
#   budget32    all-ones grid at max_steps 32: the per-ray sample budget of march_rays_train binds
# `rays` per scene: the stored code gradient grows with the texels the rays touch, so the all-ones cases (about 170 samples a ray at
# max_steps 256) use few rays and the fixture stays small.
TRAIN_EDGE_CASES = dict(floor=dict(bias=-22.0, grids=('sphere0.7', 'sphere0.5'), hw=(128, 128), max_steps=256, rays=24),
                        ones=dict(bias=1.0, grids=('ones', 'ones'), hw=(128, 128), max_steps=256, rays=10),
                        plane96x160=dict(bias=1.0, grids=('sphere0.7', 'sphere0.5'), hw=(96, 160), max_steps=256, rays=24),
                        budget32=dict(bias=1.0, grids=('ones', 'ones'), hw=(128, 128), max_steps=32, rays=12))
TRAIN_EDGE_RES, TRAIN_EDGE_DT_GAMMA = 24, (0.0, 0.004)


def train_edge_inputs(name):
    """Inputs of one train-edge case (no reference needed): code [2,3,6,H,W], decoder params, rays [2,24*24,3], bitfields [2,G^3/8]."""
    c = TRAIN_EDGE_CASES[name]
    seed = 40 + sorted(TRAIN_EDGE_CASES).index(name)
    g = torch.Generator().manual_seed(seed)
    code = (torch.randn(2, 3, 6, *c['hw'], generator=g) * 0.7).clamp(-2, 2)
    params = rp.make_decoder_params('P', seed)
    params['density_net.0.bias'] = params['density_net.0.bias'] + c['bias']
    res = TRAIN_EDGE_RES
    f = 131.25 * res / 128
    poses = torch.from_numpy(spiral_poses(2)).float()
    intr = torch.tensor([f, f, res / 2, res / 2]).expand(2, 4).contiguous()
    ro, rd = rp.get_cam_rays(poses, intr, res, res)
    bits = np.stack([np.full(64 ** 3 // 8, 255, np.uint8) if gr == 'ones' else rp.sphere_bitfield(radius=float(gr[6:])) for gr in c['grids']])
    return dict(seed=seed, code=code, params=params, rays_o=ro.reshape(2, -1, 3).contiguous(), rays_d=rd.reshape(2, -1, 3).contiguous(),
                bits=bits, max_steps=c['max_steps'])


def run_reference_train_edges():
    tri = load_reference_decoder()
    torch.Tensor.cuda = lambda self, *a, **k: self
    out = {}
    for name in sorted(TRAIN_EDGE_CASES):
        inp = train_edge_inputs(name)
        g = torch.Generator().manual_seed(1000 + inp['seed'])
        dec = tri.TriPlaneDecoder(**dict(CFG['P'], max_steps=inp['max_steps']))
        missing = dec.load_state_dict({k: torch.as_tensor(v) for k, v in inp['params'].items()}, strict=False)
        assert set(missing.missing_keys) <= {'aabb'} and not missing.unexpected_keys, missing
        dec.train()
        n_all = inp['rays_o'].shape[1]
        n_rays = TRAIN_EDGE_CASES[name]['rays']
        sel = torch.stack([torch.randperm(n_all, generator=g)[:n_rays] for _ in range(2)])
        ro_t = torch.stack([inp['rays_o'][b][sel[b]] for b in range(2)])
        rd_t = torch.stack([inp['rays_d'][b][sel[b]] for b in range(2)])
        code_t = inp['code'].clone().requires_grad_(True)
        r = dec(ro_t, rd_t, code_t, torch.from_numpy(inp['bits']), 64, dt_gamma=torch.tensor(TRAIN_EDGE_DT_GAMMA), perturb=False, return_loss=True)
        gi, gw = torch.randn(2, n_rays, 3, generator=g), torch.randn(2, n_rays, generator=g)
        ((r['image'] * gi).sum() + (r['weights_sum'] * gw).sum()).backward()
        out[f'{name}_sel'], out[f'{name}_gi'], out[f'{name}_gw'] = sel.numpy().astype(np.int16), gi.numpy(), gw.numpy()
        for k in ('weights_sum', 'depth', 'image'):
            out[f'{name}_{k}'] = r[k].detach().numpy()
        gc = code_t.grad.numpy().reshape(-1)                  # sparse: only texels next to a sample receive gradient
        nz = np.nonzero(gc)[0]
        out[f'{name}_grad_code_idx_diff'], out[f'{name}_grad_code_val'] = np.diff(nz, prepend=0).astype(np.int32), gc[nz]
        for k, p in dec.named_parameters():
            out[f'{name}_grad_{k}'] = p.grad.numpy()
    return out


if __name__ == '__main__':
    if '--train-edges' in sys.argv:
        res = run_reference_train_edges()
        path = os.path.join(HERE, 'reference_train_edges_v1.npz')
    else:
        res = run_reference()
        path = os.path.join(HERE, 'reference_decoder_v1.npz')
    np.savez_compressed(path, **res)
    print({k: v.shape for k, v in res.items() if v.ndim}, os.path.getsize(path), 'bytes')
