"""CPU suite for the oracle: golden fixtures (tests/golden/oracle_v1.npz, made by make_golden.py) + domain properties."""
import math
import os

import numpy as np
import torch

import oracle as orc
from oracle import render_port as rp
from oracle import unet_port as up
from tests.common import GOLDEN, config1

G = np.load(os.path.join(GOLDEN, 'oracle_v1.npz'))


def test_golden_rays_and_aabb():
    code, poses, intr = config1('P', res=16)
    ro, rd = rp.get_cam_rays(poses[0], intr[0], 16, 16)
    np.testing.assert_allclose(ro.reshape(-1, 3).numpy(), G['rays_o'], rtol=0, atol=0)
    np.testing.assert_allclose(rd.reshape(-1, 3).numpy(), G['rays_d'], rtol=1e-6, atol=1e-7)   # torch matmul may reorder
    n, f = orc.near_far_from_aabb(G['rays_o'], G['rays_d'], np.array([-1, -1, -1, 1, 1, 1], np.float32), 0.2)
    assert np.array_equal(n.view(np.uint32), G['nears'].view(np.uint32)) and np.array_equal(f.view(np.uint32), G['fars'].view(np.uint32))
    # unit directions, near >= min_near on hits, misses flagged with FLT_MAX
    assert np.allclose(np.linalg.norm(G['rays_d'], axis=-1), 1, atol=1e-6)
    hit = n < 1e30
    assert (n[hit] >= 0.2).all() and (f[hit] >= n[hit]).all()


def test_golden_integer_trace():
    bf = rp.sphere_bitfield()
    assert int(bf.astype(np.uint64).sum()) == int(G['sphere_bitfield_crc'][0])
    tr, ts, cnt = orc.trace_rays(G['rays_o'], G['rays_d'], G['nears'], G['fars'], 1.0, bf, 1, 64, 0.0, 256, cap=64)
    assert np.array_equal(tr, G['trace']) and np.array_equal(cnt, G['trace_counts'])
    assert np.array_equal(ts.view(np.uint32), G['trace_t'].view(np.uint32))
    # every sampled voxel is occupied; t strictly increases along a ray on the near + k*dt lattice
    for i in range(tr.shape[0]):
        idx = tr[i, :cnt[i]]
        assert ((bf[idx // 8] >> (idx % 8)) & 1).all()
        assert (np.diff(ts[i, :cnt[i]]) > 0).all()
    dt = np.float32(2 * 1.7320508075688772 / 256)
    k = (ts[cnt > 1][:, 1] - ts[cnt > 1][:, 0]) / dt
    assert np.allclose(k, np.round(k), atol=1e-3)


def test_march_quanta_equal_whole_ray_trace():
    """n_step batching changes nothing: concatenating the reference's per-quantum K9 calls == one long march"""
    bf = rp.sphere_bitfield()
    ro, rd, nears, fars = G['rays_o'], G['rays_d'], G['nears'], G['fars']
    N = ro.shape[0]
    alive = np.arange(N, dtype=np.int32)
    rays_t = nears.copy()
    got = [[] for _ in range(N)]
    for n_step in (1, 2, 8, 3, 8, 8, 8, 8, 8, 8):
        xyz, dirs, deltas, vox = orc.march_rays(N, n_step, alive, rays_t, ro, rd, 1.0, bf, 1, 64, nears, fars, max_steps=256, return_voxels=True)
        for i in range(N):
            v = vox[i * n_step:(i + 1) * n_step]
            got[i] += [int(x) for x in v[v >= 0]]
            k = (deltas[i * n_step:(i + 1) * n_step, 0] != 0).sum()
            if k == n_step:
                rays_t[i] = deltas[i * n_step + n_step - 1, 1] + deltas[i * n_step + n_step - 1, 0]
            else:
                rays_t[i] = fars[i]                 # exhausted: t < far is false from now on
    for i in range(N):
        want = [int(x) for x in G['trace'][i, :G['trace_counts'][i]]]
        assert got[i][:len(want)] == want[:len(got[i])] and len(got[i]) >= min(len(want), 62)


def test_morton_packbits_sh():
    assert np.array_equal(orc.morton3D(G['morton_coords']), G['morton_idx'])
    assert np.array_equal(orc.morton3D_invert(G['morton_idx']), G['morton_coords'])
    c = G['morton_coords'].astype(np.int64)
    manual = np.zeros(len(c), np.int64)
    for b in range(10):
        manual |= ((c[:, 0] >> b) & 1) << (3 * b) | ((c[:, 1] >> b) & 1) << (3 * b + 1) | ((c[:, 2] >> b) & 1) << (3 * b + 2)
    assert np.array_equal(manual, G['morton_idx'])
    g = np.random.RandomState(0).rand(4096).astype(np.float32)
    assert np.array_equal(orc.packbits(g, 0.5), np.packbits(g > 0.5, bitorder='little'))
    np.testing.assert_allclose(orc.sh_encode(G['sh_dirs'], 4), G['sh_out'], rtol=0, atol=0)
    # SH16 is orthonormal-ish under the sphere measure: band-0 constant, band-1 linear in (y, z, x)
    assert np.allclose(G['sh_out'][:, 0], 0.28209479)
    np.testing.assert_allclose(G['sh_out'][:, 1], -0.48860251 * G['sh_dirs'][:, 1], rtol=1e-6)


def test_golden_render_and_compositing_properties():
    code, poses, intr = config1('P', res=16)
    params = rp.make_decoder_params('P', 0)
    ref = rp.render_eval_scene(params, G['rays_o'], G['rays_d'], code[0], rp.sphere_bitfield(), max_steps=256)
    np.testing.assert_allclose(ref['image'], G['render_image'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ref['weights_sum'], G['render_ws'], rtol=1e-5, atol=1e-6)
    assert (ref['weights_sum'] <= 1 + 1e-6).all() and (ref['weights_sum'] >= 0).all()
    assert (ref['image'] <= ref['weights_sum'][:, None] * 1.002 + 1e-5).all()       # rgb in [-.001, 1.001]
    miss = G['nears'] > 1e30
    assert (ref['weights_sum'][miss] == 0).all()
    # train compositor == eval compositor while no ray terminates early, and its backward matches finite differences
    rng = np.random.RandomState(1)
    M, Nr = 40, 5
    sig, rgb = rng.rand(M).astype(np.float32) * 3, rng.rand(M, 3).astype(np.float32)
    deltas = np.stack([np.full(M, 0.0135, np.float32), np.cumsum(np.full(M, 0.0135, np.float32))], -1)
    rays = np.array([[i, 8 * i, 8] for i in range(Nr)], np.int32)
    ws, dep, img = orc.composite_rays_train_forward(sig, rgb, deltas, rays, 1e-4)
    gs, gc = orc.composite_rays_train_backward(np.ones(Nr, np.float32), np.ones((Nr, 3), np.float32), sig, rgb, deltas, rays, ws, img, 1e-4)
    eps = 1e-2
    for j in (0, 9, 23):
        sp, sm = sig.copy(), sig.copy()
        sp[j] += eps; sm[j] -= eps
        fp = sum(x.sum() for x in (lambda o: (o[0], o[2]))(orc.composite_rays_train_forward(sp, rgb, deltas, rays, 1e-4)))
        fm = sum(x.sum() for x in (lambda o: (o[0], o[2]))(orc.composite_rays_train_forward(sm, rgb, deltas, rays, 1e-4)))
        assert abs((fp - fm) / (2 * eps) - gs[j]) < 2e-3


def test_golden_unet_and_ddim_tables():
    small = up.unet_spec(image_size=16, in_channels=18, base_channels=64, channels_cfg=(1, 2), resblocks_per_downsample=1,
                         attention_res=(8,), num_heads=2)
    sd = up.random_state_dict(small, seed=0, std=0.04)
    y = up.unet_forward(sd, small, torch.from_numpy(G['unet_x']), torch.tensor([500]))
    np.testing.assert_allclose(y.numpy(), G['unet_y'], rtol=1e-4, atol=1e-5)
    dv = up.diffusion_vars(up.linear_betas())
    np.testing.assert_array_equal(dv['alphas_bar'][up.ddim_timesteps(1000, 50).numpy()], G['alphas_bar_50'])
    # a perfect denoiser (v consistent with a fixed x0) makes DDIM return that x0 (clip range wide)
    x0 = torch.randn(1, 18, 8, 8, generator=torch.Generator().manual_seed(0)).clamp(-1.5, 1.5)

    def oracle_v(x_t, t):
        sa = torch.tensor(dv['sqrt_alphas_bar'], dtype=torch.float32)[t].reshape(-1, 1, 1, 1)
        s1 = torch.tensor(dv['sqrt_one_minus_alphas_bar'], dtype=torch.float32)[t].reshape(-1, 1, 1, 1)
        return (sa * x_t - x0) / s1
    out = up.ddim_sample(oracle_v, torch.randn(1, 18, 8, 8, generator=torch.Generator().manual_seed(1)), dv, num_timesteps=50)
    np.testing.assert_allclose(out.numpy(), x0.numpy(), atol=2e-4)


# ----------------------------------------------------------------------------- differentiable (train / guidance) branch
def _train_case(n_rays=48, res=12, seed=3):
    from oracle import train_port as tp
    code, poses, intr = config1('P', seed=seed, res=res)
    ro, rd = rp.get_cam_rays(poses[0], intr[0], res, res)
    sel = np.linspace(0, res * res - 1, n_rays).astype(np.int64)       # spread over the image so most rays hit the sphere
    ro, rd = ro.reshape(-1, 3).numpy()[sel], rd.reshape(-1, 3).numpy()[sel]
    params = rp.make_decoder_params('P', seed=seed)
    bf = rp.sphere_bitfield()
    rng = np.random.default_rng(seed)
    return tp, code[0] * 0.5, ro, rd, params, bf, rng.random(ro.shape[0]).astype(np.float32)


def test_train_autograd_equals_k8_analytic_backward():
    """torch autograd through the restated K7 forward == the C restatement of K8 (raymarching.cu:606-687) on the same samples,
    including K8's rule that the sample at which T drops below T_thresh gets no gradient."""
    tp, code, ro, rd, params, bf, noises = _train_case()
    T_thresh = 0.3                                   # high threshold so many rays actually break early
    aabb = np.array([-1, -1, -1, 1, 1, 1], np.float32)
    nears, fars = orc.near_far_from_aabb(ro, rd, aabb, 0.2)
    xyzs, dirs, deltas, rays = orc.march_rays_train(ro, rd, 1.0, bf, 1, 64, nears, fars, max_steps=256, noises=noises)
    m = int(rays[:, 2].sum())
    sig, rgb = rp.point_decode(params, torch.from_numpy(xyzs[:m]), torch.from_numpy(dirs[:m]), code)
    sig = (sig * 6).detach().numpy().astype(np.float32); rgb = rgb.detach().numpy().astype(np.float32)
    ws, depth, img = orc.composite_rays_train_forward(sig, rgb, deltas[:m], rays, T_thresh)
    rng = np.random.default_rng(0)
    g_ws, g_img = rng.standard_normal(ws.shape).astype(np.float32), rng.standard_normal(img.shape).astype(np.float32)
    gs, gc = orc.composite_rays_train_backward(g_ws, g_img, sig, rgb, deltas[:m], rays, ws, img, T_thresh)
    # the same composite in torch (float64) with the crossing-sample detach
    st = torch.from_numpy(sig).double().requires_grad_(True); ct = torch.from_numpy(rgb).double().requires_grad_(True)
    tot = 0
    n_broke = 0
    for r in range(rays.shape[0]):
        off, cnt = int(rays[r, 1]), int(rays[r, 2])
        T = torch.ones((), dtype=torch.float64); w_sum = 0; im = 0
        for s in range(cnt):
            k = off + s
            crossing = float((T * torch.exp(-st[k] * float(deltas[k, 0]))).detach()) < T_thresh
            sk, ck = (st[k].detach(), ct[k].detach()) if crossing else (st[k], ct[k])
            a = 1 - torch.exp(-sk * float(deltas[k, 0]))
            w = a * T
            w_sum = w_sum + w; im = im + w * ck
            T = T * (1 - a)
            if crossing:
                n_broke += 1
                break
        tot = tot + w_sum * float(g_ws[r]) + (im * torch.from_numpy(g_img[r]).double()).sum() if cnt else tot
    g_s, g_c = torch.autograd.grad(tot, [st, ct])
    assert n_broke > 5
    np.testing.assert_allclose(g_s.numpy(), gs, rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(g_c.numpy(), gc, rtol=2e-4, atol=2e-5)


def test_train_render_gradient_finite_differences():
    """d loss / d code of the restated loss chain vs central differences (float64)"""
    tp, code, ro, rd, params, bf, noises = _train_case(n_rays=24)
    rng = np.random.default_rng(1)
    target = rng.random((1, ro.shape[0], 3)).astype(np.float32)
    kw = dict(noises=noises[None], bg_color=1.0, pixel_weight=20.0, loss_coef=0.1 / 144, scale_num_ray=ro.shape[0], reg_weight=3e-3)
    code = code[None].double()
    loss, grad, out = tp.render_loss_grad(params, code, ro[None], rd[None], target, [bf], **kw)
    assert float(loss) > 0 and float(grad.abs().max()) > 0
    # a gradient clamped by TruncExp's floor is not a derivative: every sample that passes gradient must sit above the floor
    *_, smp = tp.render_train_scene(params, code[0], ro, rd, bf, noises, return_samples=True)
    _, _, logit = rp.point_preacts(params, torch.from_numpy(smp['xyzs']), torch.from_numpy(smp['dirs']), code[0], dtype=torch.float64)
    assert smp['grad_mask'].sum() > 100 and float(logit[torch.from_numpy(smp['grad_mask'])].min()) > math.log(1e-6) + 1
    flat = grad.reshape(-1)
    idx = torch.argsort(flat.abs(), descending=True)[:6]
    eps = 1e-5
    for i in idx.tolist():
        d = torch.zeros_like(code).reshape(-1); d[i] = eps; d = d.reshape(code.shape)
        lp, _ = tp.render_loss(params, code + d, ro[None], rd[None], target, [bf], **kw)
        lm, _ = tp.render_loss(params, code - d, ro[None], rd[None], target, [bf], **kw)
        fd = float(lp - lm) / (2 * eps)
        assert abs(fd - float(flat[i])) <= 1e-5 * max(1.0, abs(fd)) + 2e-3 * abs(fd), (i, fd, float(flat[i]))


def test_golden_train_branch():
    """regression pin of the train / guidance-branch oracle: tests/golden/oracle_train_v1.npz (made by make_golden_train.py)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_golden_train', os.path.join(GOLDEN, 'make_golden_train.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    T = np.load(os.path.join(GOLDEN, 'oracle_train_v1.npz'))
    out = mod.compute()
    assert np.array_equal(out['march_rays'], T['march_rays'])                                    # integer (ray, offset, count) triples: exact
    assert np.array_equal(out['march_deltas_head'].view(np.uint32), T['march_deltas_head'].view(np.uint32))
    for k in ('ws', 'depth', 'image', 'out_rgb'):
        np.testing.assert_allclose(out[k], T[k], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(out['loss'], T['loss'], rtol=1e-10)
    assert np.array_equal(out['grad_top_idx'][:8], T['grad_top_idx'][:8])
    np.testing.assert_allclose(out['grad_top_val'], T['grad_top_val'], rtol=1e-7, atol=1e-12)
    np.testing.assert_allclose(out['grad_abs_sum_per_plane'], T['grad_abs_sum_per_plane'], rtol=1e-8)
    # domain properties: early-terminated rays exist at this threshold, weights are a sub-probability, blended colour stays in range
    assert (T['ws'] > 0).sum() >= 5 and T['ws'].max() <= 1 + 1e-9 and T['out_rgb'].min() >= -0.01 and T['out_rgb'].max() <= 1.01
