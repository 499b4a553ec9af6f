"""The fused differentiable renderer (k_render_train_p<BWD, WG> in csrc/render_train.cu: forward, gradient w.r.t. the code and, with a
trainable decoder, w.r.t. the decoder weights) where stage-1 training, single-stage training and guidance take it, against the CPU oracle
of the reference's train branch (oracle/train_port.py):

  * TruncExp's gradient floor: density logits below -20, so the density path reaches the code only through the 1e-6 floor;
  * plane borders: an all-ones occupancy grid puts samples within half a texel of every plane edge;
  * non-square, odd plane sizes;
  * a binding sample budget (max_steps 32);
  * many 32-ray tiles per warp with a ragged ray count (the per-warp weight-gradient partials carried across tiles);
  * NULL noises and NULL grad_ws;
  * the fused MSE render loss (k_mse_render_loss) on ray counts that are not a multiple of its block.

Every render case runs with a frozen decoder (code gradient only) and a trainable one (WG).  Bars as in tests/test_train_render_gpu.py:
forward within TOL_P of the float32 oracle, per-ray sample counts exact, code gradient and each decoder-parameter gradient within relative
L2 1e-3 of the float64 oracle, code gradient within 1e-4 of the per-op composition.  The preconditions that make each case meaningful need
only the oracle and run without a GPU."""
import functools

import numpy as np
import pytest
import torch

from oracle import render_port as rp
from oracle import train_port as tp
from tests.common import spiral_poses
from tests.per_op_train import per_op_train_render
from tests.test_render_config_gpu import random_rays
from tests.test_train_render_gpu import TOL_P, _rel_l2

PARAMS = ('base_net.0.weight', 'base_net.0.bias', 'density_net.0.weight', 'density_net.0.bias',
          'dir_net.0.weight', 'dir_net.0.bias', 'color_net.0.weight', 'color_net.0.bias')

# name: density bias offset, occupancy grids of the two scenes, plane size, max_steps, NULL noises, NULL grad_ws
CASES = dict(floor=(-22.0, ('sphere', 'sphere0.45'), (128, 128), 256, False, False),
             ones256=(1.5, ('ones', 'ones'), (128, 128), 256, False, False),
             ones32=(1.5, ('ones', 'ones'), (128, 128), 32, False, False),
             plane96x160=(1.5, ('sphere', 'sphere0.45'), (96, 160), 256, False, False),
             plane97x131=(1.5, ('sphere', 'sphere0.45'), (97, 131), 256, False, False),
             no_noises=(1.5, ('sphere', 'sphere0.45'), (128, 128), 256, True, False),
             no_grad_ws=(1.5, ('sphere', 'sphere0.45'), (128, 128), 256, False, True))


def _bitfield(name):
    if name == 'ones':
        return np.full(64 ** 3 // 8, 255, np.uint8)
    return rp.sphere_bitfield(radius=float(name[6:] or 0.6))


@functools.lru_cache(maxsize=None)
def _case(name, n_rays=512, seed=7, res=32):
    """_case() of tests/test_train_render_gpu.py with the named change; the float32 oracle (forward, counts, samples) and the float64
    oracle's gradients w.r.t. the code and every decoder parameter of sum(image * g_img + weights_sum * g_ws)"""
    bias, grids, hw, max_steps, no_noises, no_grad_ws = CASES[name]
    B = 2
    g = torch.Generator().manual_seed(seed)
    code = (torch.randn(B, 3, 6, *hw, generator=g) * 0.7).clamp(-2, 2)
    poses = torch.from_numpy(spiral_poses(B))
    f = 131.25 * res / 128
    intr = torch.tensor([f, f, res / 2, res / 2])
    ros, rds = [], []
    for b in range(B):
        ro, rd = rp.get_cam_rays(poses[b], intr, res, res)
        sel = torch.randperm(res * res, generator=g)[:n_rays]
        ros.append(ro.reshape(-1, 3)[sel]); rds.append(rd.reshape(-1, 3)[sel])
    rays_o, rays_d = torch.stack(ros), torch.stack(rds)
    params = rp.make_decoder_params('P', seed)
    params['density_net.0.bias'] = params['density_net.0.bias'] + bias
    bf = np.stack([_bitfield(gr) for gr in grids])
    noises = None if no_noises else torch.rand(B, n_rays, generator=g)
    dt_gamma = torch.tensor([0.0, 0.004])
    g_img = torch.randn(B, n_rays, 3, generator=g)
    g_ws = None if no_grad_ws else torch.randn(B, n_rays, generator=g)
    kw = [dict(noises=None if noises is None else noises[b].numpy(), dt_gamma=float(dt_gamma[b]), max_steps=max_steps) for b in range(B)]
    r32 = [tp.render_train_scene(params, code[b], rays_o[b].numpy(), rays_d[b].numpy(), bf[b], dtype=torch.float32, return_samples=True, **kw[b])
           for b in range(B)]
    pref = {k: torch.as_tensor(v).double().requires_grad_(True) for k, v in params.items()}
    cref = code.double().requires_grad_(True)
    tot = 0
    for b in range(B):
        ws, _, img = tp.render_train_scene(pref, cref[b], rays_o[b].numpy(), rays_d[b].numpy(), bf[b], **kw[b])
        tot = tot + (img * g_img[b].double()).sum() + (0 if g_ws is None else (ws * g_ws[b].double()).sum())
    grads = dict(zip(('code',) + PARAMS, torch.autograd.grad(tot, [cref] + [pref[k] for k in PARAMS])))
    return dict(code=code, rays_o=rays_o, rays_d=rays_d, params=params, bf=bf, noises=noises, dt_gamma=dt_gamma, max_steps=max_steps,
                g_img=g_img, g_ws=g_ws, r32=r32, grads=grads)


def _ring(hw):
    """mask [H, W] of the outer ring of texels of a plane"""
    m = torch.zeros(hw, dtype=torch.bool)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    return m


# ============================================================================================ preconditions (CPU, oracle only)
def test_floor_case_is_below_the_floor():
    """every sample that receives gradient has a density logit below -20 (float32 alpha exactly 0, the floor alone drives the density
    path), and plain exp's gradient misses TruncExp's by more than 0.5 relative on density_net.0.bias"""
    c = _case('floor')
    n_grad = 0
    for b in range(2):
        smp = c['r32'][b][3]
        _, _, logit = rp.point_preacts(c['params'], torch.from_numpy(smp['xyzs']), torch.from_numpy(smp['dirs']), c['code'][b], dtype=torch.float64)
        lg = logit[torch.from_numpy(smp['grad_mask'])]
        assert float(lg.max()) < -20.0, float(lg.max())
        n_grad += lg.numel()
        assert float(c['r32'][b][0].abs().max()) == 0.0
    assert n_grad > 1000
    pref = {k: torch.as_tensor(v).double().requires_grad_(True) for k, v in c['params'].items()}
    tot = 0
    for b in range(2):
        ws, _, img = tp.render_train_scene(pref, c['code'][b].double(), c['rays_o'][b].numpy(), c['rays_d'][b].numpy(), c['bf'][b],
                                           c['noises'][b].numpy(), dt_gamma=float(c['dt_gamma'][b]), trunc_exp=False)
        tot = tot + (img * c['g_img'][b].double()).sum() + (ws * c['g_ws'][b].double()).sum()
    k = 'density_net.0.bias'
    g_exp, = torch.autograd.grad(tot, [pref[k]])
    assert _rel_l2(g_exp, c['grads'][k]) > 0.5, _rel_l2(g_exp, c['grads'][k])


@pytest.mark.parametrize('name', ['ones256', 'ones32'])
def test_border_case_reaches_the_borders(name):
    """at least 1 % of the samples lie within half a texel of a plane edge (where grid_sample's border padding clamps), and every plane of
    every scene has outer-ring texels that receive gradient"""
    c = _case(name)
    H, W = c['code'].shape[-2:]
    near = []
    for b in range(2):
        x = c['r32'][b][3]['xyzs']
        near.append((np.abs(x) > 1 - 1 / min(H, W)).any(axis=1))
    assert np.concatenate(near).mean() >= 0.01, np.concatenate(near).mean()
    ring = _ring((H, W))
    gc = c['grads']['code']                                                  # [B, 3, 6, H, W]
    for b in range(2):
        for pl in range(3):
            assert int((gc[b, pl][:, ring] != 0).sum()) > 0, (b, pl)


def test_budget_case_binds():
    """at max_steps 32 on the all-ones grid at least 25 % of the rays stop on the sample budget"""
    c = _case('ones32')
    counts = np.concatenate([r[3]['counts'] for r in c['r32']])
    assert (counts == 32).mean() >= 0.25, (counts == 32).mean()
    assert (counts < 32).any()


# ============================================================================================ GPU: the cases against the oracle
def _gpu_run(cuda, c, want_wg):
    from ssdnerf_b200 import renderer as R
    hw = tuple(c['code'].shape[-2:])
    blob = R.pack_decoder_blob(c['params'], R.DEC_P, device=cuda)
    planes = R.pack_planes(c['code'].to(cuda), R.DEC_P)
    bft = torch.from_numpy(c['bf']).to(cuda)
    noises = None if c['noises'] is None else c['noises'].to(cuda)
    kw = dict(noises=noises, dt_gamma=c['dt_gamma'].to(cuda), max_steps=c['max_steps'])
    out = R.render_train_fwd(planes, hw, bft, blob, c['rays_o'].to(cuda), c['rays_d'].to(cuda), want_counts=True, **kw)
    g_ws = None if c['g_ws'] is None else c['g_ws'].to(cuda)
    res = R.render_train_bwd(planes, hw, bft, blob, c['rays_o'].to(cuda), c['rays_d'].to(cuda), out['weights_sum'], out['image'], g_ws,
                             c['g_img'].to(cuda), want_decoder_grad=want_wg, **kw)
    if want_wg:
        gcode, gblob = res
        gparams = dict(zip(R.DEC_P_PARAM_ORDER, (g.cpu() for g in R.unpack_decoder_blob_grad(gblob))))
    else:
        gcode, gparams = res, None
    return {k: v.cpu() for k, v in out.items()}, gcode.cpu(), gparams


@pytest.mark.gpu
@pytest.mark.parametrize('wg', [False, True], ids=['frozen', 'wg'])
@pytest.mark.parametrize('name', list(CASES))
def test_train_render_case(cuda, name, wg):
    c = _case(name)
    out, gcode, gparams = _gpu_run(cuda, c, wg)
    # forward and per-ray sample counts
    for b in range(2):
        ws, dep, img, smp = c['r32'][b]
        counts = out['num_samples'][b].numpy()
        assert np.array_equal(counts, smp['counts']), (b, int((counts != smp['counts']).sum()))
        np.testing.assert_allclose(out['weights_sum'][b].numpy(), ws.numpy(), **TOL_P)
        np.testing.assert_allclose(out['image'][b].numpy(), img.numpy(), **TOL_P)
        np.testing.assert_allclose(out['depth'][b].numpy(), dep.numpy(), rtol=2e-4, atol=1e-4)
    # code gradient against float64
    ref = c['grads']
    assert float(ref['code'].abs().max()) > 0
    err = _rel_l2(gcode, ref['code'])
    assert err < 1e-3, err
    if name.startswith('ones'):                                             # the plane borders on their own
        ring = _ring(tuple(c['code'].shape[-2:]))
        err = _rel_l2(gcode[..., ring], ref['code'][..., ring])
        assert err < 1e-3, ('ring', err)
    # decoder-parameter gradients against float64
    if wg:
        for k in PARAMS:
            assert gparams[k].shape == ref[k].shape, k
            if name == 'floor' and k.startswith(('color_net', 'dir_net')):
                # only float32-quantised terms reach the colour branch here: about 1/5000 of the density weight gradient in float64, 0 in fp32
                bound = 1e-3 * float(ref['density_net.0.weight'].norm())
                assert float(gparams[k].norm()) < bound, (k, float(gparams[k].norm()), bound)
                continue
            err = _rel_l2(gparams[k], ref[k])
            assert err < 1e-3, (k, err)
    # per-op composition (the reference's own march / composite kernels around a torch decode with the reference's trunc_exp)
    B, n = c['rays_o'].shape[:2]
    cc = c['code'].to(cuda).requires_grad_(True)
    noises = torch.zeros(B, n) if c['noises'] is None else c['noises']
    po = per_op_train_render(c['params'], c['rays_o'].to(cuda), c['rays_d'].to(cuda), cc, torch.from_numpy(c['bf']).to(cuda),
                             c['dt_gamma'].tolist(), noises.to(cuda), max_steps=c['max_steps'])
    loss = (po['image'] * c['g_img'].to(cuda)).sum() + (0 if c['g_ws'] is None else (po['weights_sum'] * c['g_ws'].to(cuda)).sum())
    gpo, = torch.autograd.grad(loss, cc)
    err = _rel_l2(gcode, gpo)
    assert err < 1e-4, ('per-op', err)


# ============================================================================================ GPU: many tiles per warp, ragged
@pytest.mark.gpu
def test_weight_gradient_many_tiles_per_warp(cuda):
    """B = 4 scenes of a ragged ray count, at least 3 x 32 rays x 4 warps per SM in all, so the WG kernel's warps (1 CTA of 4 warps per
    SM) each take several tiles and carry their weight-gradient partials across them.  Every ray contributes independently, so:
      1. the full launch's code and decoder-weight gradients equal the sum of launches over chunks of <= 1024 rays (fp32 order only);
      2. the chunks' forward outputs are bitwise those of the full launch;
      3. one ragged chunk of 1000 rays matches the float64 oracle with WG."""
    from ssdnerf_b200 import renderer as R
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    B, n = 4, 3 * 32 * sms + 13
    assert n % 32 and B * n >= 3 * 32 * 4 * sms
    g = torch.Generator().manual_seed(9)
    code = (torch.randn(B, 3, 6, 128, 128, generator=g) * 0.7).clamp(-2, 2)
    params = rp.make_decoder_params('P', 9)
    params['density_net.0.bias'] = params['density_net.0.bias'] + 1.5
    rays = [random_rays(n, 100 + b) for b in range(B)]
    rays_o = torch.from_numpy(np.stack([r[0] for r in rays]))
    rays_d = torch.from_numpy(np.stack([r[1] for r in rays]))
    bf = np.stack([_bitfield(gr) for gr in ('sphere', 'sphere0.45', 'ones', 'sphere0.8')])
    noises = torch.rand(B, n, generator=g)
    dt_gamma = torch.tensor([0.0, 0.004, 0.0076, 0.0])
    g_img, g_ws = torch.randn(B, n, 3, generator=g), torch.randn(B, n, generator=g)
    blob = R.pack_decoder_blob(params, R.DEC_P, device=cuda)
    planes = R.pack_planes(code.to(cuda), R.DEC_P)
    bft = torch.from_numpy(bf).to(cuda)

    def launch(s, e, scenes=slice(None)):
        kw = dict(noises=noises[scenes, s:e].to(cuda), dt_gamma=dt_gamma[scenes].to(cuda))
        pl = planes if scenes == slice(None) else R.pack_planes(code[scenes].to(cuda), R.DEC_P)
        ro, rd = rays_o[scenes, s:e].to(cuda), rays_d[scenes, s:e].to(cuda)
        out = R.render_train_fwd(pl, (128, 128), bft[scenes], blob, ro, rd, want_counts=True, **kw)
        gc, gb = R.render_train_bwd(pl, (128, 128), bft[scenes], blob, ro, rd, out['weights_sum'], out['image'], g_ws[scenes, s:e].to(cuda),
                                    g_img[scenes, s:e].to(cuda), want_decoder_grad=True, **kw)
        return out, gc, gb

    full, gc_full, gb_full = launch(0, n)
    gc_sum, gb_sum = torch.zeros_like(gc_full), torch.zeros_like(gb_full)
    for s in range(0, n, 256):
        e = min(s + 256, n)
        out, gc, gb = launch(s, e)
        for k in ('weights_sum', 'depth', 'image', 'num_samples'):
            assert torch.equal(out[k], full[k][:, s:e]), (k, s)
        gc_sum += gc
        gb_sum += gb
    assert int(full['num_samples'].sum()) > 50 * B * n              # tens of samples per ray: every tile does real work
    err_c, err_b = _rel_l2(gc_full, gc_sum), _rel_l2(gb_full, gb_sum)
    assert err_c < 1e-5 and err_b < 1e-5, (err_c, err_b)
    # one ragged chunk against the float64 oracle
    m = 1000
    _, gc, gb = launch(0, m, slice(0, 1))
    pref = {k: torch.as_tensor(v).double().requires_grad_(True) for k, v in params.items()}
    cref = code[0].double().requires_grad_(True)
    ws, _, img = tp.render_train_scene(pref, cref, rays_o[0, :m].numpy(), rays_d[0, :m].numpy(), bf[0], noises[0, :m].numpy(), dt_gamma=0.0)
    tot = (img * g_img[0, :m].double()).sum() + (ws * g_ws[0, :m].double()).sum()
    ref = torch.autograd.grad(tot, [cref] + [pref[k] for k in PARAMS])
    assert _rel_l2(gc[0], ref[0]) < 1e-3, _rel_l2(gc[0], ref[0])
    for k, got, want in zip(PARAMS, R.unpack_decoder_blob_grad(gb), ref[1:]):
        assert _rel_l2(got, want) < 1e-3, (k, _rel_l2(got, want))


# ============================================================================================ GPU: fused MSE render loss
@pytest.mark.gpu
@pytest.mark.parametrize('bg', [0.0, 0.25, 1.0])
@pytest.mark.parametrize('rays', [1000, 4097])
def test_mse_render_loss(cuda, rays, bg):
    """loss, grad_image, grad_ws and out_rgb of k_mse_render_loss against float64, on ray counts whose last 256-thread block is partial
    (1000: its last warp holds 8 rays; 4097: one ray)"""
    from ssdnerf_b200 import renderer as R
    g = torch.Generator().manual_seed(rays)
    image = torch.rand(1, rays, 3, generator=g)
    ws = torch.rand(1, rays, generator=g)
    target = torch.rand(1, rays, 3, generator=g)
    coef_loss, coef_grad = 0.37, 1.3
    loss, g_image, g_ws, out_rgb = R.mse_render_loss(image.to(cuda), ws.to(cuda), target.to(cuda), bg, coef_loss, coef_grad, want_rgb=True)
    o = image.double() + bg * (1 - ws.double()[..., None])
    d = o - target.double()
    want_loss = coef_loss * float((d ** 2).sum())
    want_gi = coef_grad * d
    want_gws = -bg * want_gi.sum(-1)
    assert abs(float(loss) - want_loss) <= 1e-5 * want_loss, (float(loss), want_loss)
    np.testing.assert_allclose(out_rgb.cpu().double().numpy(), o.numpy(), rtol=0, atol=3e-7)
    np.testing.assert_allclose(g_image.cpu().double().numpy(), want_gi.numpy(), rtol=0, atol=1e-6)
    np.testing.assert_allclose(g_ws.cpu().double().numpy(), want_gws.numpy(), rtol=0, atol=3e-6)
