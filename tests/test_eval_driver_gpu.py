"""`python -m ssdnerf_b200.test` on the GPU: a synthetic ShapeNet SRN tree (PNG views from `viz.encode_png`, pose and intrinsics text),
config files built from the shipped cars configs (tests/golden/reference_configs.json) and checkpoints saved in mmcv's layout.  The
driver's log_vars agree with a hand-written loop over `collate` + `val_step` with the same seed (to the device's run-to-run
round-off), for an unconditional and a `guide_optim` entry; `viz_dir` files appear for batches `i % viz_step == 0` only; the eval log is appended next to the checkpoint; `evaluate_3d`
feeds FIDKID exactly as feeding it by hand does; a checkpoint with extra and missing keys loads and lists both."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
RES = 32


def write_srn_tree(root, num_scenes, views, res, seed=0, distinct=None, device='cuda'):
    """ShapeNet SRN layout under root: <scene>/rgb/<view>.png, <scene>/pose/<view>.txt, <scene>/intrinsics.txt.  With `distinct`,
    only that many scenes are written and the others are symbolic links to them (same files, other scene names)."""
    from ssdnerf_b200 import viz
    from tests.common import spiral_poses
    os.makedirs(root, exist_ok=True)
    g = torch.Generator().manual_seed(seed)
    poses = spiral_poses(views, radius=1.3, seed=seed)
    f = 131.25 * res / 128
    names = [f'{i:032x}' for i in range(num_scenes)]
    real = num_scenes if distinct is None else distinct
    for s, name in enumerate(names):
        d = os.path.join(root, name)
        if s >= real:
            os.symlink(os.path.join(root, names[s % real]), d)
            continue
        os.makedirs(os.path.join(d, 'rgb'))
        os.makedirs(os.path.join(d, 'pose'))
        with open(os.path.join(d, 'intrinsics.txt'), 'w') as fh:
            fh.write(f'{f} {res / 2} {res / 2} 0.\n0. 0. 0.\n1.\n{res} {res}\n')
        # smooth colours: a low-resolution random image upsampled, as renders are
        low = torch.rand(views, 3, 4, 4, generator=g)
        imgs = torch.nn.functional.interpolate(low, size=(res, res), mode='bilinear', align_corners=False)
        files = viz.encode_png(pred=imgs.permute(0, 2, 3, 1).contiguous().to(device))
        for v in range(views):
            with open(os.path.join(d, 'rgb', f'{v:06d}.png'), 'wb') as fh:
                fh.write(files[v])
            np.savetxt(os.path.join(d, 'pose', f'{v:06d}.txt'), poses[v].reshape(1, 16), fmt='%.9g', delimiter=' ')
    return names


def _ref_cfg(name):
    return json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))[f'configs/paper_cfgs/{name}.py']


def write_config(path, name, tree, test_over, evaluation, samples_per_gpu):
    """a config file: the shipped config's model / train_cfg / test_cfg (test_cfg updated by test_over) with data sections over tree"""
    c = _ref_cfg(name)
    data = dict(samples_per_gpu=samples_per_gpu, workers_per_gpu=1,
                val_uncond=dict(type='ShapeNetSRN', data_prefix=tree, load_imgs=False, num_test_imgs=3, scene_id_as_name=True),
                val_cond=dict(type='ShapeNetSRN', data_prefix=tree, specific_observation_idcs=[0]))
    with open(path, 'w') as f:
        f.write(f'model = {c["model"]!r}\ntrain_cfg = {c["train_cfg"]!r}\ntest_cfg = {dict(c["test_cfg"], **test_over)!r}\n'
                f'data = {data!r}\nevaluation = {evaluation!r}\n')


def _state_dict(name, test_over):
    """the cars model's state dict with a seeded random denoiser (both the trained and the EMA copy)"""
    import ssdnerf_b200 as S
    from oracle import unet_port as up
    c = _ref_cfg(name)
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=dict(c['test_cfg'], **test_over))
    sd = up.random_state_dict(up.unet_spec(), seed=7, std=0.02)
    for diff in (model.diffusion, model.diffusion_ema):
        # the recons configs' ResBlocks hold a dropout layer before their second convolution, which shifts its index
        own = diff.denoising.state_dict()
        diff.denoising.load_state_dict({k if k in own else k.replace('.conv_2.1.', '.conv_2.2.'): v for k, v in sd.items()}, strict=True)
    return model.state_dict()


def _hand_loop(cfg_path, ckpt_sd, data_name, viz_dir=None, viz_step=1, seed=2021):
    """what the driver does, written out: seed, build, load, then collate + val_step per batch and the weighted average"""
    import ssdnerf_b200 as S
    from ssdnerf_b200.config import Config
    from ssdnerf_b200.test import set_random_seed
    cfg = Config.fromfile(cfg_path)
    set_random_seed(seed)
    model = S.build_model(cfg['model'], train_cfg=cfg['train_cfg'], test_cfg=cfg['test_cfg'])
    model.load_state_dict(ckpt_sd)
    model = model.cuda().eval()
    ds = S.build_dataset(cfg['data'][data_name])
    spg = cfg['data']['samples_per_gpu']
    logs, weights = {}, []
    for i, lo in enumerate(range(0, len(ds), spg)):
        data = S.collate([ds[j] for j in range(lo, min(lo + spg, len(ds)))], 'cuda')
        kw = dict(viz_dir=viz_dir) if viz_dir is not None and i % viz_step == 0 else {}
        out = model.val_step(data, show_pbar=True, **kw)
        for k, v in out['log_vars'].items():
            logs.setdefault(k, []).append(v)
        weights.append(out['num_samples'])
    return {k: np.average(v, weights=weights) for k, v in logs.items()}


def _check_equal(got, want):
    assert set(got) == set(want) and want, (got, want)
    for k in want:
        # the same seed and inputs, but two runs of sampling + occupancy grid + render are not bit-identical on the device: on an
        # H100 the driver and the hand loop differed by 2.6e-5 in the PSNR and 9.6e-6 in the SSIM.  A different noise draw or batch
        # order moves both by orders of magnitude more.
        print(f'{k}: driver {got[k]!r} hand {want[k]!r} diff {abs(got[k] - want[k]):.3g}')
        assert abs(got[k] - want[k]) <= 1e-4 * max(1.0, abs(want[k])), (k, got[k], want[k])


def test_unconditional_entry(cuda, tmp_path):
    from ssdnerf_b200 import test as T
    from ssdnerf_b200.inception_stat import write_stats
    tree = str(tmp_path / 'tree')
    write_srn_tree(tree, 5, 3, RES)
    over = dict(num_timesteps=2, img_size=[RES, RES])
    pkl = str(tmp_path / 'stats.pkl')
    write_stats(np.random.default_rng(0).random((6, 3), dtype=np.float32), pkl)
    viz = str(tmp_path / 'viz_uncond')
    metric = dict(type='FIDKID', num_images=6, num_subsets=2, max_subset_size=4, inception_pkl=pkl, bgr2rgb=False)
    cfg_path = str(tmp_path / 'uncond.py')
    write_config(cfg_path, 'ssdnerf_cars_uncond', tree, over,
                 [dict(type='GenerativeEvalHook3D', data='val_uncond', feed_batch_size=4, viz_dir=viz, viz_step=2, metrics=metric)], 8)
    # the metric's feature extractor is a plain function of the fed images: the real Inception weights are an external asset
    with open(cfg_path, 'a') as f:
        f.write('evaluation[0]["metrics"]["feature_fn"] = lambda x: x.mean(dim=(2, 3))\n')
    sd = _state_dict('ssdnerf_cars_uncond', over)
    ckpt = tmp_path / 'work' / 'iter_100.pth'
    ckpt.parent.mkdir()
    torch.save(dict(meta=dict(iter=100), state_dict=sd), ckpt)
    (ckpt.parent / 'iter_100_eval_log.txt').write_text('earlier line\n')
    out = T.main([cfg_path, str(ckpt), '--cfg-options', 'data.samples_per_gpu=2'])
    assert len(out) == 1 and out[0][0] == 'val_uncond'
    _, results, log_vars = out[0]
    # val_uncond has no test images: val_step logs nothing, the metric gets 5 scenes x 3 views of fakes
    assert log_vars == {} and set(results[0]) == {'fid', 'fid_mean', 'fid_cov', 'kid'}
    # viz_dir: batches 0 and 2 of [0, 1], [2, 3], [4]
    scenes = sorted({f[len('scene_'):len('scene_') + 4] for f in os.listdir(viz) if not f.endswith('_mean.png')})
    assert scenes == ['0000', '0001', '0004'], os.listdir(viz)
    log = (ckpt.parent / 'iter_100_eval_log.txt').read_text().splitlines()
    assert log[0] == 'earlier line'
    assert [line.split(' - ')[-1] for line in log if ' = ' in line] == [f'{k} = {v}' for k, v in results[0].items()]


def test_unconditional_log_vars_equal_hand_loop(cuda, tmp_path):
    """val_uncond with test images (every view a test view): the driver's log_vars against the hand-written loop"""
    from ssdnerf_b200 import test as T
    tree = str(tmp_path / 'tree')
    write_srn_tree(tree, 5, 3, RES)
    over = dict(num_timesteps=2, img_size=[RES, RES])
    cfg_path = str(tmp_path / 'uncond.py')
    viz = str(tmp_path / 'viz')
    write_config(cfg_path, 'ssdnerf_cars_uncond', tree, over,
                 [dict(data='val_uncond', feed_batch_size=4, viz_dir=viz, viz_step=2, metrics=[])], 2)
    with open(cfg_path, 'a') as f:
        f.write('data["val_uncond"].update(load_imgs=True, num_test_imgs=0, num_train_imgs=0)\n')
    sd = _state_dict('ssdnerf_cars_uncond', over)
    ckpt = tmp_path / 'iter_5.pth'
    torch.save(dict(state_dict=sd), ckpt)
    (_, _, got), = T.main([cfg_path, str(ckpt)])
    assert {'test_psnr', 'test_ssim'} <= set(got)
    want = _hand_loop(cfg_path, sd, 'val_uncond', viz_dir=str(tmp_path / 'viz_hand'), viz_step=2)
    _check_equal(got, want)
    assert sorted(os.listdir(viz)) == sorted(os.listdir(tmp_path / 'viz_hand'))
    assert (tmp_path / 'iter_5_eval_log.txt').exists()


def test_guide_optim_entry_with_ddp_checkpoint(cuda, tmp_path):
    from ssdnerf_b200 import test as T
    tree = str(tmp_path / 'tree')
    write_srn_tree(tree, 3, 3, RES)
    over = dict(num_timesteps=3, img_size=[RES, RES], n_inverse_steps=2, extra_scene_step=1, n_inverse_rays=256)
    cfg_path = str(tmp_path / 'recons.py')
    write_config(cfg_path, 'ssdnerf_cars_recons1v', tree, over,
                 [dict(data='val_cond', feed_batch_size=32, viz_dir=None, viz_step=1, metrics=[]),
                  dict(data='val_uncond', feed_batch_size=32, metrics=[])], 2)
    sd = _state_dict('ssdnerf_cars_recons1v', over)
    ckpt = tmp_path / 'latest.pth'
    torch.save(dict(state_dict={'module.' + k: v for k, v in sd.items()}), ckpt)
    out = T.main([cfg_path, str(ckpt), '--data', 'val_cond'])
    assert [o[0] for o in out] == ['val_cond']
    got = out[0][2]
    assert {'test_psnr', 'test_ssim'} <= set(got)
    _check_equal(got, _hand_loop(cfg_path, sd, 'val_cond'))


def test_checkpoint_with_extra_and_missing_keys(cuda, tmp_path):
    from ssdnerf_b200 import test as T
    tree = str(tmp_path / 'tree')
    write_srn_tree(tree, 1, 3, RES)
    over = dict(num_timesteps=2, img_size=[RES, RES])
    cfg_path = str(tmp_path / 'uncond.py')
    write_config(cfg_path, 'ssdnerf_cars_uncond', tree, over, [dict(data='val_uncond', metrics=[])], 2)
    sd = _state_dict('ssdnerf_cars_uncond', over)
    # an EMA-only file (init_model(ema_only=True) drops the trained copies) plus a key this model does not have
    ema_only = {k: v for k, v in sd.items() if not k.startswith(('diffusion.', 'decoder.'))}
    ema_only['extra_head.weight'] = torch.zeros(3)
    ckpt = tmp_path / 'ema.pth'
    torch.save(dict(state_dict=ema_only), ckpt)
    out = T.main([cfg_path, str(ckpt), '--data', 'nothing'])
    assert out == []
    log = (tmp_path / 'ema_eval_log.txt').read_text()
    assert 'unexpected key in source state_dict: extra_head.weight' in log
    missing = log.split('missing keys in source state_dict: ')[1].split('\n')[0].split(', ')
    assert sorted(missing) == sorted(k for k in sd if k.startswith(('diffusion.', 'decoder.')))


def test_evaluate_3d_feeds_fidkid_like_by_hand(cuda):
    from ssdnerf_b200 import evaluate_3d
    from ssdnerf_b200.metrics import FIDKID
    g = torch.Generator().manual_seed(1)
    preds = [torch.rand(n, 4, 3, 16, 16, generator=g).to(cuda) for n in (3, 3, 2)]

    class Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(1, device=cuda))

        def val_step(self, data, **kw):
            return dict(log_vars=dict(x=1.0), num_samples=len(data['scene_id']), pred_imgs=preds[data['i']])

    def feature_fn(x):
        return torch.cat([x.mean(dim=(2, 3)), x.square().mean(dim=(2, 3))], 1)

    kw = dict(num_images=20, num_subsets=3, max_subset_size=8, feature_fn=feature_fn)
    reals = torch.rand(24, 3, 16, 16, generator=g).to(cuda) * 2 - 1
    driven, hand = FIDKID(**kw), FIDKID(**kw)
    for m in (driven, hand):
        m.feed(reals, 'reals')
    evaluate_3d(Model(), [dict(i=i, scene_id=list(range(p.shape[0]))) for i, p in enumerate(preds)], metrics=[driven], feed_batch_size=5)
    for p in preds:
        for chunk in p.reshape(-1, 3, 16, 16).split(5):
            hand.feed(chunk * 2 - 1, 'fakes')
    assert driven.num_fake_feeded == hand.num_fake_feeded == 20
    assert all(torch.equal(a, b) for a, b in zip(driven.fake_feats, hand.fake_feats))
    assert driven.summary(torch.Generator().manual_seed(0)) == hand.summary(torch.Generator().manual_seed(0))
