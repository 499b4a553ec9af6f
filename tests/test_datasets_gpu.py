"""ShapeNetSRN + collate on the GPU against the reference's own stacked tensors (tests/golden/reference_dataset_v1.npz), val_step fed by
collate, and `python -m ssdnerf_b200.inception_stat` against the features FIDKID computes when fed the same reals."""
import os
import pickle

import numpy as np
import pytest
import torch

from ssdnerf_b200 import datasets as D
from tests.test_datasets_cpu import make_tree

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_dataset_v1.npz'))


def _prefixes(root):
    return [os.path.join(root, 'prefix_a'), os.path.join(root, 'prefix_b')]


def test_collate_equals_reference_stack(cuda, ref, tmp_path):
    root = make_tree(ref, tmp_path / 'tree')
    ds = D.ShapeNetSRN(data_prefix=_prefixes(root))
    batch = D.collate([ds[i] for i in range(len(ds))], cuda)
    n = int(ref['default/len'])
    want = np.stack([ref[f'default/{i}/cond_imgs'] for i in range(n)]).astype(np.float32) / 255
    assert batch['cond_imgs'].shape == want.shape and batch['cond_imgs'].device.type == 'cuda'
    assert np.array_equal(batch['cond_imgs'].cpu().numpy(), want)
    for k in ('cond_poses', 'cond_intrinsics'):
        assert np.array_equal(batch[k].cpu().numpy(), np.stack([ref[f'default/{i}/{k}'] for i in range(n)])), k
    assert batch['scene_id'] == list(range(n))
    assert batch['scene_name'] == [str(ref[f'default/{i}/scene_name']) for i in range(n)]
    assert [[p.replace(root, '<root>') for p in ps] for ps in batch['cond_img_paths']] == \
        [ref[f'default/{i}/cond_img_paths'].tolist() for i in range(n)]


def test_val_step_fed_by_collate(cuda, ref, tmp_path):
    from tests.test_viz_gpu import _cars_model
    root = make_tree(ref, tmp_path / 'tree')
    ds = D.ShapeNetSRN(data_prefix=_prefixes(root), num_train_imgs=0)
    data = D.collate([ds[i] for i in range(len(ds))], cuda)
    n = int(ref['default/len'])
    # the same views as the reference's default case recorded them (every view is a condition view there)
    direct = dict(scene_id=list(range(n)), scene_name=data['scene_name'], test_img_paths=data['test_img_paths'],
                  test_imgs=torch.from_numpy(np.stack([ref[f'default/{i}/cond_imgs'] for i in range(n)]).astype(np.float32) / 255).to(cuda),
                  test_poses=torch.from_numpy(np.stack([ref[f'default/{i}/cond_poses'] for i in range(n)])).to(cuda),
                  test_intrinsics=torch.from_numpy(np.stack([ref[f'default/{i}/cond_intrinsics'] for i in range(n)])).to(cuda))
    assert set(data) == set(direct) and torch.equal(data['test_imgs'], direct['test_imgs'])
    noise = torch.randn(n, 3, 6, 128, 128, generator=torch.Generator().manual_seed(3)).to(cuda)
    model, _ = _cars_model(cuda, num_timesteps=2, n_inverse_steps=0, img_size=(32, 32))
    model.lpips = None
    logs = []
    for d in (data, direct):
        torch.manual_seed(0)
        logs.append(model.val_step(dict(d, noise=noise))['log_vars'])
    assert 'test_psnr' in logs[0] and 'test_ssim' in logs[0]
    # the inputs are identical; what is left is the renderer's run-to-run float summation order (about 1e-6 in the PSNR)
    for k in ('test_psnr', 'test_ssim'):
        assert abs(logs[0][k] - logs[1][k]) <= 1e-5 * abs(logs[1][k]) + 1e-6, (k, logs)


@torch.no_grad()
def test_inception_stat_matches_fidkid(cuda, ref, tmp_path):
    from oracle import inception_port as ip
    from ssdnerf_b200 import inception_stat
    from ssdnerf_b200.metrics import FIDKID
    from tests.test_inception_cpu import GOLDEN as INCEPTION_GOLDEN, _tf_module
    root = make_tree(ref, tmp_path / 'tree')
    weights = str(tmp_path / 'inception-2015-12-05.pt')
    torch.jit.save(_tf_module(ip.fixture_state_dict(np.load(INCEPTION_GOLDEN))), weights)
    pkl = str(tmp_path / 'stats' / 'real_inception.pkl')
    args = dict(type='StyleGAN', inception_path=weights)
    cfg = tmp_path / 'cfg.py'
    cfg.write_text(f'data = dict(val=dict(type="ShapeNetSRN", data_prefix={_prefixes(root)!r}, specific_observation_idcs=[1], '
                   f'max_num_scenes=1))\n'
                   f'evaluation = [dict(data="val", metrics=dict(type="FIDKID", num_images=24, inception_pkl={pkl!r}, '
                   f'inception_args={args!r}))]\n')
    inception_stat.main([str(cfg), '--batch-size', '5'])
    with open(pkl, 'rb') as f:
        stats = pickle.load(f)
    # the fed path: every test view of every scene (all 6: num_train_imgs=0, the indices and scene limit dropped), in scene order
    ds = D.ShapeNetSRN(data_prefix=_prefixes(root), num_train_imgs=0)
    reals = D.collate([ds[i] for i in range(len(ds))], cuda)['test_imgs'].reshape(-1, 32, 32, 3).permute(0, 3, 1, 2) * 2 - 1
    fakes = reals.flip(-1) * 0.7
    fed = FIDKID(num_images=24, num_subsets=5, max_subset_size=12, inception_args=args)
    fed.feed(reals.contiguous(), 'reals')
    feats = torch.cat(fed.real_feats).cpu().numpy()
    assert stats['size'] == 24 and stats['name'] == '.pkl'
    assert stats['feats_np'].dtype == np.float32 and np.array_equal(stats['feats_np'], feats)
    assert np.array_equal(stats['mean'], np.mean(feats, axis=0)) and stats['mean'].dtype == np.float32
    assert np.array_equal(stats['cov'], np.cov(feats, rowvar=False)) and stats['cov'].dtype == np.float64
    from_pkl = FIDKID(num_images=24, num_subsets=5, max_subset_size=12, inception_pkl=pkl, inception_args=args)
    from_pkl.prepare()
    results = []
    for m in (fed, from_pkl):
        m.feed(fakes.contiguous(), 'fakes')
        results.append(m.summary(generator=torch.Generator().manual_seed(0)))
    (fid_f, _, _, kid_f), (fid_p, _, _, kid_p) = results
    assert kid_p == kid_f
    assert abs(fid_p - fid_f) <= 1e-5 * abs(fid_f) + 1e-6


def test_inception_stat_names_a_missing_weight_file(cuda, ref, tmp_path):
    from ssdnerf_b200 import inception_stat
    root = make_tree(ref, tmp_path / 'tree')
    missing = str(tmp_path / 'nowhere' / 'inception.pt')
    cfg = tmp_path / 'cfg.py'
    cfg.write_text(f'data = dict(val=dict(type="ShapeNetSRN", data_prefix={_prefixes(root)!r}))\n'
                   f'evaluation = dict(data="val", metrics=[dict(type="FID", inception_pkl={str(tmp_path / "x.pkl")!r}, '
                   f'inception_args=dict(type="StyleGAN", inception_path={missing!r}))])\n')
    with pytest.raises(RuntimeError, match='nowhere/inception.pt'):
        inception_stat.main([str(cfg)])
