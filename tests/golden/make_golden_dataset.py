"""Pins for ssdnerf_b200.datasets: the reference's OWN `ShapeNetSRN` (lib/datasets/shapenet_srn.py), executed from /root/reference on
a small synthetic SRN tree with mmcv / mmgen stubbed (`mmcv.imread` is cv2 + BGR -> RGB, `mmcv.load` / `dump` are pickle with mmcv's
protocol 2, `DataContainer` keeps `.data`).  Records every `parse_scene` output for a set of constructor arguments (seeded `random`),
the tree's files, the cache pickle the reference wrote, and the `data` / `evaluation` sections of every shipped config.
-> tests/golden/reference_dataset_v1.npz, replayed by tests/test_datasets_cpu.py and tests/test_datasets_gpu.py.

    python tests/golden/make_golden_dataset.py          (needs /root/reference and cv2)
"""
import glob
import json
import os
import pickle
import random
import shutil
import sys
import tempfile
import types

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
REF = '/root/reference'
ROOT_TOKEN = '<root>'


def stub_mm():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    def imread(path, channel_order='bgr'):
        img = cv2.imread(path, cv2.IMREAD_COLOR)
        return img[..., ::-1].copy() if channel_order == 'rgb' else img

    def dump(obj, path):
        with open(path, 'wb') as f:
            pickle.dump(obj, f, protocol=2)

    def load(path):
        with open(path, 'rb') as f:
            return pickle.load(f)

    class DC:
        def __init__(self, data, cpu_only=False, **kw):
            self.data, self.cpu_only = data, cpu_only

    class Reg:
        def register_module(self, *a, **k):
            return lambda cls: cls
    mod('mmcv', imread=imread, dump=dump, load=load).__path__ = []
    mod('mmcv.parallel', DataContainer=DC)
    mod('mmgen').__path__ = []
    mod('mmgen.datasets').__path__ = []
    mod('mmgen.datasets.builder', DATASETS=Reg())


def load_reference():
    stub_mm()
    import importlib.util
    spec = importlib.util.spec_from_file_location('ref_shapenet_srn', os.path.join(REF, 'lib/datasets/shapenet_srn.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.ShapeNetSRN


def write_scene(rng, root, name, n_views, size, names=None):
    d = os.path.join(root, name)
    os.makedirs(os.path.join(d, 'rgb'))
    os.makedirs(os.path.join(d, 'pose'))
    f = size * 1.0253
    with open(os.path.join(d, 'intrinsics.txt'), 'w') as fh:
        fh.write(f'{f:.6f} {size / 2} {size / 2} 0.\n0. 0. 0.\n1.\n{size} {size}\n')
    for i in range(n_views):
        stem = names[i] if names else f'{i:06d}'
        img = rng.integers(0, 256, (size, size, 4), dtype=np.uint8)
        img[size // 4:, :, :] = 255 - img[:size - size // 4]                 # some repetition for the deflate matches
        cv2.imwrite(os.path.join(d, 'rgb', stem + '.png'), img)
        rot, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        pose = np.eye(4)
        pose[:3, :3], pose[:3, 3] = rot, rng.normal(size=3) * 1.3
        np.savetxt(os.path.join(d, 'pose', stem + '.txt'), pose.reshape(1, 16), fmt='%.9f', delimiter=' ')


def make_tree(root):
    rng = np.random.default_rng(7)
    a, b = os.path.join(root, 'prefix_a'), os.path.join(root, 'prefix_b')
    # scene names interleave across the prefixes, so the sort by scene name is visible
    write_scene(rng, a, 'c3', 6, 32)
    write_scene(rng, a, 'a1', 6, 32, names=['000010', '000002', '000001', '000000', '000003', '000020'])
    write_scene(rng, b, 'b2', 6, 32)
    write_scene(rng, b, 'd4', 6, 32)
    write_scene(rng, os.path.join(root, 'prefix_c'), 'e5', 251, 8)       # the SRN test split's 251-view naming
    with open(os.path.join(b, 'not_a_scene.txt'), 'w') as fh:
        fh.write('ignored\n')
    ov = os.path.join(root, 'override')
    write_scene(rng, root, 'override', 4, 32)
    shutil.rmtree(os.path.join(ov, 'rgb'))
    os.makedirs(os.path.join(root, 'codes'))
    torch.save(torch.from_numpy(rng.normal(size=(3, 4, 4)).astype(np.float32)), os.path.join(root, 'codes', 'b2.pth'))
    return [a, b]


def cases(root, prefixes):
    p = prefixes
    return {
        'default': dict(data_prefix=p),
        'single_prefix': dict(data_prefix=p[0]),
        'specific_idcs': dict(data_prefix=p, specific_observation_idcs=[2], load_imgs=False),
        'num_test_imgs': dict(data_prefix=p, num_test_imgs=2, load_imgs=False),
        'num_train_imgs': dict(data_prefix=p, num_train_imgs=3, load_imgs=False),
        'random_test_imgs': dict(data_prefix=p, num_train_imgs=2, random_test_imgs=True, load_imgs=False),
        'id_as_name_step': dict(data_prefix=p, scene_id_as_name=True, max_num_scenes=1, step=2, load_imgs=False),
        'max_num_scenes': dict(data_prefix=p, max_num_scenes=3, load_imgs=False),
        'no_cond': dict(data_prefix=p, load_cond_data=False, num_train_imgs=2, load_imgs=False),
        'no_test_code': dict(data_prefix=p, load_test_data=False, code_dir=os.path.join(root, 'codes'), load_imgs=False),
        'code_only': dict(data_prefix=p, code_only=True, code_dir=os.path.join(root, 'codes')),
        'pose_override': dict(data_prefix=p, test_pose_override=os.path.join(root, 'override'), num_test_imgs=2, load_imgs=False),
        'srn_test_split': dict(data_prefix=os.path.join(root, 'prefix_c'), specific_observation_idcs=[64], load_imgs=False),
        'cached': dict(data_prefix=p, cache_path=os.path.join(root, 'cache.pkl'), load_imgs=False),
    }


def rel(x, root):
    return x.replace(root, ROOT_TOKEN)


def record(out, key, item, root):
    for k, v in item.items():
        v = getattr(v, 'data', v)
        name = f'{key}/{k}'
        if isinstance(v, torch.Tensor):
            out[name] = v.numpy()
            if k.endswith('_imgs'):
                out[name] = np.round(v.numpy() * 255).astype(np.uint8)        # exactly u8 / 255
        elif k.endswith('_paths'):
            out[name] = np.array([rel(s, root) for s in v])
        else:
            out[name] = np.array(v)


def main():
    ShapeNetSRN = load_reference()
    out = {}
    with tempfile.TemporaryDirectory() as root:
        prefixes = make_tree(root)
        random.seed(1234)
        for case, kw in cases(root, prefixes).items():
            ds = ShapeNetSRN(**kw)
            out[f'{case}/len'] = np.array(len(ds))
            for i in range(len(ds)):
                record(out, f'{case}/{i}', ds[i], root)
            if case == 'cached':          # the second construction reads the cache the first one wrote
                with open(kw['cache_path'], 'rb') as f:
                    out['cache_pkl'] = np.frombuffer(f.read(), np.uint8)
                out['cache_root'] = np.array(root)
                ds2 = ShapeNetSRN(**kw)
                for i in range(len(ds2)):
                    record(out, f'cached_reread/{i}', ds2[i], root)
        files = sorted(p for p in glob.glob(os.path.join(root, '**'), recursive=True) if os.path.isfile(p) and not p.endswith('.pkl'))
        blobs = [open(p, 'rb').read() for p in files]
        out['tree_paths'] = np.array([os.path.relpath(p, root) for p in files])
        out['tree_offsets'] = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
        out['tree_bytes'] = np.frombuffer(b''.join(blobs), np.uint8)
    out['random_seed'] = np.array(1234)
    out['cases'] = np.array(json.dumps({k: {kk: (rel(vv, root) if isinstance(vv, str) else [rel(x, root) for x in vv] if isinstance(vv, list)
                                               and vv and isinstance(vv[0], str) else vv) for kk, vv in v.items()}
                                        for k, v in cases(root, [os.path.join(root, 'prefix_a'), os.path.join(root, 'prefix_b')]).items()}))
    from ssdnerf_b200 import Config
    cfgs = {}
    for path in sorted(glob.glob(os.path.join(REF, 'configs', '**', '*.py'), recursive=True)):
        cfg = Config.fromfile(path)
        if 'data' in cfg:
            cfgs[os.path.relpath(path, REF)] = dict(data=cfg['data'], evaluation=cfg.get('evaluation', []))
    out['configs'] = np.array(json.dumps(cfgs, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, 'reference_dataset_v1.npz'), **out)
    print(len(out), 'arrays;', os.path.getsize(os.path.join(HERE, 'reference_dataset_v1.npz')), 'bytes')


if __name__ == '__main__':
    main()
