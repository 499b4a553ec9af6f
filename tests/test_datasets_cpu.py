"""ssdnerf_b200.datasets without a GPU: `ShapeNetSRN` against the reference's own outputs (tests/golden/reference_dataset_v1.npz),
`build_dataset` on every shipped config's data sections, the host PNG decoder (the device decoder's validation code) against
cv2.imread on the corpus of tests/golden/reference_png_v1.npz and its malformed set, and the host-side refusals."""
import json
import os
import pickle
import random
import struct
import zlib

import numpy as np
import pytest
import torch

from ssdnerf_b200 import build_dataset, datasets as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
TOKEN = '<root>'


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_dataset_v1.npz'))


@pytest.fixture(scope='module')
def png():
    return np.load(os.path.join(GOLDEN, 'reference_png_v1.npz'))


def make_tree(ref, root):
    offs = ref['tree_offsets']
    for i, rel in enumerate(ref['tree_paths']):
        p = os.path.join(root, str(rel))
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'wb') as f:
            f.write(ref['tree_bytes'][offs[i]:offs[i + 1]].tobytes())
    return str(root)


def resolve(x, root):
    if isinstance(x, str):
        return x.replace(TOKEN, root)
    if isinstance(x, list):
        return [resolve(v, root) for v in x]
    return x


def check_item(ref, key, item, root):
    want = sorted(k.rsplit('/', 1)[1] for k in ref.files if k.startswith(key + '/') and k.count('/') == key.count('/') + 1)
    assert sorted(item) == want, key
    for k, v in item.items():
        exp = ref[f'{key}/{k}']
        if k.endswith('_imgs'):
            got = np.stack([D.decode_png_host(b, f'{key} {k}[{j}]')[0] for j, b in enumerate(v)])
            assert np.array_equal(got, exp.astype(np.float32) / 255), (key, k)
        elif k.endswith('_paths'):
            assert [p.replace(root, TOKEN) for p in v] == exp.tolist(), (key, k)
        elif isinstance(v, torch.Tensor):
            assert v.dtype == torch.float32 and np.array_equal(v.numpy(), exp), (key, k)
        else:
            assert v == exp.item(), (key, k)


def test_shapenet_srn_equals_reference(ref, tmp_path):
    root = make_tree(ref, tmp_path / 'tree')
    random.seed(int(ref['random_seed']))
    for case, kw in json.loads(str(ref['cases'])).items():
        ds = D.ShapeNetSRN(**{k: resolve(v, root) for k, v in kw.items()})
        assert len(ds) == int(ref[f'{case}/len']), case
        for i in range(len(ds)):
            check_item(ref, f'{case}/{i}', ds[i], root)
        if case == 'cached':
            with open(kw['cache_path'].replace(TOKEN, root), 'rb') as f:
                assert isinstance(pickle.load(f), list)
            ds2 = D.ShapeNetSRN(**{k: resolve(v, root) for k, v in kw.items()})
            for i in range(len(ds2)):
                check_item(ref, f'cached_reread/{i}', ds2[i], root)


def test_loads_the_cache_the_reference_wrote(ref, tmp_path):
    cache = tmp_path / 'ref_cache.pkl'
    cache.write_bytes(ref['cache_pkl'].tobytes())
    gen_root = str(ref['cache_root'])
    ds = D.ShapeNetSRN(data_prefix='/nonexistent', cache_path=str(cache), load_imgs=False)
    assert len(ds) == int(ref['cached/len'])
    for i in range(len(ds)):
        check_item(ref, f'cached/{i}', ds[i], gen_root)


def test_getitem_does_not_touch_cuda(ref, tmp_path, monkeypatch):
    root = make_tree(ref, tmp_path / 'tree')
    monkeypatch.setattr(torch.cuda, 'current_device', lambda: (_ for _ in ()).throw(AssertionError('CUDA touched')))
    item = D.ShapeNetSRN(data_prefix=[os.path.join(root, 'prefix_a')])[0]
    assert isinstance(item['cond_imgs'][0], bytes)


def test_build_dataset_from_every_shipped_config(ref, tmp_path):
    root = make_tree(ref, tmp_path / 'tree')
    cfgs = json.loads(str(ref['configs']))
    assert len(cfgs) >= 20
    built = 0
    for path, c in cfgs.items():
        for split, dcfg in c['data'].items():
            if not isinstance(dcfg, dict) or dcfg.get('type') != 'ShapeNetSRN':
                continue
            d = dict(dcfg, data_prefix=os.path.join(root, 'prefix_c'), cache_path=None)
            if d.get('test_pose_override'):
                d['test_pose_override'] = os.path.join(root, 'override')
            ds = build_dataset(d)
            assert len(ds) == 1, (path, split)
            item = ds[0]
            assert item['scene_name'] in ('e5', '0000'), (path, split)
            built += 1
    assert built >= 40


def corpus(npz, prefix):
    b, o = npz[f'{prefix}_bytes'], npz[f'{prefix}_offsets']
    return [(str(n), b[o[i]:o[i + 1]].tobytes()) for i, n in enumerate(npz[f'{prefix}_names'])]


def test_host_decoder_equals_cv2_on_the_corpus(png):
    shapes = png['valid_shapes']
    po = np.cumsum([0] + [int(np.prod(s)) for s in shapes])
    files = corpus(png, 'valid')
    assert len(files) >= 50
    for i, (name, data) in enumerate(files):
        img, status = D.decode_png_host(data, name)
        assert status == 0, name
        want = png['valid_pixels'][po[i]:po[i + 1]].reshape(shapes[i]).astype(np.float32) / 255
        assert np.array_equal(img, want), name


def test_host_decoder_statuses_on_the_malformed_set(png):
    for (name, data), want, match in zip(corpus(png, 'mal'), png['mal_status'], png['mal_match']):
        if want < 0:
            with pytest.raises(ValueError, match=str(match)):
                D.decode_png_host(data, name)
        else:
            _, status = D.decode_png_host(data, name)
            assert status == want, (name, status, D.STATUS_REASONS.get(status))


def _chunk(t, body):
    return struct.pack('>I', len(body)) + t + body + struct.pack('>I', zlib.crc32(t + body))


def _png(w, h, ct=2, depth=8, interlace=0, extra=b'', rows=None):
    bpp = {0: 1, 2: 3, 6: 4}[ct] * depth // 8
    raw = rows if rows is not None else b''.join(b'\0' + bytes(w * bpp) for _ in range(h))
    return (D.PNG_SIGNATURE + _chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, depth, ct, 0, 0, interlace)) + extra
            + _chunk(b'IDAT', zlib.compress(raw)) + _chunk(b'IEND', b''))


def test_host_refusals_before_any_launch():
    dev = 'cuda:0'    # never reached: every refusal is raised by the host parser
    with pytest.raises(NotImplementedError, match='sixteen.png: bit depth 16'):
        D.decode_png([_png(4, 4), _png(4, 4, depth=16)], dev, names=['ok.png', 'sixteen.png'])
    with pytest.raises(NotImplementedError, match='interlaced.png: Adam7'):
        D.decode_png([_png(4, 4, interlace=1)], dev, names=['interlaced.png'])
    with pytest.raises(NotImplementedError, match='exif.png: eXIf'):
        D.decode_png([_png(4, 4, extra=_chunk(b'eXIf', b'MM\0*'))], dev, names=['exif.png'])
    with pytest.raises(ValueError, match='c.png: size 5 x 4 differs from a.png'):
        D.decode_png([_png(4, 4), _png(4, 4), _png(5, 4)], dev, names=['a.png', 'b.png', 'c.png'])
    bomb = _png(1, 1).replace(struct.pack('>II', 1, 1), struct.pack('>II', 60000, 60000), 1)
    ihdr_end = 8 + 8 + 13
    bomb = bomb[:ihdr_end] + struct.pack('>I', zlib.crc32(bomb[12:ihdr_end])) + bomb[ihdr_end + 4:]
    with pytest.raises(ValueError, match='bomb.png: IHDR size 60000 x 60000'):
        D.decode_png([bomb], dev, names=['bomb.png'])
    with pytest.raises(ValueError, match='no files'):
        D.decode_png([], dev)
