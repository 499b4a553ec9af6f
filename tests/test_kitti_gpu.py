"""`python -m ssdnerf_b200.kitti_preproc` on the GPU against the reference's own tools/kitti_preproc.py output
(tests/golden/reference_kitti_v1.npz): the same instance directories, every PNG equal bit for bit when decoded, the text files byte
for byte; the raw decode of the corpus; a corrupt input named; and the reconskitti config's val_step on the output."""
import json
import os

import numpy as np
import pytest
import torch

from ssdnerf_b200 import kitti as K
from tests.test_kitti_cpu import GOLDEN, stems, write_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_kitti_v1.npz'))


def _decode(data, name):
    arr, st = K.decode_png_raw_host(data, name)
    assert st == 0, name
    return arr


@pytest.mark.parametrize('batch_frames', [1, 16])
def test_tool_equals_reference(cuda, ref, tmp_path, batch_frames):
    tree = write_tree(ref, tmp_path / 'kitti')
    out = tmp_path / 'out'
    n = K.preprocess(tree, str(out), 128, 4, device=cuda, batch_frames=batch_frames)
    insts = ref['instances'].tolist()
    assert n == len(insts) and sorted(os.listdir(out)) == insts
    for name in insts:
        d = out / name
        assert sorted(os.listdir(d)) == ['000000.png', 'intrinsics.txt', 'pose', 'rgb']
        for rel in ('rgb/000000.png', '000000.png'):
            got = _decode((d / rel).read_bytes(), f'{name}/{rel}')
            assert np.array_equal(got, ref[f'out/{name}/{rel}']), (name, rel)
        for rel in ('pose/000000.txt', 'intrinsics.txt'):
            assert (d / rel).read_text() == str(ref[f'out/{name}/{rel}']), (name, rel)


def test_raw_decode_equals_imread_unchanged(cuda, ref):
    keys = [k for k in ref.files if k.startswith('in/') and k.endswith('.png')]
    buf, desc = K.decode_png_raw([ref[k].tobytes() for k in keys], keys, cuda)
    host = buf.cpu().numpy()
    for k, d in zip(keys, desc):
        want = ref['raw/' + k[3:]]
        got = host[int(d['out_offset']):int(d['out_offset']) + want.nbytes].view(want.dtype).reshape(want.shape)
        assert np.array_equal(got, want), k


def test_encode_bgr_round_trip(cuda):
    rng = np.random.default_rng(2)
    shapes = [(1, 1), (7, 13), (128, 128), (143, 61), (7, 13), (375, 1242)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    offs, o = [], 0
    for im in imgs:
        offs.append(o)
        o += (im.nbytes + 15) // 16 * 16
    buf = np.zeros(o, np.uint8)
    for im, off in zip(imgs, offs):
        buf[off:off + im.nbytes] = im.reshape(-1)
    files = K.encode_bgr(torch.from_numpy(buf).to(cuda), shapes, offs, cuda)
    for f, im in zip(files, imgs):
        assert f[25] == 2                                     # colour type 2: RGB, as cv2.imwrite writes a 3-channel image
        assert np.array_equal(_decode(f, 'round trip'), im)


def test_corrupt_input_is_named(cuda, ref, tmp_path):
    tree = write_tree(ref, tmp_path / 'kitti')
    p = os.path.join(tree, 'instance_2', '000001.png')
    data = bytearray(open(p, 'rb').read())
    # flip bits inside the zlib stream of the first IDAT and fix up its CRC so that only the device decode can notice
    import struct
    import zlib
    pos = 8
    while data[pos + 4:pos + 8] != b'IDAT':
        pos += 12 + struct.unpack('>I', data[pos:pos + 4])[0]
    length = struct.unpack('>I', data[pos:pos + 4])[0]
    for k in range(20, min(length, 400), 7):
        data[pos + 8 + k] ^= 0x5A
    data[pos + 8 + length:pos + 12 + length] = struct.pack('>I', zlib.crc32(bytes(data[pos + 4:pos + 8 + length])))
    open(p, 'wb').write(bytes(data))
    with pytest.raises(ValueError, match='instance_2/000001.png'):
        K.preprocess(tree, str(tmp_path / 'out'), device=cuda)
    with open(os.path.join(tree, 'label_2', '000002.txt'), 'w') as f:
        f.write('Car 0.0 zero\n')
    with pytest.raises(ValueError, match='label_2/000002.txt'):
        K.preprocess(tree, str(tmp_path / 'out2'), device=cuda)


def test_reconskitti_val_step_on_output(cuda, ref, tmp_path):
    import ssdnerf_b200 as S
    from oracle import unet_port as up
    from ssdnerf_b200 import datasets as D
    tree = write_tree(ref, tmp_path / 'kitti')
    out = tmp_path / 'cars_kitti'
    K.preprocess(tree, str(out), device=cuda)
    # a small camera spiral for test_pose_override, in the layout of demo/camera_spiral_cars
    spiral = tmp_path / 'spiral'
    (spiral / 'pose').mkdir(parents=True)
    for v in range(3):
        a = 2 * np.pi * v / 3
        c2w = np.array([[np.cos(a), 0, np.sin(a), 1.3 * np.sin(a)], [0, -1, 0, 0], [np.sin(a), 0, -np.cos(a), -1.3 * np.cos(a)], [0, 0, 0, 1]])
        np.savetxt(spiral / 'pose' / f'{v:06d}.txt', c2w.reshape(1, -1))
    (spiral / 'intrinsics.txt').write_text('131.250000 64.000000 64.000000 0.\n0. 0. 0.\n1.\n128 128\n')
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/supp_cfgs/ssdnerf_cars_reconskitti.py']
    ds = D.ShapeNetSRN(data_prefix=str(out), specific_observation_idcs=[0], test_pose_override=str(spiral))
    assert len(ds) == len(ref['instances'])
    data = D.collate([ds[i] for i in range(2)], cuda)
    assert data['cond_imgs'].shape == (2, 1, 128, 128, 3)
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'],
                          test_cfg=dict(c['test_cfg'], num_timesteps=2, n_inverse_steps=2, n_inverse_rays=2 ** 10, img_size=(32, 32)))
    # the config's dropout (0.1) sits between a residual block's norm and its second convolution: conv_2.1 -> conv_2.2
    sd = {k.replace('conv_2.1.', 'conv_2.2.'): v for k, v in up.random_state_dict(up.unet_spec(), seed=7, std=0.02).items()}
    for diff in (model.diffusion, model.diffusion_ema):
        diff.denoising.load_state_dict(sd, strict=True)
    model = model.to(cuda).eval()
    model.lpips = None
    assert model.test_cfg['cond_mode'] == 'guide_optim'
    res = model.val_step(dict(data, noise=torch.randn(2, 3, 6, 128, 128, generator=torch.Generator().manual_seed(3)).to(cuda)))
    img = res['pred_imgs']
    assert img.shape[:2] == (2, 3) and torch.isfinite(img).all()
