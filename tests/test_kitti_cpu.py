"""KITTI preprocessing on the CPU against the reference's own tools/kitti_preproc.py output (tests/golden/reference_kitti_v1.npz):
label / calibration parsing, poses and intrinsics text byte for byte, the host twins of the raw PNG decode and of the resize, and the
resize against cv2.resize where cv2 is importable."""
import os

import numpy as np
import pytest

from ssdnerf_b200 import kitti as K

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_kitti_v1.npz'))


def write_tree(ref, root):
    """the fixture's KITTI tree under root; returns root as a string"""
    for k in ref.files:
        if k.startswith('in/'):
            p = os.path.join(str(root), k[3:])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, 'wb') as f:
                f.write(ref[k].tobytes())
    return str(root)


def stems(ref):
    return sorted(k[len('in/label_2/'):-4] for k in ref.files if k.startswith('in/label_2/'))


def host_instances(ref, out_size=128, out_border=4):
    """the reference's per-instance decisions from host code only: {name: (c2w, pad_tgt, pad_x, pad_y, box, whitening priors, text)}"""
    got = {}
    for s in stems(ref):
        labels = K.parse_labels(ref[f'in/label_2/{s}.txt'].tobytes().decode(), s)
        proj = K.parse_calib(ref[f'in/calib/{s}.txt'].tobytes().decode(), s)
        cam_t = K.camera_offset(proj)
        seg = ref[f'raw/instance_2/{s}.png']
        whitening = []
        for i, lab in enumerate(labels):
            if not (lab[1] == 0 and lab[2] == 0):
                continue
            ys, xs = (seg == 1000 + i).nonzero()
            if len(ys) == 0:
                continue
            y0, y1, x0, x1 = ys.min(), ys.max() + 1, xs.min(), xs.max() + 1
            c2w, pad, scale, px, py, text = K.instance_geometry(lab, cam_t, proj, y0, y1, x0, x1, out_size, out_border)
            priors = list(whitening)
            whitening.append((y0, y1, x0, x1, 1000 + i))
            if scale > 1:
                continue
            got[f'{s}_{i:03d}'] = (c2w, pad, px, py, (y0, y1, x0, x1, 1000 + i), priors, text)
    return got


def test_poses_and_intrinsics_text(ref):
    got = host_instances(ref)
    assert sorted(got) == ref['instances'].tolist()
    for name, (c2w, _, _, _, _, _, text) in got.items():
        assert K.pose_text(c2w) == str(ref[f'out/{name}/pose/000000.txt']), name
        assert text == str(ref[f'out/{name}/intrinsics.txt']), name


def test_corpus_covers_the_cases(ref):
    got = host_instances(ref)
    pads = [(v[1], max(v[4][1] - v[4][0], v[4][3] - v[4][2])) for v in got.values()]
    assert any(p > hw for p, hw in pads) and any(p == hw for p, hw in pads)          # pad_tgt from the 3-D box and from max(h, w)
    assert any(v[5] for v in got.values())                                           # earlier whitening boxes in play
    assert any(p == 240 for p, _ in pads)                                             # exactly half size: cv2's 2 x 2 average


def test_raw_decode_host(ref):
    for k in ref.files:
        if k.startswith('in/') and k.endswith('.png'):
            arr, st = K.decode_png_raw_host(ref[k].tobytes(), k)
            want = ref['raw/' + k[3:]]
            assert st == 0 and arr.dtype == want.dtype and np.array_equal(arr, want), k


def whitened_crop(ref, stem, box, priors):
    y0, y1, x0, x1, val = box
    img = ref[f'raw/image_2/{stem}.png'][y0:y1, x0:x1].copy()
    seg = ref[f'raw/instance_2/{stem}.png'][y0:y1, x0:x1]
    white = seg != val
    yy, xx = np.mgrid[y0:y1, x0:x1]
    for (a0, a1, b0, b1, _) in priors:
        white |= (yy >= a0) & (yy < a1) & (xx >= b0) & (xx < b1)
    img[white] = 255
    return img


def test_views_by_host_resize(ref):
    for name, (_, pad, px, py, box, priors, _) in host_instances(ref).items():
        crop = whitened_crop(ref, name[:6], box, priors)
        assert np.array_equal(crop, ref[f'out/{name}/000000.png']), name
        sq = np.full((pad, pad, 3), 255, np.uint8)
        sq[py:py + crop.shape[0], px:px + crop.shape[1]] = crop
        view = np.full((128, 128, 3), 255, np.uint8)
        view[4:124, 4:124] = K.resize_host(sq, 120, 120)
        assert np.array_equal(view, ref[f'out/{name}/rgb/000000.png']), name


def test_resize_equals_cv2_on_random_sizes():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(5)
    for it in range(120):
        sh, sw = (int(v) for v in rng.integers(1, 400, 2))
        dh, dw = (int(v) for v in rng.integers(1, 200, 2))
        if it % 3 == 0:                                   # the tool's case: a square shrunk to at most its size
            sw = sh = max(sh, 2)
            dh = dw = int(rng.integers(1, sh + 1))
        if it % 10 == 0:
            sh, sw = 2 * dh, 2 * dw
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        want = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(K.resize_host(img, dh, dw), want), (sh, sw, dh, dw)


def test_malformed_text_is_named():
    with pytest.raises(ValueError, match='lab.txt'):
        K.parse_labels('Car 0.0 0 x\n', 'lab.txt')
    with pytest.raises(ValueError, match='cal.txt'):
        K.parse_calib('P0: 1 2\n', 'cal.txt')
