"""Writes tests/golden/reference_kitti_v1.npz: a small synthetic KITTI object tree and what the reference's own
tools/kitti_preproc.py main() makes of it.

mmcv is not needed: a minimal `mmcv` module with mmcv's cv2 mappings is injected (imread(p, 'unchanged') -> cv2.imread(p,
IMREAD_UNCHANGED), imresize(img, (w, h)) -> cv2.resize(img, (w, h), interpolation=INTER_LINEAR), imwrite -> cv2.imwrite after
creating the parent directory, track_iter_progress -> identity).

Stored: every input file's bytes (`in/<rel path>`), the IMREAD_UNCHANGED arrays of the PNG inputs (`raw/<rel path>`), and per output
instance directory the decoded `rgb/000000.png` and `000000.png` (IMREAD_UNCHANGED) and the exact text of `pose/000000.txt` and
`intrinsics.txt` (`out/<instance>/...`).

Corpus: instances skipped for truncation, occlusion and an empty mask; a `scale > 1` instance that still whitens a later one's box;
overlapping boxes; boxes on all four frame edges; pad_tgt from the 3-D box and from max(h, w); odd crop sizes; a frame with no kept
instance; non-car types; two frames at KITTI's 1242 x 375 and two smaller ones.

    python tests/golden/make_golden_kitti.py --reference <checkout of Lakonik/SSDNeRF>
"""
import argparse
import os
import sys
import tempfile
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FX, CX, CY = 721.5377, 609.5593, 172.854
P2_T = (44.85728, 0.2163791, 0.002745884)


def _mmcv():
    m = types.ModuleType('mmcv')
    m.imread = lambda p, flag='color': cv2.imread(p, cv2.IMREAD_UNCHANGED if flag == 'unchanged' else cv2.IMREAD_COLOR)
    m.imresize = lambda img, size: cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)

    def imwrite(img, path):
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        return cv2.imwrite(path, img)
    m.imwrite = imwrite
    m.track_iter_progress = lambda x: x
    return m


def _calib(fx=FX, cx=CX, cy=CY):
    rows = []
    for k in range(4):
        t = P2_T if k == 2 else (0.0, 0.0, 0.0)
        rows.append(f'P{k}: {fx:.12e} 0.000000000000e+00 {cx:.12e} {t[0] * fx:.12e} 0.000000000000e+00 {fx:.12e} {cy:.12e} '
                    f'{t[1] * fx:.12e} 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 {t[2]:.12e}')
    rows.append('R0_rect: 1 0 0 0 1 0 0 0 1')
    return '\n'.join(rows) + '\n'


def _label(typ, trunc, occ, box2d, dims, loc, ry):
    return (f'{typ} {trunc:.2f} {occ} -1.57 {box2d[0]:.2f} {box2d[1]:.2f} {box2d[2]:.2f} {box2d[3]:.2f} '
            f'{dims[0]:.2f} {dims[1]:.2f} {dims[2]:.2f} {loc[0]:.2f} {loc[1]:.2f} {loc[2]:.2f} {ry:.2f}')


def make_tree(root, seed=0):
    """the synthetic tree: {stem: (H, W, [(label line, mask drawer or None)])}"""
    rng = np.random.default_rng(seed)
    frames = {
        # KITTI-sized frame: skips of every kind, overlap in order, the scale > 1 whitener, edges left / top
        '000000': (375, 1242, [
            (_label('Car', 0.0, 0, (100, 150, 300, 260), (1.5, 1.6, 3.9), (-4.0, 1.7, 12.0), 0.3), ('ellipse', (200, 210), (95, 50))),
            (_label('Car', 0.5, 0, (400, 150, 500, 260), (1.5, 1.6, 3.9), (1.0, 1.7, 15.0), -0.2), ('rect', (400, 150, 500, 260))),
            (_label('Van', 0.0, 1, (520, 150, 620, 260), (2.0, 1.8, 4.5), (3.0, 1.7, 15.0), 1.0), ('rect', (520, 150, 620, 260))),
            (_label('Car', 0.0, 0, (700, 150, 760, 200), (1.5, 1.6, 3.9), (6.0, 1.7, 20.0), 0.0), None),           # empty mask
            (_label('Car', 0.0, 0, (250, 180, 281, 201), (1.5, 1.6, 3.9), (-2.0, 1.7, 80.0), 2.0), ('rect', (250, 180, 281, 201))),
            (_label('Car', 0.0, 0, (230, 170, 420, 320), (1.5, 1.6, 3.9), (-1.5, 1.7, 10.0), -1.1), ('ellipse', (320, 245), (88, 73))),
            (_label('Pedestrian', 0.0, 0, (0, 0, 61, 143), (1.7, 0.6, 0.8), (-9.0, 1.5, 9.0), 0.5), ('ellipse', (25, 60), (30, 70))),
        ]),
        # KITTI-sized frame: edges right / bottom, pad_tgt from max(h, w) (far 3-D box), odd sizes
        '000001': (375, 1242, [
            (_label('Car', 0.0, 0, (1100, 250, 1242, 375), (1.5, 1.6, 3.9), (9.0, 1.7, 60.0), 0.7), ('rect', (1101, 251, 1242, 375))),
            (_label('Cyclist', 0.0, 0, (800, 100, 927, 229), (1.8, 0.6, 1.8), (4.0, 1.6, 30.0), -0.4), ('ellipse', (863, 164), (63, 64))),
            (_label('DontCare', -1, -1, (10, 10, 50, 50), (-1, -1, -1), (-1000, -1000, -1000), -10), None),
        ]),
        # small frame with no kept instance
        '000002': (120, 200, [
            (_label('Car', 0.3, 0, (10, 10, 100, 90), (1.5, 1.6, 3.9), (0.0, 1.7, 8.0), 0.0), ('rect', (10, 10, 100, 90))),
            (_label('Car', 0.0, 2, (100, 20, 190, 110), (1.5, 1.6, 3.9), (1.0, 1.7, 8.0), 0.0), ('rect', (100, 20, 190, 110))),
        ]),
        # small frame: a whole-frame instance (pad_tgt exactly 2 x 120 takes cv2's 2 x 2 average) and a 1-pixel-wide one
        '000003': (240, 240, [
            (_label('Truck', 0.0, 0, (0, 0, 240, 240), (3.0, 2.5, 8.0), (0.0, 1.7, 100.0), 0.9), ('rect', (0, 0, 240, 240))),
            (_label('Car', 0.0, 0, (0, 0, 1, 130), (1.5, 1.6, 3.9), (0.0, 1.7, 200.0), 0.0), ('rect', (0, 0, 1, 130))),
        ]),
    }
    for d in ('image_2', 'instance_2', 'label_2', 'calib'):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for stem, (H, W, insts) in frames.items():
        yy, xx = np.mgrid[:H, :W]
        # a random 20 x 30 tile repeated over the frame: neighbouring pixels differ for the resize to average, and the repeats keep
        # the fixture's raw arrays small
        tile = rng.integers(0, 256, (20, 30, 3), dtype=np.uint8)
        img = tile[yy % 20, xx % 30]
        seg = np.zeros((H, W), np.uint16)
        seg[H // 2:, :W // 3] = 26                                          # a background class id below 1000
        lines = []
        for i, (line, mask) in enumerate(insts):
            lines.append(line)
            if mask is None:
                continue
            m = np.zeros((H, W), np.uint8)
            if mask[0] == 'rect':
                x0, y0, x1, y1 = mask[1]
                m[y0:y1, x0:x1] = 1
            else:
                cv2.ellipse(m, mask[1], mask[2], 15.0, 0, 360, 1, -1)
            seg[m.astype(bool)] = 1000 + i
        if stem == '000003':                                               # the second instance steals a column of the first
            seg[:130, 0] = 1001
        cv2.imwrite(os.path.join(root, 'image_2', stem + '.png'), img, [cv2.IMWRITE_PNG_COMPRESSION, 9])
        cv2.imwrite(os.path.join(root, 'instance_2', stem + '.png'), seg, [cv2.IMWRITE_PNG_COMPRESSION, 9])
        with open(os.path.join(root, 'label_2', stem + '.txt'), 'w') as f:
            f.write('\n'.join(lines) + '\n')
        with open(os.path.join(root, 'calib', stem + '.txt'), 'w') as f:
            f.write(_calib())


def run_reference(reference, kitti_dir, out_dir):
    sys.modules['mmcv'] = _mmcv()
    sys.path.insert(0, os.path.join(reference, 'tools'))
    import kitti_preproc
    argv = sys.argv
    sys.argv = ['kitti_preproc.py', '--kitti-dir', kitti_dir, '--out-dir', out_dir]
    try:
        kitti_preproc.main()
    finally:
        sys.argv = argv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', required=True, help='a checkout of the reference repository (Lakonik/SSDNeRF)')
    ap.add_argument('--out', default=os.path.join(HERE, 'reference_kitti_v1.npz'))
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        kitti, out = os.path.join(tmp, 'kitti'), os.path.join(tmp, 'out')
        make_tree(kitti)
        run_reference(a.reference, kitti, out)
        data = {}
        for d in ('image_2', 'instance_2', 'label_2', 'calib'):
            for name in sorted(os.listdir(os.path.join(kitti, d))):
                rel = f'{d}/{name}'
                with open(os.path.join(kitti, rel), 'rb') as f:
                    data[f'in/{rel}'] = np.frombuffer(f.read(), np.uint8)
                if name.endswith('.png'):
                    data[f'raw/{rel}'] = cv2.imread(os.path.join(kitti, rel), cv2.IMREAD_UNCHANGED)
        insts = sorted(os.listdir(out))
        data['instances'] = np.array(insts)
        for inst in insts:
            for rel in ('rgb/000000.png', '000000.png'):
                data[f'out/{inst}/{rel}'] = cv2.imread(os.path.join(out, inst, rel), cv2.IMREAD_UNCHANGED)
            for rel in ('pose/000000.txt', 'intrinsics.txt'):
                with open(os.path.join(out, inst, rel)) as f:
                    data[f'out/{inst}/{rel}'] = np.array(f.read())
        np.savez_compressed(a.out, **data)
        print(a.out, 'instances:', insts)


if __name__ == '__main__':
    main()
