"""Pins for the H.264 orbit-video path (csrc/h264.cu, oracle/h264_port.py, video.write_mp4): a corpus of RGB u8 frames, the MP4
files the numpy encoder writes for them, and what FFmpeg's decoder (through cv2.VideoCapture) makes of each file: the SHA-256 of
every decoded luma plane (CAP_PROP_CONVERT_RGB = 0), and the luma and BGR samples of each frame's top-left WINDOW x WINDOW corner
(the whole frame when it is smaller).  So the decoder match is checked where cv2 is not installed, bit for bit on every plane through
the digests, while the file stays small.

Corpus: sizes 2x2, 16x16, 18x34 (cropped), 64x64, 128x128, 256x256, 254x258 and one 1024x1024 frame; flat, noise, render-like
gradients over white, black / white macroblock patterns whose residuals reach the level escape (level_prefix 15), and noise whose
slice data holds 00 00 0x runs (emulation prevention, asserted); QPs MIN_QP (10), 20, 30 and 51.

    python tests/golden/make_golden_h264.py          (needs cv2 with FFmpeg)
-> tests/golden/reference_h264_v1.npz, replayed by tests/test_h264_cpu.py and tests/test_h264_gpu.py.
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import h264_port as H  # noqa: E402

FPS = 30
WINDOW = 128


def gradient(h, w, rng):
    """a render-like frame: a shaded ellipse over white, smooth edges"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    cy, cx = (h - 1) * rng.uniform(0.4, 0.6), (w - 1) * rng.uniform(0.4, 0.6)
    d = ((y - cy) / (0.35 * h + 0.5)) ** 2 + ((x - cx) / (0.3 * w + 0.5)) ** 2
    base = rng.uniform(40, 220, 3)
    shade = (1 - 0.5 * d)[..., None] * base + 12 * np.sin(x / 7 + y / 11)[..., None]
    a = np.clip(1.5 - d, 0, 1)[..., None]
    return np.clip(np.rint(a * shade + (1 - a) * 255), 0, 255).astype(np.uint8)


def patterns(h, w):
    """black / white macroblock checkers, 4x4 and 1x1 checkers and their mixtures: the largest residuals 8-bit input gives"""
    yy, xx = np.mgrid[0:h, 0:w]
    p = [((xx // 16 + yy // 16) % 2) * 255, ((xx // 4 + yy // 4) % 2) * 255, ((xx + yy) % 2) * 255,
         (((xx // 16 + yy // 16) % 2) ^ ((xx % 4 < 2) ^ (yy % 4 < 2))) * 255]
    out = [np.repeat(q[..., None], 3, -1) for q in p] + [np.stack([p[0], 255 - p[0], p[1]], -1)]
    return np.stack(out).astype(np.uint8)


def corpus():
    """[(name, qp, frames u8 [n, h, w, 3])]"""
    rng = np.random.default_rng(264)
    noise = lambda n, h, w, seed: np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    flat = lambda h, w, v: np.full((1, h, w, 3), v, np.uint8)
    items = []
    tiny = np.concatenate([noise(1, 2, 2, 1), flat(2, 2, 77), noise(1, 2, 2, 2)])
    for qp in (10, 30):
        items.append((f'tiny_q{qp}', qp, tiny))
    mb = np.concatenate([gradient(16, 16, rng)[None], noise(1, 16, 16, 3), flat(16, 16, 255)])
    for qp in (20, 51):
        items.append((f'mb16_q{qp}', qp, mb))
    crop = np.concatenate([noise(1, 18, 34, 4), gradient(18, 34, rng)[None], flat(18, 34, 0)])
    for qp in (10, 20, 30, 51):
        items.append((f'crop_q{qp}', qp, crop))
    pat = patterns(64, 64)
    for qp in (10, 20):
        items.append((f'pattern_q{qp}', qp, pat))
    items.append(('epb_q10', 10, noise(2, 64, 64, 1)))
    r128 = np.stack([gradient(128, 128, rng) for _ in range(3)])
    for qp in (20, 30):
        items.append((f'r128_q{qp}', qp, r128))
    items.append(('r256_q20', 20, np.concatenate([np.stack([gradient(256, 256, rng) for _ in range(2)]), flat(256, 256, 255)])))
    items.append(('odd_q30', 30, np.concatenate([gradient(254, 258, rng)[None], noise(1, 254, 258, 5)])))
    items.append(('big_q20', 20, gradient(1024, 1024, rng)[None]))
    return items


def unescape(nal):
    """the RBSP of a NAL unit's payload: every 0x03 that follows two zero bytes removed"""
    out, zeros = bytearray(), 0
    for b in nal[1:]:
        if zeros == 2 and b == 3:
            zeros = 0
            continue
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


def digest(plane):
    """SHA-256 of a u8 plane's C-order bytes, as 32 u8"""
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(plane, np.uint8).tobytes()).digest(), np.uint8)


def decode(path):
    """(Y [n, h, w], BGR [n, h, w, 3]) u8 of cv2's decode of `path`"""
    import cv2
    ys, bgrs = [], []
    cap = cv2.VideoCapture(path)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    w, h = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    while True:
        ok, f = cap.read()
        if not ok:
            break
        ys.append(f.reshape(-1)[:h * w].reshape(h, w))
    cap = cv2.VideoCapture(path)
    while True:
        ok, f = cap.read()
        if not ok:
            break
        bgrs.append(f)
    return np.stack(ys), np.stack(bgrs)


def main():
    from ssdnerf_b200.video import write_mp4
    out = {}
    epb = 0
    with tempfile.TemporaryDirectory() as tmp:
        for name, qp, frames in corpus():
            sps, pps, aus = H.encode(frames, qp, FPS)
            epb += sum(len(a) - 5 - len(unescape(a[4:])) for a in aus)
            path = os.path.join(tmp, name + '.mp4')
            write_mp4(path, sps, pps, aus, frames.shape[2], frames.shape[1], FPS)
            y, bgr = decode(path)
            assert y.shape[0] == len(frames), name
            out[f'{name}/mp4'] = np.frombuffer(open(path, 'rb').read(), np.uint8)
            out[f'{name}/y_sha256'] = np.stack([digest(p) for p in y])
            out[f'{name}/y'] = y[:, :WINDOW, :WINDOW]
            out[f'{name}/bgr'] = bgr[:, :WINDOW, :WINDOW]
            print(name, qp, frames.shape, len(out[f'{name}/mp4']), 'bytes', flush=True)
    assert epb > 0, 'no emulation-prevention byte in the corpus'
    print('emulation-prevention bytes', epb)
    np.savez_compressed(os.path.join(HERE, 'reference_h264_v1.npz'), **out)


if __name__ == '__main__':
    main()
