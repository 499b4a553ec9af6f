"""Time the orbit export of `python -m ssdnerf_b200.orbit` at the GUI's defaults (120 frames of 256 x 256, quality 95):
  * encode: `video.encode_jpeg` of 120 fp32 render-like frames in one call (CUDA events around the launch sequence, then the host copy
    of the files with a host clock), against `cv2.imencode` of the same u8 frames on one host thread when cv2 imports;
  * split of one orbit of one scene (cars unconditional model, random decoder weights, a smooth random code and its occupancy grid):
    render (`orbit.render_frames` in batches of 30, CUDA events), encode (events + copy) and the AVI write (host clock, temporary dir).
Rounds after one warm-up; prints one JSON line with the card's name, power limit and max SM clock read in the same run.
Run from the repository root: python tests/perf/orbit_timing.py [--rounds R]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch

import ssdnerf_b200 as S
from ssdnerf_b200 import orbit, video

FRAMES, RES, QUALITY, BATCH = 120, 256, 95, 30
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'golden')


def frames_like_renders(n, res, dev):
    """fp32 [n, res, res, 3]: shaded ellipses over white with a soft edge, moving over the sequence"""
    y, x = torch.meshgrid(torch.arange(res, device=dev, dtype=torch.float32), torch.arange(res, device=dev, dtype=torch.float32),
                          indexing='ij')
    out = []
    for k in range(n):
        cx, cy = float(res * (0.5 + 0.1 * np.cos(k / 9))), float(res * (0.5 + 0.1 * np.sin(k / 7)))
        d = ((x - cx) / (0.3 * res)) ** 2 + ((y - cy) / (0.22 * res)) ** 2
        base = torch.tensor([0.7, 0.25 + 0.2 * float(np.sin(k / 13)), 0.2], device=dev)
        shade = (1 - 0.5 * d)[..., None] * base + 0.04 * torch.sin(x / 5 + y / 9 + k)[..., None]
        a = (1.5 - d).clamp(0, 1)[..., None]
        out.append((a * shade + (1 - a)).clamp(-0.001, 1.001).float())
    return torch.stack(out)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def encode_ms(frames):
    """(files, CUDA-event ms around encode_jpeg, host-clock ms of the same call): both include the copy of the files to the host"""
    t0 = time.perf_counter()
    files, ms = timed(lambda: video.encode_jpeg(frames, QUALITY))
    return files, ms, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    dev = torch.device('cuda:0')
    frames = frames_like_renders(FRAMES, RES, dev)
    u8 = np.round(frames.cpu().numpy() * 255).astype(np.uint8)
    res = dict(gpu=gpu, frames=FRAMES, res=RES, quality=QUALITY, rounds=args.rounds)
    # --- encode alone
    enc, enc_dev = [], []
    for r in range(args.rounds + 1):
        files, ms, wall = encode_ms(frames)
        if r:
            enc.append(wall)
            enc_dev.append(ms)
    res['encode_120_ms'] = [round(x, 2) for x in enc]
    res['encode_120_device_ms'] = [round(x, 2) for x in enc_dev]
    res['jpeg_bytes_mean'] = int(np.mean([len(f) for f in files]))
    try:
        import cv2
        cv2.setNumThreads(1)
        bgr = [np.ascontiguousarray(f[..., ::-1]) for f in u8]
        cpu = []
        for r in range(args.rounds + 1):
            t0 = time.perf_counter()
            ref = [cv2.imencode('.jpg', b, [cv2.IMWRITE_JPEG_QUALITY, QUALITY])[1].tobytes() for b in bgr]
            if r:
                cpu.append((time.perf_counter() - t0) * 1e3)
        res['cv2_imencode_120_ms_one_thread'] = [round(x, 2) for x in cpu]
        res['cv2_bytes_equal'] = ref == files
    except ImportError:
        res['cv2_imencode_120_ms_one_thread'] = 'cv2 not importable: not measured'
    # --- one orbit: render, encode, write
    c = json.load(open(os.path.join(GOLDEN, 'reference_configs.json')))['configs/paper_cfgs/ssdnerf_cars_uncond.py']
    torch.manual_seed(0)
    model = S.build_model(c['model'], train_cfg=c['train_cfg'], test_cfg=c['test_cfg']).to(dev).eval()
    g = torch.Generator().manual_seed(1)
    coarse = torch.randn(3 * 6, 1, 8, 8, generator=g) * 1.5
    code = torch.nn.functional.interpolate(coarse, size=(128, 128), mode='bilinear', align_corners=True).reshape(3, 6, 128, 128).to(dev)
    _, bitfield = model.get_density(model.decoder_ema, code[None], cfg=dict(density_thresh=0.1, density_step=16))
    bitfield = bitfield[0]
    pose = torch.from_numpy(np.load(os.path.join(GOLDEN, 'reference_video_v1.npz'))['gui_pose'])
    poses = video.surround_views(pose, num_frames=FRAMES)
    intr, hw = torch.tensor([131.25, 131.25, 64.0, 64.0]) * (RES / 128), (RES, RES)
    split = dict(render_ms=[], encode_ms=[], write_ms=[])
    with tempfile.TemporaryDirectory() as d:
        for r in range(args.rounds + 1):
            t_r = t_e = 0.0
            jpegs = []
            for lo in range(0, FRAMES, BATCH):
                img, ms = timed(lambda: orbit.render_frames(model, code, bitfield, poses[lo:lo + BATCH], intr, hw))
                t_r += ms
                files, _, wall = encode_ms(img)
                t_e += wall
                jpegs += files
            t0 = time.perf_counter()
            video.write_avi(os.path.join(d, 'o.avi'), jpegs, hw[1], hw[0], 30)
            t_w = (time.perf_counter() - t0) * 1e3
            if r:
                split['render_ms'].append(round(t_r, 2))
                split['encode_ms'].append(round(t_e, 2))
                split['write_ms'].append(round(t_w, 2))
    res['orbit_split'] = split
    res['orbit_avi_bytes'] = sum(len(j) for j in jpegs)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
