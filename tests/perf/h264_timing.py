"""Time the H.264 export of `python -m ssdnerf_b200.orbit --format mp4` at the GUI's defaults (120 frames of 256 x 256, QP 20) and
set it against the Motion-JPEG AVI path (quality 95) in the same run:
  * encode: the C ABI's ssdnerf_h264_encode_f32 of 120 fp32 render-like frames into preallocated buffers (CUDA events around the
    launch sequence), and `video.encode_h264` of the same frames (host clock, the copy of the access units to the host included);
  * split of one orbit of one scene (the scene of tests/perf/orbit_timing.py): render (`orbit.render_frames` in batches of 30, CUDA
    events), encode (host clock, copy included) and the file write (host clock, temporary dir), for mp4 and for avi;
  * file size and PSNR of the decoded RGB against the u8 frames for mp4 at QP 20 / 23 / 26 and avi at quality 95: the MP4 frames
    are the decoder's planes (oracle/h264_port.py's deblocked reconstruction, equal to FFmpeg's decode on the test corpus) in
    BT.601 limited range to RGB with nearest chroma, the AVI frames cv2.imdecode's ("not measured" without cv2).
Rounds after one warm-up; prints one JSON line with the card's name, power limit and max SM clock read in the same run.
Run from the repository root: python tests/perf/h264_timing.py [--rounds R]"""
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
from ssdnerf_b200 import _lib as N
from ssdnerf_b200 import orbit, video
from tests.perf.orbit_timing import FRAMES, RES, QUALITY, BATCH, GOLDEN, frames_like_renders, timed

QP = 20


def psnr(decoded_rgb, u8):
    err = np.mean([((d.astype(np.float64) - s) ** 2).mean() for d, s in zip(decoded_rgb, u8)])
    return round(float(10 * np.log10(255 ** 2 / err)), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    dev = torch.device('cuda:0')
    frames = frames_like_renders(FRAMES, RES, dev)
    u8 = np.round(frames.cpu().numpy() * 255).astype(np.uint8)
    res = dict(gpu=gpu, frames=FRAMES, res=RES, qp=QP, quality=QUALITY, rounds=args.rounds)
    # --- encode alone: device time through the C ABI, then the Python call with its copy
    L, n = N.lib(), FRAMES
    ws, ob = L.ssdnerf_h264_workspace_bytes(n, RES, RES), L.ssdnerf_h264_output_bound(n, RES, RES)
    work = torch.empty(ws, dtype=torch.uint8, device=dev)
    out = torch.empty(ob, dtype=torch.uint8, device=dev)
    offs = torch.empty(n + 3, dtype=torch.int64, device=dev)
    dev_ms, wall_ms = [], []
    for r in range(args.rounds + 1):
        _, ms = timed(lambda: N.check(L.ssdnerf_h264_encode_f32(N.ptr(frames), n, RES, RES, QP, 30, 1, 0, N.ptr(work), ws, N.ptr(out),
                                                                ob, N.ptr(offs), N.stream_ptr())))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        enc = video.encode_h264(frames, QP, 30)
        wall = (time.perf_counter() - t0) * 1e3
        if r:
            dev_ms.append(round(ms, 2))
            wall_ms.append(round(wall, 2))
    res['h264_encode_120_device_ms'] = dev_ms
    res['h264_encode_120_ms'] = wall_ms
    res['h264_bytes_mean'] = int(np.mean([len(a) for a in enc[2]]))
    # --- one orbit: render, encode, write, mp4 against avi
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
    split = {f'{k}_{f}': [] for f in ('mp4', 'avi') for k in ('render_ms', 'encode_ms', 'write_ms')}
    with tempfile.TemporaryDirectory() as d:
        for r in range(args.rounds + 1):
            for fmt in ('mp4', 'avi'):                   # alternated within a round
                t_r = t_e = 0.0
                payload = []
                for lo in range(0, FRAMES, BATCH):
                    img, ms = timed(lambda: orbit.render_frames(model, code, bitfield, poses[lo:lo + BATCH], intr, hw))
                    t_r += ms
                    t0 = time.perf_counter()
                    if fmt == 'mp4':
                        sps, pps, aus = video.encode_h264(img, QP, 30, first_frame=lo)
                        payload += aus
                    else:
                        payload += video.encode_jpeg(img, QUALITY)
                    t_e += (time.perf_counter() - t0) * 1e3
                t0 = time.perf_counter()
                if fmt == 'mp4':
                    video.write_mp4(os.path.join(d, 'o.mp4'), sps, pps, payload, hw[1], hw[0], 30)
                else:
                    video.write_avi(os.path.join(d, 'o.avi'), payload, hw[1], hw[0], 30)
                t_w = (time.perf_counter() - t0) * 1e3
                if r:
                    split[f'render_ms_{fmt}'].append(round(t_r, 2))
                    split[f'encode_ms_{fmt}'].append(round(t_e, 2))
                    split[f'write_ms_{fmt}'].append(round(t_w, 2))
        res['orbit_split'] = split
        # --- size and quality on the render-like frames
        from oracle import h264_port as H
        from tests.test_h264_cpu import bgr_of
        quality = {}
        for qp in (20, 23, 26):
            p = os.path.join(d, f'q{qp}.mp4')
            sps, pps, aus = video.encode_h264(frames, qp, 30)
            video.write_mp4(p, sps, pps, aus, RES, RES, 30)
            dec = [bgr_of(*H.decoded_planes(u8[i], qp, i & 1))[..., ::-1] for i in range(FRAMES)]
            quality[f'mp4_qp{qp}'] = dict(bytes=os.path.getsize(p), psnr_db=psnr(dec, u8))
        p = os.path.join(d, 'q95.avi')
        jpegs = video.encode_jpeg(frames, QUALITY)
        video.write_avi(p, jpegs, RES, RES, 30)
        quality['avi_q95'] = dict(bytes=os.path.getsize(p))
        try:
            import cv2
            dec = [cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR)[..., ::-1] for j in jpegs]
            quality['avi_q95']['psnr_db'] = psnr(dec, u8)
        except ImportError:
            quality['avi_q95']['psnr_db'] = 'cv2 not importable: not measured'
        res['size_quality'] = quality
    print(json.dumps(res))


if __name__ == '__main__':
    main()
