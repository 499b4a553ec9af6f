"""A/B timing of the variant-P renderer (`ssdnerf_render_fwd`) on bench.py's render workload, two builds of the library in one process.

    python tests/perf/render_p_timing.py --baseline-lib OLD.so [--lib NEW.so] [--reps 7] [--warmup 2] [--out result.json]

Inputs are built the way bench.py builds them: the cars config model (seed 0), the rank-0 noise (seed 1234), the 50-step DDIM sample,
the occupancy bitfield from `get_density` and 16 scenes x 251 orbit views x 128^2 rays.  Both libraries (`--lib` defaults to the
working tree's) are loaded with ctypes and get identical inputs; after warm-up the two are called alternately `--reps` times, each call
timed with CUDA events.  Reported per library: ms per render, rays/s and SM-cycles per composited sample (at the SM clock read from
nvidia-smi right after the timed calls), with min / median / max over the reps; then the largest differences of `image`, `depth` and
`weights_sum` between the two and whether every ray's `num_samples` is identical.  The card's name and power limit are read in the
same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from ssdnerf_b200 import _lib as N  # noqa: E402
from ssdnerf_b200 import renderer as R  # noqa: E402
import bench  # noqa: E402


def load(path):
    L = ctypes.CDLL(os.path.abspath(path))
    L.ssdnerf_last_error.restype = ctypes.c_char_p
    L.ssdnerf_render_workspace_bytes.restype = ctypes.c_size_t
    return L


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), f'--query-gpu={q}', '--format=csv,noheader,nounits'],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    f = [x.strip() for x in out.split(',')]
    return dict(name=f[0], power_limit_w=float(f[1]), sm_mhz=float(f[2]), sm_max_mhz=float(f[3]))


class Call:
    """one library's ssdnerf_render_fwd on fixed inputs, writing into its own output buffers"""

    def __init__(self, L, inp):
        self.L = L
        B, V, h, w = inp['B'], inp['V'], inp['h'], inp['w']
        n = V * h * w
        dev = inp['planes'].device
        f32 = dict(dtype=torch.float32, device=dev)
        self.out = dict(weights_sum=torch.empty(B, n, **f32), depth=torch.empty(B, n, **f32), image=torch.empty(B, n, 3, **f32),
                        rgb=torch.empty(B, n, 3, **f32), num_samples=torch.empty(B, n, dtype=torch.int32, device=dev))
        ws = L.ssdnerf_render_workspace_bytes(N.c_u32(B), N.c_u32(n), N.c_u32(inp['max_steps']))
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=dev)
        a = N.RenderArgs()
        a.variant = R.DEC_P
        a.num_scenes, a.rays_per_scene = B, n
        a.poses, a.intrinsics = N.ptr(inp['poses']), N.ptr(inp['intr'])
        a.num_views, a.img_h, a.img_w = V, h, w
        a.planes, a.plane_h, a.plane_w = N.ptr(inp['planes']), 128, 128
        a.bitfield, a.grid_size = N.ptr(inp['bitfield']), inp['grid_size']
        a.decoder_blob, a.dt_gamma = N.ptr(inp['blob']), N.ptr(inp['dt_gamma'])
        a.bound, a.min_near, a.T_thresh, a.bg_color = inp['bound'], inp['min_near'], 1e-4, inp['bg_color']
        a.max_steps, a.emulate_schedule = inp['max_steps'], 1
        a.weights_sum, a.depth, a.image = N.ptr(self.out['weights_sum']), N.ptr(self.out['depth']), N.ptr(self.out['image'])
        a.rgb_blend, a.num_samples = N.ptr(self.out['rgb']), N.ptr(self.out['num_samples'])
        a.voxel_trace, a.trace_cap = None, 0
        a.workspace, a.workspace_bytes = N.ptr(self.workspace), ws
        self.args = a

    def __call__(self):
        e = self.L.ssdnerf_render_fwd(ctypes.byref(self.args), N.stream_ptr())
        if e != 0:
            raise N.SSDNeRFNativeError(f'render_fwd error {e}: {self.L.ssdnerf_last_error().decode()}')


def workload(dev):
    model, _ = bench.build_model(dev, seed=0)
    diffusion, decoder = model.diffusion_ema, model.decoder_ema
    B, V, IMG = bench.B_PER_GPU, bench.NUM_VIEWS, bench.IMG
    g = torch.Generator().manual_seed(1234)
    noise = torch.randn(B, *model.code_size, generator=g).to(dev)
    poses = bench.orbit_poses(V)[None].repeat(B, 1, 1, 1).contiguous().to(dev)
    intr = torch.tensor([131.25, 131.25, 64.0, 64.0]).expand(B, V, 4).contiguous().to(dev)
    with torch.no_grad():
        code = model.code_diff_pr_inv(diffusion(model.code_diff_pr(noise), return_loss=False)).contiguous()
        _, bitfield = model.get_density(decoder, code, cfg=model.test_cfg)
    variant = decoder.fused_variant()
    assert variant == R.DEC_P, 'the bench decoder is expected to be variant P'
    dt_scale = model.test_cfg.get('dt_gamma_scale', 0.0)
    dt_gamma = dt_scale * 2 / (intr[..., 0] + intr[..., 1]).mean(dim=-1) if dt_scale != 0 else None
    return dict(B=B, V=V, h=IMG, w=IMG, planes=R.pack_planes(code, variant), bitfield=bitfield.reshape(B, -1).contiguous(),
                blob=decoder.packed_blob(), poses=poses, intr=intr, dt_gamma=None if dt_gamma is None else dt_gamma.float().contiguous(),
                grid_size=int(model.grid_size), bound=float(decoder.bound), min_near=float(decoder.min_near),
                max_steps=int(decoder.max_steps), bg_color=float(model.bg_color))


def spread(v):
    return dict(min=float(np.min(v)), median=float(np.median(v)), max=float(np.max(v)))


def diff(a, b):
    d = (a - b).abs()
    rel = d / b.abs().clamp_min(1e-30)
    over = (d > 2e-5) & (d > 2e-4 * b.abs())
    big = d > 2e-5
    return dict(max_abs=float(d.max()), max_rel_where_abs_over_2e_5=float(rel[big].max()) if bool(big.any()) else 0.0,
                count_over_both_bars=int(over.sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-lib', required=True)
    ap.add_argument('--lib', default=os.path.join(ROOT, 'ssdnerf_b200', 'libssdnerf_b200.so'))
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('render_p_timing.py needs a CUDA device')
    assert os.path.realpath(args.lib) != os.path.realpath(args.baseline_lib), 'the two libraries must be different files'
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    inp = workload(dev)
    calls = {'new': Call(load(args.lib), inp), 'baseline': Call(load(args.baseline_lib), inp)}
    for _ in range(args.warmup):
        for c in calls.values():
            c()
    torch.cuda.synchronize()
    ms = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, c in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            c()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    gpu = gpu_info()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rays = inp['B'] * inp['V'] * inp['h'] * inp['w']
    res = dict(gpu=gpu, sms=sms, rays=rays, lib=args.lib, baseline_lib=args.baseline_lib, reps=args.reps)
    for k, c in calls.items():
        samples = int(c.out['num_samples'].sum(dtype=torch.int64))
        v = np.array(ms[k])
        res[k] = dict(samples=samples, samples_per_ray=samples / rays, ms=spread(v), rays_per_s=spread(rays / (v * 1e-3)),
                      sm_cycles_per_sample=spread(v * 1e-3 * gpu['sm_mhz'] * 1e6 * sms / samples), ms_all=[float(x) for x in v])
    res['speedup_median'] = res['baseline']['ms']['median'] / res['new']['ms']['median']
    res['speedup_worst'] = res['baseline']['ms']['min'] / res['new']['ms']['max']
    a, b = calls['new'].out, calls['baseline'].out
    res['num_samples_identical'] = bool(torch.equal(a['num_samples'], b['num_samples']))
    res['num_samples_mismatched_rays'] = int((a['num_samples'] != b['num_samples']).sum())
    res['diff'] = {k: diff(a[k], b[k]) for k in ('image', 'depth', 'weights_sum', 'rgb')}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
