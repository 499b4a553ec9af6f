"""Time mesh export per scene over the bench's 16 scenes at the reference's default 256^3 lattice: `extract_fields` (density lattice,
CUDA events), `mesh.marching_cubes` (host clock around the synchronised count / read / emit), the copy to the host with the world mapping
of `extract_geometry`, and `mesh.write_stl` (host clock, to a temporary directory).  Random P-decoder weights; two kinds of random codes,
since the cost after the lattice scales with the triangle count: `smooth` (noise on an 8 x 8 grid, bilinearly upsampled to 128 x 128:
an object-like surface) and `rough` (independent noise per texel: a surface folded at every lattice cell).  The threshold is the 60 %
quantile of the positive densities of the first scene.  Prints one JSON line per kind with the card's name, power limit and max SM clock
read in the same run.  Run from the repository root: python tests/perf/mesh_timing.py"""
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
from oracle import render_port as rp
from ssdnerf_b200 import mesh
from ssdnerf_b200.nerf import extract_fields

SCENES, RES = 16, 256


def run(dec, codes, kind, gpu):
    with torch.no_grad():
        u0 = extract_fields(dec, codes[0], RES)
    thr = float(torch.quantile(u0[u0 > 0][:1 << 24].float(), 0.6))
    lo, hi = (dec.aabb[:3] - 0.1).cpu().numpy(), (dec.aabb[3:] + 0.1).cpu().numpy()
    t_fields, t_mc, t_host, t_stl, tris, verts = [], [], [], [], [], []
    with tempfile.TemporaryDirectory() as d, torch.no_grad():
        for i in range(-1, SCENES):                          # scene -1: warm-up of every step, not recorded
            code = codes[max(i, 0)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            u = extract_fields(dec, code, RES)
            e1.record()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            v, t = mesh.marching_cubes(u, thr)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            vn, tn = v.cpu().numpy(), t.cpu().numpy()
            vn = vn / (RES - 1.0) * (hi - lo)[None, :] + lo[None, :]
            t2 = time.perf_counter()
            mesh.write_stl(os.path.join(d, f'{i}.stl'), vn, tn)
            t3 = time.perf_counter()
            if i >= 0:
                t_fields.append(e0.elapsed_time(e1))
                t_mc.append((t1 - t0) * 1e3)
                t_host.append((t2 - t1) * 1e3)
                t_stl.append((t3 - t2) * 1e3)
                tris.append(len(tn))
                verts.append(len(vn))
    ms = lambda x: round(float(np.mean(x)), 3)
    return dict(kind=kind, scenes=SCENES, resolution=RES, threshold=round(thr, 4), triangles_mean=int(np.mean(tris)),
                vertices_mean=int(np.mean(verts)), extract_fields_ms=ms(t_fields), marching_cubes_ms=ms(t_mc),
                marching_cubes_ms_max=round(float(np.max(t_mc)), 3), to_host_world_ms=ms(t_host), write_stl_ms=ms(t_stl), gpu=gpu)


def main():
    dev = torch.device('cuda:0')
    dec = S.build_module(dict(type='TriPlaneDecoder', base_layers=[18, 64], density_layers=[64, 1], color_layers=[64, 3], use_dir_enc=True,
                              dir_layers=[16, 64], max_steps=256))
    sd = dec.state_dict(); sd.update(rp.make_decoder_params('P', 7)); dec.load_state_dict(sd)
    dec = dec.to(dev).eval()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    g = torch.Generator().manual_seed(0)
    coarse = torch.randn(SCENES * 3, 6, 8, 8, generator=g) * 1.5
    smooth = torch.nn.functional.interpolate(coarse, size=(128, 128), mode='bilinear', align_corners=True).reshape(SCENES, 3, 6, 128, 128)
    rough = (torch.randn(SCENES, 3, 6, 128, 128, generator=g) * 0.7).clamp(-2, 2)
    for kind, codes in (('smooth', smooth), ('rough', rough)):
        print(json.dumps(run(dec, codes.clamp(-2, 2).contiguous().to(dev), kind, gpu)), flush=True)


if __name__ == '__main__':
    main()
