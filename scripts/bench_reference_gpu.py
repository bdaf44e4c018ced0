"""The "reference-style GPU path" of BASELINE.md section 3: the oracle port run in eager PyTorch ON the GPU with the
reference's own structure -- python chunk loop of 90 000 rays (`--batch 90000`), one autograd `grid_sample` field query
per chunk, `cumprod` compositing, and the max-depth step on the CPU (neus_head.py:329-374, 430-438).  It stands in for
"the reference GPU path" (the reference itself cannot be installed offline) in the north-star's >= 10x comparison.
Render only (that is what the reference's eval spends its time on); 1 camera x 900 x 1600 rays, scaled x6.
    python scripts/bench_reference_gpu.py   -> one JSON line"""
import json, os, sys, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.mapping import GridMeterMappingRef
from oracle import render as orender, rays as orays
from selfocc_b200 import synth

dev = torch.device('cuda:0')
mref = GridMeterMappingRef(**synth.NUSC_MAPPING)
H, W, Z = mref.size_h, mref.size_w, mref.size_d
g = torch.Generator().manual_seed(0)
vol = (0.3 * torch.randn(1, H, W, Z, generator=g)).to(dev)
_, i2l = synth.camera_rig()
i2l = torch.tensor(np.asarray(i2l), dtype=torch.float32, device=dev)[None, :1]
pix = orays.fixed_ray_grid([900, 1600], [900, 1600]).to(dev)
origin, direction = orays.img2lidar_rays(i2l, pix)


def run():
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = orender.head_render_ref(vol, mref, origin, direction, synth.NUSC_RANGE, 20.0, batch=90000, S=256, max_depth_on_cpu=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


run()
ts = [run()[0] for _ in range(2)]
t = min(ts)
rays = 900 * 1600
print(json.dumps({'impl': 'reference-style eager PyTorch on the GPU (oracle port, chunked 90000 rays, CPU max-depth)',
                  'rays': rays, 'seconds': t, 'rays_per_s_render_only': rays / t,
                  'frame_ms_extrapolated_6cams': 6 * t * 1e3}))
