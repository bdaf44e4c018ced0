"""Device timing of the training-form render kernels at BASELINE configs[4] sizes (nuScenes_occ training step:
6 cams x 48 x 100 rays x 256 samples, TPV 257x257x25, Cf = 1 + 24) -> one JSON line with achieved GB/s against
the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).  python scripts/bench_train_render.py [--cf 25|1]"""
import argparse, json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfocc_b200 import ops, synth, _lib
from selfocc_b200.mapping import GridMeterMapping

ap = argparse.ArgumentParser()
ap.add_argument('--cf', type=int, default=25)
ap.add_argument('--iters', type=int, default=20)
ap.add_argument('--fwd-only', action='store_true', help='time the forward kernel only (no backward pass)')
ap.add_argument('--fwd32', action='store_true', help='force the 32-samples-per-warp-step forward kernel')
ap.add_argument('--no-pair', action='store_true', help='gather from the sdf volume itself (no z-pair repack)')
ap.add_argument('--tag', default='')
ap.add_argument('--frames', type=int, default=1, help='temporal frames rendered in ONE launch (neus_head.py:513-531 renders curr + prev + next: 3 x 6 cameras)')
a = ap.parse_args()
dev = torch.device('cuda:0')
margs = dict(synth.NUSC_MAPPING, d_size=[24, 0], d_range=[-4.0, 4.0, 4.0])
aabb = [-51.2, -51.2, -4.0, 51.2, 51.2, 4.0]
m = GridMeterMapping(**margs)
n_feat = a.cf - 1
desc = m.volume_desc(n_feat)
g = torch.Generator().manual_seed(0)
sdf = synth.analytic_sdf_volume(m, noise=0.02)
vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev).requires_grad_(True)
vf = (0.5 * torch.randn(desc.H, desc.W, desc.Z, desc.feat_pitch, generator=g)).to(dev).requires_grad_(True) if n_feat else None
_, i2l = synth.camera_rig()
i2l = torch.tensor(i2l, dtype=torch.float32, device=dev).repeat(a.frames, 1, 1)
for f in range(a.frames):                    # the temporal frames: the rig displaced along y
    i2l[6 * f:6 * f + 6, 1, 3] += 0.8 * f
ncam = 6 * a.frames
ny, nx, S = 48, 100, 256
n = ncam * ny * nx
jit = torch.rand(n, S + 1, device=dev)
bk = torch.rand(n, 3, device=dev)
invs = torch.tensor([20.0], device=dev, requires_grad=True)
want = ['depth', 'acc', 'fars', 'weights', 'ts', 'deltas', 'eik_grad'] + (['rgb'] if n_feat >= 3 else []) + (['sem'] if n_feat > 3 else [])
cfg = dict(desc=desc, cam_mats=i2l, rays=ops.make_ray_desc(ncam, grid=(ny, nx, 16.0, 3.0, 16.0, 5.0)),
           params=ops.make_render_params(aabb, S, 20.0, training=True, bkgd='random' if n_feat else 'white'), jitter=jit,
           bkgd_rand=bk if n_feat else None, want=want, zpair=not a.no_pair)
_lib.profile_enable(True)
if a.fwd32:
    _lib.load().so_render_train_force_fwd32(1)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for it in range(a.iters + 3):
    if it == 3:
        torch.cuda.synchronize(); _lib.profile_reset()
    flush.zero_()
    res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, cfg)))
    loss = res['depth'].sum() + res['weights'].sum() + res['eik_grad'].sum() + (res['rgb'].sum() if n_feat >= 3 else 0) \
        + (res['sem'].sum() if n_feat > 3 else 0)
    if not a.fwd_only:
        loss.backward()
torch.cuda.synchronize()
prof = _lib.profile_read()
peak = 3350.0                                # H100 SXM data sheet, HBM3
fwd_ms = prof['render_train_fwd'][0] / prof['render_train_fwd'][1]
bwd_ms = prof['render_train_bwd'][0] / max(prof['render_train_bwd'][1], 1) if 'render_train_bwd' in prof else float('nan')
out_bytes = n * (S * (4 + 4 + 4 + 12) + 4 * 3 + (12 if n_feat >= 3 else 0) + 4 * max(n_feat - 3, 0))
in_bytes = n * (S + 1) * 4 + desc.H * desc.W * desc.zpitch * 4 + (desc.H * desc.W * desc.Z * desc.feat_pitch * 4 if n_feat else 0)
fwd_gbs = (out_bytes + in_bytes) / (fwd_ms * 1e-3) / 1e9
print(json.dumps({'kernel': 'render_train_fwd_kernel' if a.fwd32 else 'render_train_fwd5_kernel (+ zpair_pack_kernel)', 'tag': a.tag, 'lib': os.environ.get('SELFOCC_B200_LIB', 'default'), 'workload': 'nuscenes_occ_train %dx48x100 rays x256, Cf=%d' % (ncam, a.cf),
                  'rays': n, 'fwd_ms': fwd_ms, 'bwd_ms': bwd_ms, 'algorithmic_bytes_fwd': out_bytes + in_bytes,
                  'roofline': {'bound': 'hbm', 'achieved': fwd_gbs, 'peak': peak, 'unit': 'GB/s', 'frac': fwd_gbs / peak},
                  'rays_per_s_fwd': n / (fwd_ms * 1e-3), 'rays_per_s_fwd_bwd': n / ((fwd_ms + bwd_ms) * 1e-3)}))
