"""GPU: novel-view depth evaluation (so_novel_depth_errors, selfocc_b200.metric.NovelDepthMetric) against the fp64 oracle at
both shipped geometries and on the golden fixture's ragged edge cases, its sampling against metric.depth_sample, run-to-run
bit identity, render_poses + NovelDepthMetric against the reference's per-source loop on head.render outputs, and a frame's
step without a host synchronisation."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import novel_depth as ond
from selfocc_b200.metric import NovelDepthMetric, depth_sample, novel_depth_errors, pack_novel_depth

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden_novel_depth.npz'))

# Kernel vs fp64 oracle, per metric.  The per-point terms are fp32 (as the reference computes them) and summed in fp64:
# relative error a few fp32 ulps.  a1-a3 compare thresh = max(gt / pred, pred / gt) in fp32 against the thresholds: a
# point within an ulp of a threshold may count on the other side than in fp64, one point in the segment's count.
RTOL = dict(abs_rel=2e-6, sq_rel=2e-6, rmse=2e-6, rmse_log=2e-6)
FLIPS = dict(a1=1, a2=1, a3=1)

# (cameras, eval ray grid h x w, source poses, LiDAR points per source) of eval_novel_depth.py (nuscenes_novel_depth.py,
# --num-rays 96 200) and eval_novel_depth_kitti.py (kitti_novel_depth.py, the 'kitti' eval grid 176 x 608)
GEOMETRIES = {'nuscenes': (6, 96, 200, 5, 34720), 'kitti': (1, 176, 608, 4, 19000)}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def loader_frame(N, h, w, S, n, seed=0, dists=None):
    """Depth maps [S, N, h, w] and loader-shaped metas: every LiDAR point projected into every camera (float64 locations,
    a few beyond [0, 1]), about a sixth of them in front of a given camera (the mask), ground truth in (1, 80)."""
    g = np.random.default_rng(seed)
    maps = torch.from_numpy((g.random((S, N, h, w)) * 60 + 0.5).astype(np.float32))
    meta = dict(depth_loc=[], depth_gt=[], depth_mask=[],
                frame_dists=list(dists) if dists is not None else list(g.random(S) * 6))
    for s in range(S):
        loc = g.random((N, n, 2)) * 1.1 - 0.05
        gt = g.random((N, n)) * 79 + 1.0
        gt[:, ::3] = maps[s, :, 0, 0].numpy()[:, None] * (1 + 0.3 * g.standard_normal((N, 1)))  # near the prediction
        meta['depth_loc'].append(loc)
        meta['depth_gt'].append(np.abs(gt) + 0.5)
        meta['depth_mask'].append((g.random((N, n)) < (1.0 if N == 1 else 1 / 6)) & (loc > 0).all(-1) & (loc < 1).all(-1))
    return maps, meta


def kernel_frame(maps, meta, dev):
    """One frame through pack_novel_depth and so_novel_depth_errors -> [S, N, 7] on the device."""
    S, N, h, w = maps.shape
    buf, lay = pack_novel_depth(meta, N, 1000)
    d = buf.to(dev)
    part = lambda name, dt: d[lay[name][0]:lay[name][0] + lay[name][1]].view(dt)
    o0, ob = lay['offsets']
    T = lay['T']
    err = novel_depth_errors(maps.reshape(S * N, h, w).to(dev), part('offsets', torch.int64), part('loc', torch.float32).view(T, 2),
                             part('gt', torch.float32), part('mask', torch.uint8), offsets_host=buf[o0:o0 + ob].view(torch.int64))
    return err.view(S, N, 7)


def assert_close_to_oracle(got, maps, meta):
    got = got.cpu().double()
    for s, (_, ref) in enumerate(ond.frame_errors_ref(maps, meta)):
        count = torch.as_tensor(meta['depth_mask'][s]).sum(-1).double()
        assert torch.equal(torch.isnan(got[s]), torch.isnan(ref)), s           # NaN exactly where a segment is empty
        for j, key in enumerate(ond.KEYS):
            g, r = got[s, :, j], ref[:, j]
            ok = ~torch.isnan(r)
            if key in RTOL:
                bad = ((g - r).abs() > RTOL[key] * r.abs() + 1e-12) & ok
            else:
                bad = ((g - r).abs() * count > FLIPS[key] + 1e-3) & ok
            assert not bad.any(), (s, key, g[bad], r[bad])


@pytest.mark.parametrize('name', sorted(GEOMETRIES))
def test_kernel_matches_oracle_at_shipped_geometry(name):
    dev = _dev()
    N, h, w, S, n = GEOMETRIES[name]
    maps, meta = loader_frame(N, h, w, S, n, seed=len(name))
    meta['depth_mask'][1][0] = False                                   # one empty (pose, camera) segment
    got = kernel_frame(maps, meta, dev)
    assert torch.isnan(got[1, 0]).all() and not torch.isnan(got[0]).any()
    counts = np.concatenate([m.sum(-1) for m in meta['depth_mask']])
    assert counts[counts > 0].min() > (500 if N > 1 else 10000)            # thousands of points per camera
    assert_close_to_oracle(got, maps, meta)


def test_kernel_on_ragged_edge_cases():
    """The golden fixture (locations at 0, 1, on cell edges and beyond, an empty camera, clamped predictions) against the
    oracle and the reference's fp32 numbers; plus sources with no point at all (zero-length segments)."""
    dev = _dev()
    for f in range(3):
        dists = [float(d) for d in G['f%d_dists' % f]]
        meta = {k: [G['f%d_s%d_%s' % (f, s, k)] for s in range(len(dists))] for k in ('depth_loc', 'depth_gt', 'depth_mask')}
        meta['frame_dists'] = dists
        maps = torch.from_numpy(G['f%d_maps' % f])
        got = kernel_frame(maps, meta, dev)
        assert_close_to_oracle(got, maps, meta)
        for s in range(len(dists)):
            assert np.allclose(got[s].cpu().numpy(), G['f%d_s%d_errors' % (f, s)], rtol=1e-5, atol=1e-6, equal_nan=True)
    maps, meta = loader_frame(3, 7, 9, 3, 50, seed=4)
    for k in ('depth_loc', 'depth_gt', 'depth_mask'):
        meta[k][1] = meta[k][1][:, :0]
    got = kernel_frame(maps, meta, dev)
    assert torch.isnan(got[1]).all() and not torch.isnan(got[0]).any() and not torch.isnan(got[2]).any()
    assert_close_to_oracle(got, maps, meta)


def test_sampling_is_bit_identical_to_depth_sample():
    """Ground truth set to metric.depth_sample's value at every point: the segment's abs_rel (a sum of |gt - pred| / gt
    over all points) is exactly 0 only if every sampled value is bit for bit the same."""
    dev = _dev()
    N, h, w, n = 6, 96, 200, 3000
    g = torch.Generator().manual_seed(7)
    maps = (torch.rand(N, h, w, generator=g) * 60 + 0.5).to(dev)
    loc = torch.rand(N, n, 2, generator=g) * 1.2 - 0.1
    loc[:, :8] = torch.tensor([[0, 0], [1, 1], [0, 1], [1, 0], [1 / 199, 1 / 95], [0.5, 0.5], [-1, 2], [1.0 - 1e-7, 1e-7]])
    loc = loc.to(dev)
    sampled = depth_sample(maps, loc)
    offsets = torch.arange(N + 1, dtype=torch.int64) * n
    err = novel_depth_errors(maps, offsets.to(dev), loc.reshape(-1, 2), sampled.reshape(-1),
                             torch.ones(N * n, dtype=torch.uint8, device=dev), offsets_host=offsets)
    assert torch.equal(err[:, :4].cpu(), torch.zeros(N, 4)) and torch.equal(err[:, 4:].cpu(), torch.ones(N, 3))
    sampled[0, 5] = torch.nextafter(sampled[0, 5], torch.tensor(100.0, device=dev))   # one ulp off: seen
    err = novel_depth_errors(maps, offsets.to(dev), loc.reshape(-1, 2), sampled.reshape(-1),
                             torch.ones(N * n, dtype=torch.uint8, device=dev), offsets_host=offsets)
    assert err[0, 0] > 0 and torch.equal(err[1:, 0].cpu(), torch.zeros(N - 1))


def test_two_runs_bit_identical():
    dev = _dev()
    maps, meta = loader_frame(6, 96, 200, 5, 34720, seed=11)
    meta['depth_mask'][2][3] = False
    a, b = kernel_frame(maps, meta, dev), kernel_frame(maps, meta, dev)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _reference_loop(head, metas, num_rays, agg, n_frames):
    """eval_novel_depth.py:159-208 on head.render outputs: one render per source pose, grid_sample, the boolean mask per
    camera, compute_depth_errors_torch (utils/metric_util.py:424-445, fp32), summed per ceil(distance)."""
    m = metas[0]
    for s, dist in enumerate(m['frame_dists']):
        loc = torch.tensor(m['depth_loc'][s], dtype=torch.float32, device='cuda')
        gt = torch.tensor(m['depth_gt'][s], dtype=torch.float32, device='cuda')
        mask = torch.from_numpy(m['depth_mask'][s]).cuda()
        N = gt.shape[0]
        m['render_img2lidar'] = m['temImg2lidars'][s]
        pred = head.render(metas=metas)['ms_depths'][0].reshape(N, 1, *num_rays)
        pred = F.grid_sample(pred, loc[:, None] * 2 - 1, mode='bilinear', padding_mode='border', align_corners=True).reshape(N, -1)
        cams = []
        for c in range(N):
            g, p = gt[c][mask[c]], pred[c][mask[c]].clone()
            p[p < 1e-3] = 1e-3
            p[p > 80] = 80
            th = torch.maximum(g / p, p / g)
            cams.append(torch.stack([torch.mean(torch.abs(g - p) / g), torch.mean((g - p) ** 2 / g),
                                     torch.sqrt(((g - p) ** 2).mean()), torch.sqrt(((torch.log(g) - torch.log(p)) ** 2).mean()),
                                     (th < 1.25).float().mean(), (th < 1.25 ** 2).float().mean(), (th < 1.25 ** 3).float().mean()]))
        cams = torch.stack(cams)
        k = math.ceil(dist)
        if k not in agg:
            agg[k], n_frames[k] = cams, torch.ones(1, dtype=torch.int, device='cuda')
        else:
            agg[k] += cams
            n_frames[k] += 1


def test_render_poses_and_metric_equal_the_reference_loop():
    dev = _dev()
    from selfocc_b200 import synth, configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    margs, rng = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)
    num_rays = (9, 16)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=64, ray_number=num_rays, ray_img_size=(90, 160))
    model = build_head(cfg).eval().to(dev)
    head = model.head
    head.return_max_depth = True
    head.model.field.deviation_network.variance.data.fill_(0.25)
    l2i, i2l = synth.camera_rig(synth.NUSC_YAWS, f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    planes = [0.5 * torch.randn_like(p) for p in (model.lifter.tpv_hw, model.lifter.tpv_zh, model.lifter.tpv_wz)]
    metric = NovelDepthMetric(num_cams=6, max_distance=8)
    agg, n_frames = {}, {}
    frame_dists = ([1.3, 2.7, 2.2], [0.4, 5.0], [2.9, 7.6, 1.05, 4.4])      # shared bins within and across frames
    saved = head.img2lidar.trans_kw, head.img2lidar.trans_kw_eval
    with torch.no_grad():
        head.prepare(representation=planes)
        for f, dists in enumerate(frame_dists):
            poses = []
            for s in range(len(dists)):
                T = np.eye(4); T[0, 3] = 0.3 * s - 0.2 * f; T[1, 3] = 0.5 * s
                poses.append([T @ np.asarray(m) for m in i2l])
            _, meta = loader_frame(6, 1, 1, len(dists), 4000, seed=20 + f, dists=dists)
            metas = [dict(meta, lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(90, 160), temImg2lidars=poses)]
            out = head.render_poses(metas=metas)
            metric._after_step(metas, out['ms_depths'][0].reshape(len(dists), 6, *num_rays))
            head.img2lidar.trans_kw = head.img2lidar.trans_kw_eval = ['render_img2lidar']
            try:
                _reference_loop(head, metas, num_rays, agg, n_frames)
            finally:
                head.img2lidar.trans_kw, head.img2lidar.trans_kw_eval = saved
    got, got_n = metric._after_epoch()
    assert sorted(got) == sorted(agg) == [1, 2, 3, 5, 8]
    assert {k: int(v) for k, v in got_n.items()} == {k: int(v) for k, v in n_frames.items()}
    for k in agg:
        assert got[k].shape == (6, 7) and got_n[k].shape == (1,)
        assert torch.allclose(got[k].float(), agg[k], rtol=1e-5, atol=1e-6), (k, got[k], agg[k])


def test_after_step_enqueues_no_host_sync():
    dev = _dev()
    maps, meta = loader_frame(6, 96, 200, 5, 34720, seed=3)
    maps = maps.to(dev)
    metric = NovelDepthMetric(num_cams=6, max_distance=6)
    metric._after_step([meta], maps)                                   # warm-up: module load, first pinned block
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        metric._after_step([meta], maps)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    agg, n = metric._after_epoch()
    assert sum(int(v) for v in n.values()) == 10
