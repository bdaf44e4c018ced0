"""CPU: novel-view depth evaluation -- the fp64 oracle pinned to the reference's arithmetic
(tests/golden/reference_golden_novel_depth.npz), the frame packing of NovelDepthMetric from loader-shaped metas, the
distance-bin refusal, the argument checks of so_novel_depth_errors and the end-of-epoch all-reduce over gloo."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import novel_depth as ond
from selfocc_b200.metric import NovelDepthMetric, novel_depth_errors, pack_novel_depth

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden_novel_depth.npz'))
FRAMES = 3


def golden_frame(f):
    """(depth maps [S, N, h, w], loader metas) of golden frame f."""
    dists = [float(d) for d in G['f%d_dists' % f]]
    meta = {k: [G['f%d_s%d_%s' % (f, s, k)] for s in range(len(dists))] for k in ('depth_loc', 'depth_gt', 'depth_mask')}
    meta['frame_dists'] = dists
    return torch.from_numpy(G['f%d_maps' % f]), meta


def test_oracle_equals_the_reference_loop_body():
    per_source = []
    for f in range(FRAMES):
        maps, meta = golden_frame(f)
        for s, (k, e) in enumerate(ond.frame_errors_ref(maps, meta)):
            ref = G['f%d_s%d_errors' % (f, s)]
            assert np.allclose(e.numpy(), ref, rtol=1e-5, atol=1e-6, equal_nan=True), (f, s)
            pred = ond.sample_ref(maps[s], torch.from_numpy(meta['depth_loc'][s]).float())
            assert np.allclose(pred.numpy(), G['f%d_s%d_sampled' % (f, s)], rtol=1e-6, atol=1e-5), (f, s)
        per_source += ond.frame_errors_ref(maps, meta)
    assert np.isnan(G['f0_s1_errors'][2]).all()                    # the fixture holds an empty segment
    agg, n = ond.aggregate_ref(per_source)
    assert sorted(agg) == list(G['bins'])
    assert [n[k] for k in sorted(n)] == list(G['n_frames'])
    for i, k in enumerate(G['bins']):
        assert np.allclose(agg[int(k)].numpy(), G['agg_errors'][i], rtol=1e-5, atol=1e-6, equal_nan=True), k


@pytest.mark.parametrize('num_cams', [3, 1])
def test_pack_from_loader_metas(num_cams):
    """Sections of the packed frame: segment offsets in render_poses' [S, N] order, the rounds of distance bins, the
    float32 conversion of the loader's float64 arrays (as input_imgs.new_tensor does) and the uint8 mask."""
    g = np.random.default_rng(0)
    counts = [5, 0, 7, 3]
    dists = [2.5, 0.0, 3.0, 2.1]                                    # bins 3, 0, 3, 3
    meta = dict(depth_loc=[g.random((num_cams, n, 2)) for n in counts], depth_gt=[g.random((num_cams, n)) * 50 for n in counts],
                depth_mask=[g.random((num_cams, n)) < 0.5 for n in counts], frame_dists=dists)
    buf, lay = pack_novel_depth(meta, num_cams, 4, pin=False)
    S, N = len(counts), num_cams
    assert (lay['S'], lay['N'], lay['T']) == (S, N, N * sum(counts))
    part = lambda name, dt: buf[lay[name][0]:lay[name][0] + lay[name][1]].view(dt)
    seg = np.repeat(counts, N)
    assert part('offsets', torch.int64).tolist() == [0] + np.cumsum(seg).tolist()
    assert part('perm', torch.int64).tolist() == [0, 1, 2, 3]
    assert part('bins', torch.int64).tolist() == [3, 0, 3, 3]
    assert lay['rounds'] == [(0, 2), (2, 3), (3, 4)]                # each round holds a bin at most once
    cat = lambda k, dt: torch.cat([torch.as_tensor(a, dtype=dt).reshape(-1) for a in meta[k]])
    assert torch.equal(part('loc', torch.float32), cat('depth_loc', torch.float32))
    assert torch.equal(part('gt', torch.float32), cat('depth_gt', torch.float32))
    assert torch.equal(part('mask', torch.uint8), cat('depth_mask', torch.bool).to(torch.uint8))
    assert all(lay[k][0] % 16 == 0 for k in ('offsets', 'perm', 'bins', 'loc', 'gt', 'mask'))


def test_pack_refuses_distances_beyond_the_bins_and_bad_shapes():
    meta = dict(depth_loc=[np.zeros((2, 3, 2))], depth_gt=[np.ones((2, 3))], depth_mask=[np.ones((2, 3), bool)], frame_dists=[4.2])
    with pytest.raises(ValueError, match='bin 5, outside'):
        pack_novel_depth(meta, 2, 4, pin=False)
    pack_novel_depth(meta, 2, 5, pin=False)
    with pytest.raises(ValueError, match='outside'):
        pack_novel_depth(dict(meta, frame_dists=[-1.5]), 2, 5, pin=False)
    with pytest.raises(ValueError, match='expected depth_loc'):
        pack_novel_depth(meta, 3, 5, pin=False)                       # 2 cameras delivered, 3 expected
    with pytest.raises(ValueError, match='one entry per source'):
        pack_novel_depth(dict(meta, frame_dists=[1.0, 2.0]), 2, 5, pin=False)


def test_wrapper_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        novel_depth_errors(torch.zeros(1, 2, 2), torch.zeros(2, dtype=torch.int64), torch.zeros(0, 2), torch.zeros(0),
                           torch.zeros(0, dtype=torch.uint8))


def test_entry_point_rejects_bad_arguments_without_a_gpu():
    """Null pointers, no segment, bad map sizes, offsets that do not start at 0, do not end at T or decrease:
    SO_ERR_INVALID_ARG (-1) before any CUDA call."""
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    f = lib.so_novel_depth_errors
    N, one = None, C.c_void_p(16)
    host = lambda *v: (C.c_int64 * len(v))(*v)
    ok = host(0, 3, 5)
    assert f(N, 2, 4, 4, one, ok, 5, one, one, one, one, N) == -1           # no depth maps
    assert f(one, 2, 4, 4, N, ok, 5, one, one, one, one, N) == -1           # no device offsets
    assert f(one, 2, 4, 4, one, N, 5, one, one, one, one, N) == -1          # no host offsets
    assert f(one, 2, 4, 4, one, ok, 5, one, one, one, N, N) == -1           # no output
    assert f(one, 2, 4, 4, one, ok, 5, N, one, one, one, N) == -1           # points but no locations
    assert f(one, 2, 4, 4, one, ok, 5, one, N, one, one, N) == -1
    assert f(one, 2, 4, 4, one, ok, 5, one, one, N, one, N) == -1
    assert f(one, 0, 4, 4, one, ok, 5, one, one, one, one, N) == -1         # zero segments
    assert f(one, -1, 4, 4, one, ok, 5, one, one, one, one, N) == -1
    assert f(one, 2, 0, 4, one, ok, 5, one, one, one, one, N) == -1         # empty map
    assert f(one, 2, 4, 0, one, ok, 5, one, one, one, one, N) == -1
    assert f(one, 2, 4, 4, one, host(0, 4, 3), 3, one, one, one, one, N) == -1   # decreasing offsets
    assert f(one, 2, 4, 4, one, host(1, 3, 5), 5, one, one, one, one, N) == -1   # not starting at 0
    assert f(one, 2, 4, 4, one, ok, 6, one, one, one, one, N) == -1              # not ending at T
    assert f(one, 2, 4, 4, one, ok, -5, one, one, one, one, N) == -1
    assert f(one, 2, 65536, 65536, one, ok, 5, one, one, one, one, N) == -2      # map indices beyond 32 bits
    assert lib.so_abi_version() == 10


def _epoch_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    m = NovelDepthMetric(num_cams=2, max_distance=5, device='cpu')
    # rank 0 holds bins 1 and 3, rank 1 bins 3 and 4: the reference's per-bin reduction would pair different bins
    for k in ((1, 3) if rank == 0 else (3, 4)):
        m.errors[k] = (rank + 1) * 10 + k + torch.arange(14, dtype=torch.float64).reshape(2, 7)
        m.n_frames[k] = rank + k
    agg, n = m._after_epoch()
    q.put((rank, {k: v.tolist() for k, v in agg.items()}, {k: v.tolist() for k, v in n.items()}))
    dist.barrier()
    dist.destroy_process_group()


def test_after_epoch_all_reduce_gloo_world2():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_epoch_worker, args=(r, 2, 29747, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(60) for p in procs]
    base = torch.arange(14, dtype=torch.float64).reshape(2, 7)
    want_agg = {1: (11 + base).tolist(), 3: (13 + base + 23 + base).tolist(), 4: (24 + base).tolist()}
    want_n = {1: [1], 3: [3 + 4], 4: [5]}
    for rank, agg, n in res:
        assert agg == want_agg and n == want_n, rank


def test_as_dicts_takes_the_kitti_form_for_one_camera():
    m = NovelDepthMetric(num_cams=1, max_distance=3, device='cpu')
    m.errors[2, 0] = torch.arange(7, dtype=torch.float64)
    m.n_frames[2] = 4
    agg, n = m.as_dicts()
    assert list(agg) == [2] and n == {2: 4}
    assert isinstance(agg[2], np.ndarray) and agg[2].shape == (7,) and isinstance(n[2], int)
