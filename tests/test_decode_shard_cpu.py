"""CPU: the volume exchange of the decode-sharded training step (selfocc_b200/dist.py all_gather_volume: each rank's slab of
h rows of vol_sdf / vol_feat -> the full volume, one all_gather forward, one reduce-scatter backward) over gloo at world 2,
3 and 4 with H not divisible by the world size, through injected collectives, its refusals, and the argument checks of
so_bev_decode_rows."""
import ctypes as C
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from selfocc_b200.dist import all_gather_volume, pack_volume_rows, volume_exchange_bytes, volume_slab

H, W, Z, ZP, FP = 7, 3, 5, 8, 4          # world 2: 4+3;  world 3: 3+3+1;  world 4: 2+2+2+1


def _volume(feat, salt=0.0):
    vs = torch.arange(H * W * ZP, dtype=torch.float64).reshape(H, W, ZP) * (1 + salt) + salt
    vf = -torch.arange(H * W * Z * FP, dtype=torch.float64).reshape(H, W, Z, FP) * (1 + salt) if feat else None
    return vs, vf


def _grads(seed, feat):
    """integer-valued: a sum over the ranks is exact in any order"""
    g = torch.Generator().manual_seed(seed)
    gs = torch.randint(-50, 50, (H, W, ZP), generator=g).to(torch.float64)
    gf = torch.randint(-50, 50, (H, W, Z, FP), generator=g).to(torch.float64) if feat else None
    return gs, gf


def _slab(t, rank, world):
    b, c = volume_slab(H, rank, world)
    return None if t is None else t[b:b + c]


def _check_rank(rank, world, feat, gather=None, reduce_scatter=None, g_all=None):
    vs, vf = _volume(feat)
    ls = _slab(vs, rank, world).clone().requires_grad_(True)
    lf = _slab(vf, rank, world).clone().requires_grad_(True) if feat else None
    gs_, gf_ = all_gather_volume(ls, lf, H, rank, world, gather, reduce_scatter)
    ok = torch.equal(gs_, vs) and gs_.is_contiguous() and (gf_ is None if not feat else torch.equal(gf_, vf) and gf_.is_contiguous())
    # backward: this rank's slab of the SUM over the ranks of their incoming volume gradients
    g_all = g_all or [_grads(11 + r, feat) for r in range(world)]
    outs, ins, gos = [gs_], [ls], [g_all[rank][0]]
    if feat:
        outs, ins, gos = outs + [gf_], ins + [lf], gos + [g_all[rank][1]]
    got = torch.autograd.grad(outs, ins, gos)
    ok = ok and torch.equal(got[0], _slab(sum(g[0] for g in g_all), rank, world))
    if feat:
        ok = ok and torch.equal(got[1], _slab(sum(g[1] for g in g_all), rank, world))
    return bool(ok)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    q.put((rank, _check_rank(rank, world, True) and _check_rank(rank, world, False)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3, 4])
def test_volume_gather_gloo(world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, 29841 + world, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(world))
    [p.join(60) for p in procs]
    assert res == [(r, True) for r in range(world)]


@pytest.mark.parametrize('feat', [True, False])
@pytest.mark.parametrize('world', [2, 3, 4])
def test_volume_gather_injected_collectives(world, feat):
    """The collective hooks: an in-process gather of every rank's padded slab rows and a reduce-scatter over given
    gradients; one call of each per rank."""
    per = -(-H // world)
    vols = _volume(feat)
    rows = [pack_volume_rows(_slab(vols[0], r, world), _slab(vols[1], r, world)) for r in range(world)]
    width = rows[0].shape[1]
    bufs = [torch.cat([x, x.new_zeros(per - x.shape[0], width)]) for x in rows]
    g_all = [_grads(r, feat) for r in range(world)]
    g_bufs = []
    for gs, gf in g_all:
        full = pack_volume_rows(gs, gf)
        g_bufs.append(torch.cat([full, full.new_zeros(world * per - H, width)]))
    for r in range(world):
        calls = []

        def gather(out, buf, r=r):
            calls.append('all_gather')
            assert torch.equal(buf, bufs[r])                   # this rank's rows, padded to ceil(H / world)
            torch.cat(bufs, out=out)

        def reduce_scatter(out, buf, r=r):
            calls.append('reduce_scatter')
            assert buf.shape == (world * per, width)
            out.copy_(sum(b.view(world, per, width)[r] for b in g_bufs))
        assert _check_rank(r, world, feat, gather, reduce_scatter, g_all)
        assert calls == ['all_gather', 'reduce_scatter']


def test_volume_slab_and_refusals():
    assert [volume_slab(H, r, 3) for r in range(3)] == [(0, 3), (3, 3), (6, 1)]
    assert volume_slab(H, 0, 1) == (0, H)
    with pytest.raises(ValueError, match='ranks'):
        volume_slab(3, 0, 4)
    none = lambda o, b: None
    with pytest.raises(ValueError, match='ranks'):
        all_gather_volume(torch.zeros(1, W, ZP), None, 3, 0, 4, none, none)
    with pytest.raises(ValueError, match='slab'):                   # rank 1 of 2 holds 3 rows, not 4
        all_gather_volume(torch.zeros(4, W, ZP), None, H, 1, 2, none, none)
    with pytest.raises(ValueError, match='slab'):
        all_gather_volume(torch.zeros(3, W, ZP), torch.zeros(2, W, Z, FP), H, 1, 2, none, none)


def test_exchange_bytes_at_the_shipped_volumes():
    from selfocc_b200 import _lib
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = 257, 257, 25, 28, 24, 24
    row = 257 * 28 + 257 * 25 * 24
    assert volume_exchange_bytes(d, 1) == dict(all_gather=0, reduce_scatter=0)
    assert volume_exchange_bytes(d, 4) == dict(all_gather=4 * 3 * 65 * row, reduce_scatter=4 * 3 * 65 * row)
    d.n_feat = 0
    assert volume_exchange_bytes(d, 2)['all_gather'] == 4 * 129 * 257 * 28


def test_bev_decode_rows_rejects_bad_ranges_without_a_gpu():
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one = None, C.c_void_p(16)
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = 5, 7, 25, 32, 24, 24
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 10.0, 4.0
    f = lib.so_bev_decode_rows
    assert f(N, 96, one, one, one, one, C.byref(d), 0, 5, one, one, N) == -1                   # no bev
    assert f(one, 96, one, one, one, one, None, 0, 5, one, one, N) == -1                       # no volume desc
    assert f(one, 96, one, one, one, one, C.byref(d), -1, 2, one, one, N) == -1                # negative begin
    assert f(one, 96, one, one, one, one, C.byref(d), 0, -1, one, one, N) == -1                # negative count
    assert f(one, 96, one, one, one, one, C.byref(d), 3, 3, one, one, N) == -1                 # rows beyond H
    assert f(one, 96, one, one, one, one, C.byref(d), 2, 2 ** 31 - 1, one, one, N) == -1       # begin + count overflows
    assert f(one, 96, one, one, one, one, C.byref(d), 5, 0, one, one, N) == 0                  # empty slab: nothing to do
    assert f(one, 128, one, one, one, one, C.byref(d), 0, 1, one, one, N) == -2                # C other than 96
    assert f(one, 96, one, one, one, one, C.byref(d), 4, 1, one, N, N) == -1                   # features without vol_feat
    assert f(C.c_void_p(20), 96, one, one, one, one, C.byref(d), 0, 1, one, one, N) == -1      # misaligned bev
