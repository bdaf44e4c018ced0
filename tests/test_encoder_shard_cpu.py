"""CPU: the exchange of the query-sharded encoder (selfocc_b200/dist.py all_gather_rows) over gloo at world 2 and 3 with
plane sizes that do not divide by the world size, and its padding / assembly on their own."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from selfocc_b200.dist import (all_gather_rows, assemble_rows, local_rows, pad_rows, per_rank_rows, plane_slices, split_rows,
                               unpad_rows)

SIZES = [11, 7, 5]          # world 2: 6+5 | 4+3 | 3+2;  world 3: 4+4+3 | 3+3+1 | 2+2+1
C = 4


def _full(salt=0.0):
    return torch.arange(sum(SIZES) * C, dtype=torch.float64).reshape(-1, C) * (1 + salt) + salt


def _grad(seed):
    """integer-valued: a sum over the ranks is exact in any order"""
    return torch.randint(-50, 50, (sum(SIZES), C), generator=torch.Generator().manual_seed(seed)).to(torch.float64)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    full = _full()
    local = local_rows(full, SIZES, rank, world).clone().requires_grad_(True)
    got = all_gather_rows(local, SIZES, rank, world)
    # forward: the ranks' rows put back in plane order, i.e. torch.cat of every rank's rows plane by plane
    parts = []
    off = 0
    for i, n in enumerate(SIZES):
        for r in range(world):
            b, c = plane_slices(SIZES, r, world)[i]
            parts.append(full[off + b:off + b + c])
        off += n
    ok = torch.equal(got, torch.cat(parts, 0)) and torch.equal(got, full)
    # backward: this rank's rows of the SUM over the ranks of their incoming gradients
    g_out = [_grad(11 + r) for r in range(world)]
    (g,) = torch.autograd.grad(got, [local], g_out[rank])
    ok = ok and g.shape == local.shape and torch.equal(g, local_rows(sum(g_out), SIZES, rank, world))
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_row_gather_gloo(world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, 29771 + world, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(world))
    [p.join(60) for p in procs]
    assert res == [(r, True) for r in range(world)]


@pytest.mark.parametrize('world', [1, 2, 3, 4])
def test_padding_and_assembly(world):
    full = _full(0.5)
    R = per_rank_rows(SIZES, world)
    bufs = [pad_rows(local_rows(full, SIZES, r, world), SIZES, r, world) for r in range(world)]
    assert all(b.shape == (R, C) for b in bufs)
    for r, b in enumerate(bufs):                               # own rows first in each plane's block, zeros after
        off = 0
        for (_, c), n in zip(plane_slices(SIZES, r, world), SIZES):
            per = -(-n // world)
            assert not b[off + c:off + per].any()
            off += per
        assert torch.equal(unpad_rows(b, SIZES, r, world), local_rows(full, SIZES, r, world))
    stacked = torch.stack(bufs, 0)
    assert torch.equal(assemble_rows(stacked, SIZES, world), full)
    assert torch.equal(split_rows(full, SIZES, world), stacked)              # the backward's layout is the inverse


@pytest.mark.parametrize('world', [2, 3])
def test_row_gather_injected_collectives(world):
    """The collective hooks: an in-process gather of every rank's buffer and a reduce-scatter over given gradients."""
    full = _full()
    locs = [local_rows(full, SIZES, r, world).clone().requires_grad_(True) for r in range(world)]
    bufs = [pad_rows(l.detach(), SIZES, r, world) for r, l in enumerate(locs)]
    g_out = [_grad(r) for r in range(world)]
    g_bufs = [split_rows(g, SIZES, world).reshape(-1, C) for g in g_out]
    for r in range(world):
        def gather(out, buf):
            torch.cat(bufs, out=out)

        def reduce_scatter(out, buf, r=r):
            out.copy_(sum(b.view(world, -1, C)[r] for b in g_bufs))
        got = all_gather_rows(locs[r], SIZES, r, world, collective=gather, reduce_scatter=reduce_scatter)
        assert torch.equal(got, full)
        (g,) = torch.autograd.grad(got, [locs[r]], g_out[r])
        assert torch.equal(g, local_rows(sum(g_out), SIZES, r, world))


def test_row_gather_refuses_wrong_row_count():
    with pytest.raises(ValueError, match='rows'):
        all_gather_rows(torch.zeros(3, C), SIZES, 0, 2, collective=lambda o, b: None, reduce_scatter=lambda o, b: None)
