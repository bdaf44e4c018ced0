"""CPU: the per-camera ray-payload gather of ray-sharded training (selfocc_b200/dist.py all_gather_ray_payload) and
all_gather_planar over gloo at world 2 and 3 with uneven and empty slices, and MultiLoss's two-stage evaluation of the torch-side terms (RGB with SSIM,
edge smoothness, semantics) on emulated ranks: the same loss values, bit for bit, and the same gradients."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from selfocc_b200.dist import all_gather_planar, all_gather_ray_payload, pack_planar, ray_slice

N_CAM, R_FULL = 3, 7 * 5          # 3 cameras x a 7x5 ray grid: uneven slices at world 2 (18 + 17) and 3 (12 + 12 + 11)


def _full(total, k, salt):
    return (torch.arange(N_CAM * total * k, dtype=torch.float32).reshape(N_CAM, total, k) + salt) * (1 + salt)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    ok = True
    # a [3, 35, 1] and a [3, 35, 3] payload, a 2-ray one (empty slice at world 3) and a per-rank scalar, in one collective
    specs = [(R_FULL, 1), (R_FULL, 3), (2, 2)]
    fulls = [_full(n, k, i) for i, (n, k) in enumerate(specs)]
    local = [f[:, b:b + c].clone().requires_grad_(True) for f, (n, _) in zip(fulls, specs) for b, c in [ray_slice(n, world, rank)]]
    scalar = torch.tensor([[[float(rank), 1.0]]], dtype=torch.float64, requires_grad=True)
    got = all_gather_ray_payload(local + [scalar], [n for n, _ in specs] + [world], rank, world)
    ok = ok and all(torch.equal(g, f) and g.dtype == f.dtype for g, f in zip(got, fulls))
    ok = ok and torch.equal(got[3], torch.tensor([[[float(r), 1.0] for r in range(world)]], dtype=torch.float64))
    # backward: world x the incoming gradient at this rank's own rows, nothing for the rows of the other ranks
    g_out = [torch.randn(g.shape, generator=torch.Generator().manual_seed(7 + i), dtype=g.dtype) for i, g in enumerate(got)]
    grads = torch.autograd.grad(got, local + [scalar], g_out)
    for (n, _), gl, go, loc in zip(specs + [(world, 2)], grads, g_out, local + [scalar]):
        b, c = ray_slice(n, world, rank)
        ok = ok and gl.shape == loc.shape and torch.equal(gl, world * go[:, b:b + c])
    # all_gather_planar (flat ray order) with a 2-ray total: rank 2 of world 3 holds an empty slice
    b, c = ray_slice(2, world, rank)
    d = torch.arange(b, b + c, dtype=torch.float32)
    fd, frgb = all_gather_planar([d, torch.stack([d, 2 * d, 3 * d], -1)], 2)
    ok = ok and torch.equal(fd, torch.arange(2, dtype=torch.float32)) and torch.equal(frgb[:, 2], 3 * fd) and frgb.shape == (2, 3)
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_ray_payload_gather_gloo(world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, 29751 + world, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(world))
    [p.join(60) for p in procs]
    assert res == [(r, True) for r in range(world)]


def emulated_ranks(ml, inputs, world):
    """MultiLoss on ``world`` ranks emulated in one process: inputs[r] is rank r's inputs (with 'ray_shard'); the collective
    hands rank r every rank's packed payload, its own through the autograd gather.  -> [(tot_loss, loss_dict)] per rank."""
    payloads = [ml.local_payload(inp) for inp in inputs]
    bufs = [pack_planar([t.detach() for term in p for t, _ in term], [n for term in p for _, n in term], world, torch.float64)
            for p in payloads]
    out = []
    try:
        for r in range(world):
            ml.collective = lambda o, buf, r=r: torch.cat(bufs[:r] + [buf] + bufs[r + 1:], out=o)
            out.append(ml.from_gathered(ml.gather(payloads[r], r, world), inputs[r]))
    finally:
        ml.collective = None
    return out


def _torch_terms_case(seed=0):
    g = torch.Generator().manual_seed(seed)
    rr, img, n, C = [6, 10], [48, 80], 3, 5
    R = rr[0] * rr[1]
    ys, xs = torch.meshgrid(torch.arange(rr[0]), torch.arange(rr[1]), indexing='ij')
    rays = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * 8, (ys.flatten() + torch.rand(R, generator=g)) * 8], -1)
    leaves = dict(colors=torch.rand(1, n, R, 3, generator=g), depths=1 + 40 * torch.rand(1, n, R, generator=g),
                  accs=torch.rand(1, n, R, generator=g), maxd=40 + 10 * torch.rand(1, n, R, generator=g),
                  sem=torch.softmax(3 * torch.randn(1, n, R, C, generator=g), -1))
    fixed = dict(curr_imgs=torch.rand(1, n, 3, 24, 40, generator=g), color_imgs=torch.rand(1, n, 3, 24, 40, generator=g),
                 metas=[dict(sem=torch.randint(0, C, (n, 48, 80), generator=g).to(torch.uint8).numpy())], ms_rays=rays)
    cfgs = [dict(type='RGBLossMS', img_size=img, no_ssim=False, ray_resize=rr, weight=0.1,
                 input_dict=dict(gt_imgs='color_imgs', ms_colors='ms_colors', ms_rays='ms_rays')),
            dict(type='EdgeLoss3DMS', img_size=img, ray_resize=rr, use_inf_mask=True, weight=0.01,
                 input_dict=dict(curr_imgs='curr_imgs', ms_depths='ms_depths', ms_rays='ms_rays', ms_accs='ms_accs',
                                 max_depths='max_depths')),
            dict(type='SemCELossMS', img_size=img, ray_resize=rr, weight=0.1),
            dict(type='SemLossMS', img_size=img, ray_resize=rr, weight=0.1)]
    return cfgs, leaves, fixed, R


def _inputs(leaves, fixed, rays):
    return dict(fixed, ms_rays=rays, ms_colors=[leaves['colors']], ms_depths=[leaves['depths']], ms_accs=[leaves['accs']],
                max_depths=[leaves['maxd']], sem=[leaves['sem']])


@pytest.mark.parametrize('world', [2, 3, 7])
def test_torch_side_terms_on_emulated_ranks_equal_the_unsharded_objective(world):
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss  # noqa: F401
    cfgs, full, fixed, R = _torch_terms_case()
    ml = LOSSES.build(dict(type='MultiLoss', loss_cfgs=cfgs))
    leaves = {k: v.clone().requires_grad_(True) for k, v in full.items()}
    tot, ref = ml(_inputs(leaves, fixed, fixed['ms_rays']))
    ref_g = torch.autograd.grad(tot, list(leaves.values()))
    ranks = []
    for r in range(world):
        b, c = ray_slice(R, world, r)
        own = {k: v[:, :, b:b + c].clone().requires_grad_(True) for k, v in full.items()}
        ranks.append((own, dict(_inputs(own, fixed, fixed['ms_rays'][b:b + c]), ray_shard=(r, world, R))))
    res = emulated_ranks(ml, [inp for _, inp in ranks], world)
    for tot_r, d in res:
        assert list(d) == list(ref)
        for k in ref:
            assert torch.equal(d[k], ref[k]), (k, d[k].item(), ref[k].item())
    # every rank's own-slice gradients / world, put side by side, are the unsharded gradients
    got = [torch.autograd.grad(tot_r, list(own.values())) for (tot_r, _), (own, _) in zip(res, ranks)]
    for i, g_ref in enumerate(ref_g):
        g = torch.cat([gr[i] / world for gr in got], 2)
        assert (g - g_ref).abs().max().item() <= 1e-6 * g_ref.abs().max().item(), list(full)[i]


def test_unsharded_terms_still_refuse_a_partial_ray_set():
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss  # noqa: F401
    cfgs, full, fixed, R = _torch_terms_case()
    ml = LOSSES.build(dict(type='MultiLoss', loss_cfgs=cfgs[:2]))
    half = {k: v[:, :, :R // 2] for k, v in full.items()}
    with pytest.raises(ValueError, match='ray_resize'):
        ml(_inputs(half, fixed, fixed['ms_rays'][:R // 2]))
    with pytest.raises(ValueError, match='ray_resize'):                 # world 1: the unsharded path
        ml(dict(_inputs(half, fixed, fixed['ms_rays'][:R // 2]), ray_shard=(0, 1, R)))
