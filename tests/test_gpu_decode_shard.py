"""GPU: the decode-sharded training step (NeuSHead.decode_shard: each rank decodes its slab of the volume's h rows,
dist.all_gather_volume assembles the volume, its backward reduce-scatters the volume gradient).

* so_bev_decode_rows against the same rows of so_bev_decode, bit for bit, rows outside the range untouched;
* emulated ranks' slabs, gathered, against the unsharded decode at the shipped nuscenes_occ (TPV) and nuscenes_occ_bev
  volumes (257 x 257, Z 25, 25 channels), bit for bit;
* lockstep emulated training steps against the unsharded step: loss values, and DDP-mean gradients of every parameter and
  of the FPN features.  Ranks run one after the other from the same RNG state.  The exchange is emulated in two backward
  passes: the emulated reduce-scatter records every rank's volume gradient and returns zeros; a second pass then sends each
  rank's slab (recorded from the field's decode) the sum over the ranks of their gradients there, which is what the
  reduce-scatter hands it.  The sum of the two passes over the ranks, divided by world, is DDP's mean;
* a two-process run on one GPU over gloo (host-staged collectives), and a torchrun / NCCL / DDP run on >= 2 GPUs (skipped
  below 2)."""
import copy
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import ops, synth
from selfocc_b200.dist import all_gather_rows, all_gather_volume, local_rows, pack_volume_rows, pad_rows, volume_slab
from selfocc_b200.mapping import GridMeterMapping

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from test_gpu_ray_shard import CFGS, _build, _check_values  # noqa: E402
from test_gpu_encoder_shard import _check_grads, _objective_inputs, _place, _rng, _set_rng, _wrt, small_training_model  # noqa: E402
from test_ray_shard_cpu import emulated_ranks  # noqa: E402

NUSC_OCC = dict(nonlinear_mode='linear', h_size=[128, 0], h_range=[40.0, 0], h_half=False, w_size=[128, 0], w_range=[40.0, 0],
                w_half=False, d_size=[24, 0], d_range=[-1.0, 5.4, 5.4])        # nuscenes_occ and nuscenes_occ_bev: 257 x 257 x 25
SPARSITY = dict(type='SoftSparsityLoss', weight=0.001, input_dict=dict(density='uniform_sdf'))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _mlp(n_in, n_out, g, dev):
    return [t.to(dev) for t in (torch.randn(n_in, n_in, generator=g) / n_in ** 0.5, 0.1 * torch.randn(n_in, generator=g),
                                torch.randn(n_out, n_in, generator=g) / n_in ** 0.5, 0.1 * torch.randn(n_out, generator=g))]


# --------------------------------------------------------------------------------------------- so_bev_decode_rows
def _margs(h, w, d):
    return dict(NUSC_OCC, h_size=[h, 0], w_size=[w, 0], d_size=[d, 0])


# (h, w, d) half sizes -> H = 2h + 1, W = 2w + 1, Z = d + 1; n_feat.  The kernel works on 128-row tiles of BEV cells, so a
# slab starting at h_begin starts its tiles at BEV row h_begin * W.
BEV_ROWS_CASES = {
    'shipped 257x257, Z 25, Cf 25': ((128, 128, 24), 24, [(0, 257), (0, 1), (256, 1), (128, 1), (1, 64), (65, 65), (193, 64)]),
    'W 9 (tile edge inside row 14), Cf 4': ((10, 4, 6), 3, [(0, 21), (13, 2), (14, 1), (14, 7), (20, 1), (3, 0)]),
    'W 43 (128 = 2 rows + 42), Cf 1': ((6, 21, 2), 0, [(0, 13), (2, 1), (2, 3), (12, 1), (0, 6)]),
}


@pytest.mark.parametrize('case', list(BEV_ROWS_CASES))
def test_bev_decode_rows_equals_the_same_rows_of_the_full_decode(case):
    dev = _dev()
    from selfocc_b200 import _lib
    (h, w, d), n_feat, ranges = BEV_ROWS_CASES[case]
    desc = GridMeterMapping(**_margs(h, w, d)).volume_desc(n_feat)
    H, W, Z, Cf = desc.H, desc.W, desc.Z, 1 + n_feat
    g = torch.Generator().manual_seed(H * 7 + Cf)
    bev = (0.7 * torch.randn(H * W, 96, generator=g)).to(dev)
    mlp = _mlp(96, Z * Cf, g, dev)
    full_s, full_f = ops.bev_decode(bev, *mlp, desc)
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    SENT = 7.25
    for b, c in ranges:
        vs = torch.full((H, W, desc.zpitch), SENT, device=dev)
        vf = torch.full((H, W, Z, desc.feat_pitch), SENT, device=dev) if n_feat else None
        assert lib.so_bev_decode_rows(p(bev), 96, *map(p, mlp), C.byref(desc), b, c, p(vs), p(vf), st) == 0
        assert torch.equal(vs[b:b + c], full_s[b:b + c]), (case, b, c)           # sdf and its zero pads
        assert (vs[:b] == SENT).all() and (vs[b + c:] == SENT).all(), (case, b, c)
        if n_feat:
            assert torch.equal(vf[b:b + c, ..., :n_feat], full_f[b:b + c, ..., :n_feat]), (case, b, c)
            assert (vf[b:b + c, ..., n_feat:] == SENT).all()                      # pad channels never written
            assert (vf[:b] == SENT).all() and (vf[b + c:] == SENT).all(), (case, b, c)
        s2, f2 = ops.bev_decode(bev, *mlp, desc, rows=(b, c), out=(vs.clone(), None if vf is None else vf.clone()))
        assert torch.equal(s2, vs) and (f2 is None or torch.equal(f2[..., :n_feat], vf[..., :n_feat]))
    vs = torch.full((H, W, desc.zpitch), SENT, device=dev)
    vf = torch.full((H, W, Z, desc.feat_pitch), SENT, device=dev) if n_feat else None
    for b, c in ((-1, 2), (0, -1), (H - 1, 2), (1, 2 ** 31 - 1)):
        assert lib.so_bev_decode_rows(p(bev), 96, *map(p, mlp), C.byref(desc), b, c, p(vs), p(vf), st) == -1, (b, c)
    torch.cuda.synchronize()
    assert (vs == SENT).all() and (vf is None or (vf == SENT).all())


# --------------------------------------------------------------------------------------------- the gathered volume
def _gathered(world, slabs, H):
    """Every rank's all_gather_volume over the emulated all_gather of every rank's padded slab rows."""
    per = -(-H // world)
    bufs = []
    for r, (s, f) in enumerate(slabs):
        x = pack_volume_rows(s, f)
        bufs.append(torch.cat([x, x.new_zeros(per - x.shape[0], x.shape[1])]))
    none = lambda o, b: None
    return [all_gather_volume(s, f, H, r, world, lambda o, b: torch.cat(bufs, out=o), none) for r, (s, f) in enumerate(slabs)]


@pytest.mark.parametrize('tpv', [True, False])
def test_gathered_slabs_equal_the_unsharded_decode_at_the_shipped_volume(tpv):
    dev = _dev()
    desc = GridMeterMapping(**NUSC_OCC).volume_desc(24)
    H, W, Z = desc.H, desc.W, desc.Z
    assert (H, W, Z, 1 + desc.n_feat) == (257, 257, 25, 25)
    g = torch.Generator().manual_seed(3)
    if tpv:
        planes = [(0.5 * torch.randn(n, 96, generator=g)).to(dev) for n in (H * W, Z * H, W * Z)]
        mlp = _mlp(96, 25, g, dev)
        fn = lambda rows: ops.TPVDecodeFunction.apply(*planes, *mlp, desc, rows)
    else:
        bev = (0.7 * torch.randn(H * W, 96, generator=g)).to(dev)
        mlp = _mlp(96, Z * 25, g, dev)
        fn = lambda rows: ops.BEVDecodeFunction.apply(bev, *mlp, desc, rows)
    with torch.no_grad():
        ref_s, ref_f = fn(None)
        for world in (1, 2, 3, 4):                               # 257 = 129+128 | 86+86+85 | 65+65+65+62
            slabs = [fn(volume_slab(H, r, world)) for r in range(world)]
            assert [s.shape[0] for s, _ in slabs] == [volume_slab(H, r, world)[1] for r in range(world)]
            for s, f in _gathered(world, slabs, H):
                assert torch.equal(s, ref_s), (tpv, world)
                assert torch.equal(f[..., :24], ref_f[..., :24]), (tpv, world)


# --------------------------------------------------------------------------------------------- lockstep training steps
def _tpv_case(dev, sparsity=True):
    """test_gpu_encoder_shard's small nuscenes_occ-shaped model (second_grad opt-in), dropout 0, with a SoftSparsity term on
    uniform_sdf added to the config's MultiLoss."""
    model, ml, feats, metas, imgs = small_training_model(dev, dropout=0.0)
    if sparsity:
        cfg = copy.deepcopy(CFGS['nuscenes/nuscenes_occ.py'])
        cfg['loss_cfgs'].append(SPARSITY)
        ml = _build(cfg)
        model.head.return_uniform_sdf = True
    return model, ml, feats, metas, imgs


def _bev_case(dev):
    """test_gpu_bev's small nuscenes_occ_bev-shaped model (17 x 17 x 9; SoftSparsity and second_grad as the config sets
    them) with the config's MultiLoss."""
    from test_gpu_bev import _frame, _small_cfg
    from selfocc_b200.registry import build_head
    cfg = _small_cfg(8, 8, 8)
    cfg['head'].update(second_grad_assumption=True)
    torch.manual_seed(0)
    model = build_head(dict(type='TPVHotPath', **cfg)).to(dev).train()
    with torch.no_grad():
        model.head.model.field.deviation_network.variance.fill_(0.25)
    img_size = tuple(cfg['head']['ray_img_size'])
    metas, feats, _, _ = _frame(seed=6, img=img_size, fpn=synth.fpn_level_shapes(*img_size), rig={})
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6,) + img_size, generator=torch.Generator().manual_seed(2)).to(torch.uint8).numpy()
    metas[0].update(sem=lab, img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                    img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))
    imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
    feats = [f.to(dev).requires_grad_(True) for f in feats]
    return model, _build(CFGS['nuscenes/nuscenes_occ_bev.py']), feats, metas, imgs


def _head_kwargs(model, imgs):
    return dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2]) if model.head.fused_objective is not None else {}


def _planes(model, feats, metas):
    r = model.lifter(ms_img_feats=feats)
    return model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)['representation']


def _check_grads_spread(got, ref, ref2, tol=1e-5):
    """test_gpu_encoder_shard._check_grads, each tensor held to 1e-5 of its max-abs or to three times the unsharded step's
    own run-to-run spread (ref vs ref2) where that is larger: the render scatters the volume gradient with atomics, and
    the spread of that order reaches some gradients through sums whose terms cancel."""
    assert len(got) == len(ref) == len(ref2)
    bad = []
    for i, (g, g1, g2) in enumerate(zip(got, ref, ref2)):
        if g1 is None:
            assert g is None or not g.any(), i
            continue
        assert g is not None, i
        err, scale, spread = (g - g1).abs().max().item(), g1.abs().max().item(), (g2 - g1).abs().max().item()
        if err > max(tol * scale, 3 * spread):
            bad.append((i, tuple(g1.shape), err / scale, spread / scale))
    assert not bad, bad


def unsharded(model, ml, feats, metas, imgs, seed=0):
    torch.manual_seed(seed)
    np.random.seed(seed)
    model.head.ray_shard = model.head.decode_shard = None
    rep = _planes(model, feats, metas)
    out = model.head(representation=rep, metas=metas, **_head_kwargs(model, imgs))
    tot, d = ml(_objective_inputs(out, imgs, metas))
    return d, torch.autograd.grad(tot, _wrt(model, feats), allow_unused=True)


def _query_sharded_planes(model, feats, metas, world):
    """Every rank's planes of test_gpu_encoder_shard.lockstep_step's query-sharded encoder (dropout 0)."""
    enc = model.encoder
    H, W, Z = enc.tpv_size
    sizes = [H * W, Z * H, W * Z]
    Q = sum(sizes)
    reps = [model.lifter(ms_img_feats=feats)['representation'] for _ in range(world)]
    sts = [enc.shard_state(feats, metas) for _ in range(world)]
    qfull = [torch.cat([p[0] for p in rep], 0) for rep in reps]
    idx = [local_rows(torch.arange(Q, device=qfull[0].device), sizes, r, world) for r in range(world)]
    for li in range(len(enc.layers)):
        locs = [enc.shard_layer(li, qfull[r], sts[r], r, world) for r in range(world)]
        bufs = [pad_rows(l.detach(), sizes, r, world) for r, l in enumerate(locs)]
        C_ = locs[0].shape[1]
        for r in range(world):
            full = all_gather_rows(locs[r], sizes, r, world, collective=lambda out, buf: torch.cat(bufs, out=out),
                                   reduce_scatter=lambda out, buf, r=r: out.copy_(buf.view(world, -1, C_)[r]))
            for s_ in range(world):
                if s_ != r:
                    p = _place(locs[s_], idx[s_], Q)
                    full = full + (p - p.detach())
            qfull[r] = full
    return [[t[None] for t in torch.split(q, sizes, 0)] for q in qfull]


def decode_sharded_grads(model, ml, feats, metas, imgs, world, ray_shard=True, query_shard=False, seed=0, decode_shard=True):
    """``world`` emulated ranks of the decode-sharded step in lockstep -> (per-rank loss dicts, DDP-mean gradients).
    decode_shard=False: the same lockstep step with the decode replicated."""
    head, f = model.head, model.head.model.field
    H = f.desc.H
    torch.manual_seed(seed)
    np.random.seed(seed)
    planes = _query_sharded_planes(model, feats, metas, world) if query_shard else [_planes(model, feats, metas)] * world
    with torch.no_grad():                                      # the values every rank's all_gather receives
        per = -(-H // world)
        bufs = []
        for r in range(world):
            vs, vf = f.decode(planes[r], train=True, rows=volume_slab(H, r, world))
            x = pack_volume_rows(vs, vf if f.desc.n_feat else None)
            bufs.append(torch.cat([x, x.new_zeros(per - x.shape[0], x.shape[1])]))
    width = bufs[0].shape[1]
    slabs, g_vol, cur = [None] * world, [None] * world, [0]
    decode = f.decode

    def spy(rep, train=False, rows=None):                  # records each rank's slab, autograd-connected
        out = decode(rep, train=train, rows=rows)
        if rows is not None:
            slabs[cur[0]] = out
        return out
    s = _rng()
    inputs = []
    f.decode = spy
    try:
        for r in range(world):
            _set_rng(s)
            cur[0] = r
            head.ray_shard = (r, world) if ray_shard else None
            head.decode_shard = (r, world) if decode_shard else None

            def gather(out, buf, r=r):
                assert torch.equal(buf, bufs[r])               # this rank's slab is the one the others receive
                torch.cat(bufs, out=out)

            def reduce_scatter(out, buf, r=r):
                g_vol[r] = buf.clone()
                out.zero_()
            head.decode_shard_collectives = (gather, reduce_scatter)
            out = head(representation=planes[r], metas=metas, **_head_kwargs(model, imgs))
            inputs.append(_objective_inputs(out, imgs, metas))
    finally:
        del f.decode
        head.ray_shard = head.decode_shard = head.decode_shard_collectives = None
    res = emulated_ranks(ml, inputs, world) if ray_shard else [ml(inp) for inp in inputs]
    wrt = _wrt(model, feats)
    g1 = torch.autograd.grad(sum(t for t, _ in res), wrt, allow_unused=True, retain_graph=decode_shard)
    if not decode_shard:
        return [d for _, d in res], [None if g is None else g / world for g in g1]
    assert all(g is not None for g in g_vol)
    outs, gos = [], []
    n_sdf = f.desc.W * f.desc.zpitch
    for r, (vs, vf) in enumerate(slabs):                       # slab r receives the sum over the ranks at its rows
        c = vs.shape[0]
        gsum = sum(g.view(world, per, width)[r] for g in g_vol)[:c]
        outs.append(vs)
        gos.append(gsum[:, :n_sdf].reshape(vs.shape))
        if f.desc.n_feat:
            outs.append(vf)
            gos.append(gsum[:, n_sdf:].reshape(vf.shape))
    g2 = torch.autograd.grad(outs, wrt, gos, allow_unused=True)
    got = [None if a is None and b is None else ((a if a is not None else 0) + (b if b is not None else 0)) / world
           for a, b in zip(g1, g2)]
    return [d for _, d in res], got


STEP_CASES = {
    'tpv ray_shard': ('tpv', dict()),
    'tpv ray_shard + query_shard': ('tpv', dict(query_shard=True)),
    'bev ray_shard': ('bev', dict()),
}


@pytest.mark.parametrize('world', [2, 3])
@pytest.mark.parametrize('case', list(STEP_CASES))
def test_decode_sharded_step_equals_unsharded(case, world):
    """Loss values as the unsharded step's.  Gradients: the TPV cases against the unsharded step.  The BEV case against the
    same ray-sharded step without decode sharding: on the small BEV model ray sharding alone moves a few encoder gradients
    by up to 2e-5 of their max-abs from the unsharded step (every rank's render scatters world x its rays' gradients into
    one pillar row), while decode sharding alone stays within the unsharded step's run-to-run spread
    (test_decode_sharded_step_without_ray_shard)."""
    dev = _dev()
    kind, kw = STEP_CASES[case]
    model, ml, feats, metas, imgs = _tpv_case(dev) if kind == 'tpv' else _bev_case(dev)
    ref, ref_g = unsharded(model, ml, feats, metas, imgs)
    ref_g2 = unsharded(model, ml, feats, metas, imgs)[1]
    ds, got = decode_sharded_grads(model, ml, feats, metas, imgs, world, **kw)
    for d in ds:
        _check_values(ref, d)
    if kind == 'bev':
        ref_g = decode_sharded_grads(model, ml, feats, metas, imgs, world, decode_shard=False, **kw)[1]
    _check_grads_spread(got, ref_g, ref_g2)


@pytest.mark.parametrize('kind', ['tpv', 'bev'])
def test_decode_sharded_step_without_ray_shard(kind):
    """Every rank renders all rays: each rank's volume gradient is the whole one, unscaled, and the rule still holds."""
    dev = _dev()
    model, ml, feats, metas, imgs = _tpv_case(dev) if kind == 'tpv' else _bev_case(dev)
    ref, ref_g = unsharded(model, ml, feats, metas, imgs)
    ref_g2 = unsharded(model, ml, feats, metas, imgs)[1]
    ds, got = decode_sharded_grads(model, ml, feats, metas, imgs, 2, ray_shard=False)
    for d in ds:
        _check_values(ref, d)
    _check_grads_spread(got, ref_g, ref_g2)


def test_decode_sharded_step_with_the_fused_objective():
    dev = _dev()
    from selfocc_b200.loss import fuse_objective
    model, ml, feats, metas, imgs = _tpv_case(dev, sparsity=False)
    fuse_objective(model.head, ml)
    ref, ref_g = unsharded(model, ml, feats, metas, imgs)
    ds, got = decode_sharded_grads(model, ml, feats, metas, imgs, 2)
    for d in ds:
        _check_values(ref, d)
    _check_grads(got, ref_g)


def test_decode_shard_switch():
    """None, world 1, eval and no_grad keep the existing decode; H < world is refused."""
    dev = _dev()
    model, ml, feats, metas, imgs = _tpv_case(dev, sparsity=False)
    head, f = model.head, model.head.model.field
    rep = [p.detach() for p in _planes(model, feats, metas)]
    from selfocc_b200.head_train import decode_train
    ref = f.decode(rep, train=True)
    calls = []
    hooks = (lambda o, b: calls.append(1), lambda o, b: calls.append(1))
    try:
        head.decode_shard_collectives = hooks
        for shard in (None, (0, 1)):
            head.decode_shard = shard
            out = decode_train(head, rep)
            assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
        head.decode_shard = (0, 2)
        with torch.no_grad():
            out = decode_train(head, rep)
        head.eval()
        out2 = decode_train(head, rep)
        head.train()
        assert not calls and torch.equal(out[0], ref[0]) and torch.equal(out2[0], ref[0])
        head.decode_shard = (0, f.desc.H + 1)
        with pytest.raises(ValueError, match='ranks'):
            decode_train(head, rep)
    finally:
        head.decode_shard = head.decode_shard_collectives = None


GLOO_WORKER = r'''
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, %r); sys.path.insert(0, %r)
from test_gpu_decode_shard import _tpv_case, unsharded
from test_gpu_encoder_shard import _objective_inputs, _wrt
rank, world = int(sys.argv[1]), int(sys.argv[2])
os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=sys.argv[3])
dist.init_process_group('gloo', rank=rank, world_size=world)
dev = torch.device('cuda', 0)


def host(op):
    def run(out, buf):
        o = torch.empty(out.shape, dtype=out.dtype)
        op(o, buf.cpu())
        out.copy_(o)
    return run
gather = host(lambda o, b: dist.all_gather_into_tensor(o, b))
reduce_scatter = host(lambda o, b: dist.reduce_scatter_tensor(o, b, op=dist.ReduceOp.SUM))
model, ml, feats, metas, imgs = _tpv_case(dev)
ml.collective = gather
torch.manual_seed(0)
np.random.seed(0)
model.head.ray_shard = (rank, world)
model.head.decode_shard = (rank, world)
model.head.decode_shard_collectives = (gather, reduce_scatter)
r = model.lifter(ms_img_feats=feats)
rep = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)['representation']
tot, d = ml(_objective_inputs(model.head(representation=rep, metas=metas), imgs, metas))
grads = torch.autograd.grad(tot, _wrt(model, feats), allow_unused=True)
mean = []
for g in grads:                                            # DDP's gradient mean, explicitly
    if g is None:
        mean.append(None)
        continue
    h = g.cpu()
    dist.all_reduce(h)
    mean.append(h / world)
vals = torch.stack([v.detach().cpu() for v in d.values()])
hi, lo = vals.clone(), vals.clone()
dist.all_reduce(hi, op=dist.ReduceOp.MAX)
dist.all_reduce(lo, op=dist.ReduceOp.MIN)
ok = torch.equal(hi, lo)
if rank == 0:
    model1, ml1, feats1, _, _ = _tpv_case(dev)
    d1, ref = unsharded(model1, ml1, feats1, metas, imgs)
    ok = ok and all(abs(d[k].item() - d1[k].item()) <= 1e-6 * abs(d1[k].item()) for k in d1)
    for g, g1 in zip(mean, ref):
        if g1 is not None:
            ok = ok and g is not None and (g - g1.cpu()).abs().max().item() <= 1e-5 * g1.abs().max().item()
flag = torch.tensor([int(bool(ok))])
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print('SHARD_OK' if int(flag) == 1 else 'SHARD_MISMATCH', world)
dist.destroy_process_group()
'''


def test_decode_sharded_step_two_processes_one_gpu(tmp_path):
    """The real per-rank path in two processes on one GPU: gloo carries host-staged buffers through the collective hooks of
    the loss gather and the volume exchange; the gradients are averaged with an explicit all_reduce."""
    _dev()
    script = tmp_path / 'gloo_worker.py'
    script.write_text(GLOO_WORKER % (ROOT, HERE))
    env = dict(os.environ, PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), '2', '29861'], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                              text=True, env=env) for r in range(2)]
    outs = []
    try:
        for p in procs:
            outs.append(p.communicate(timeout=900))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert 'SHARD_OK 2' in outs[0][0], outs[0][0][-3000:] + outs[0][1][-3000:] + outs[1][1][-3000:]


NCCL_WORKER = r'''
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, %r); sys.path.insert(0, %r)
from test_gpu_decode_shard import _tpv_case, unsharded
from test_gpu_encoder_shard import _objective_inputs
rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)
exchange = dist.new_group(backend='nccl')                 # the volume exchange on its own communicator
model, ml, feats, metas, imgs = _tpv_case(dev)
feats = [f.detach() for f in feats]
net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False)
model.head.ray_shard = (rank, world)
model.head.decode_shard = (rank, world)
model.head.decode_shard_group = exchange


def step(feats, metas):
    torch.manual_seed(0)
    np.random.seed(0)
    r = model.lifter(ms_img_feats=feats)
    rep = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)['representation']
    return _objective_inputs(model.head(representation=rep, metas=metas), imgs, metas)
model.forward = step                                       # DDP sees one module call per step
tot, d = ml(net(feats, metas))
tot.backward()
vals = torch.stack(list(d.values()))
hi, lo = vals.clone(), vals.clone()
dist.all_reduce(hi, op=dist.ReduceOp.MAX)
dist.all_reduce(lo, op=dist.ReduceOp.MIN)
ok = torch.equal(hi, lo)
params = [p for p in model.parameters() if p.requires_grad]
ddp = [None if p.grad is None else p.grad.clone() for p in params]
if rank == 0:                                              # the unsharded step on one GPU, on a model built the same way
    model1, ml1, _, _, _ = _tpv_case(dev)
    d1, ref = unsharded(model1, ml1, feats, metas, imgs)
    ok = ok and all(abs(d[k].item() - d1[k].item()) <= 1e-6 * abs(d1[k].item()) for k in d1)
    for g, g1 in zip(ddp, ref):
        if g1 is not None:
            ok = ok and g is not None and (g - g1).abs().max().item() <= 1e-5 * g1.abs().max().item()
flag = torch.tensor([int(bool(ok))], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print('SHARD_OK' if int(flag) == 1 else 'SHARD_MISMATCH', world)
dist.destroy_process_group()
'''


def test_decode_sharded_training_step_over_nccl_with_ddp(tmp_path):
    """Needs >= 2 GPUs: DDP + NCCL with head.decode_shard and head.ray_shard; every rank reports the same loss values and
    the DDP-averaged gradients equal the unsharded step's computed on rank 0."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    n = 3 if torch.cuda.device_count() >= 3 else 2
    script = tmp_path / 'worker.py'
    script.write_text(NCCL_WORKER % (ROOT, HERE))
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n), '--master-addr',
                        '127.0.0.1', '--master-port', '29871', str(script)], capture_output=True, text=True, timeout=900)
    assert 'SHARD_OK %d' % n in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
