"""CPU: the sparsity terms of loss/sparsity_loss.py (SparsityLoss, HardSparsityLoss, AdaptiveSparsityLoss).  The fp64 oracle
against the reference's own outputs (golden vectors), the configs' commented loss blocks built through LOSSES / MultiLoss,
fuse_objective's rules on them, the input left uncropped, AdaptiveSparsityLoss over gloo on two ranks against one, and the
argument checks of the new entry points."""
import json
import os
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'reference_golden_sparsity.npz')
CFGS = os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')

# the commented blocks of the shipped configs (config/*/*.py): SparsityLoss in all seven, AdaptiveSparsityLoss in
# nuscenes_occ.py just before it; AdaptiveSparsityLoss's sdfs mapped to the head's sample_sdf (its default key is not
# emitted by NeuSHead)
SPARSITY_BLOCK = dict(type='SparsityLoss', weight=0.001, scale=0.1, input_dict={'density': 'uniform_sdf'})
ADAPTIVE_BLOCK = dict(type='AdaptiveSparsityLoss', weight=0.001, slack=4.0,
                      input_dict={'sdfs': 'sample_sdf', 'ts': 'ts', 'ms_depths': 'ms_depths'})


def _gold(dtype):
    z = np.load(GOLD)
    return z, (lambda k: torch.from_numpy(z[k]).to(dtype))


def _hard_cfg(z, tag):
    c = z['HardSparsityLoss_%s_cfg' % tag]
    return float(c[0]), float(c[1]), [[int(c[2]), int(c[3])], [int(c[4]), int(c[5])], [int(c[6]), int(c[7])]]


def _check(loss, grad, z, tag, name, rtol=1e-6):
    ref = float(z[tag + '_loss'])
    if np.isnan(ref):
        assert torch.isnan(loss), tag
    else:
        assert abs(float(loss) - ref) <= rtol * max(abs(ref), 1e-30), (tag, float(loss), ref)
    r = z['%s_grad_%s' % (tag, name)]
    g = grad.double().numpy()
    fin = np.isfinite(r)
    scale = np.abs(r[fin]).max() if fin.any() else 0.
    assert np.abs(g[fin] - r[fin]).max() <= rtol * scale, (tag, np.abs(g[fin] - r[fin]).max(), scale)
    return fin


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_oracle_matches_reference_golden(dtype):
    import oracle.sparsity as O
    z, t = _gold(dtype)
    for tag, scale in (('s01', 0.1), ('s1', 1.0)):
        x = t('dens').requires_grad_(True)
        loss = O.sparsity_ref(x, scale)
        loss.backward()
        fin = _check(loss.detach(), x.grad, z, 'SparsityLoss_' + tag, 'dens')
        # where the reference's fp32 cosh overflows its gradient is 0 * inf = NaN; the oracle (and the kernel) give 0
        over = np.abs(z['dens'].astype(np.float64)) / (2 * scale) > 89.
        assert over.any() and np.array_equal(~fin, over), tag
        assert np.abs(x.grad.numpy()[over]).max() <= 1e-30 and torch.isfinite(x.grad).all()   # 0 once fp32 underflows
    for tag in ('nocrop', 'crop', 'allcrop', 'inactive', 'slope'):
        scale, thresh, crop = _hard_cfg(z, tag)
        x = t('dens').requires_grad_(True)
        before = x.detach().clone()
        loss = O.hard_sparsity_ref(x, scale, thresh, crop)
        loss.backward()
        _check(loss.detach(), x.grad, z, 'HardSparsityLoss_' + tag, 'dens')
        assert torch.equal(x.detach(), before)
    for tag, dk in (('masked', 'depths'), ('empty', 'depths_far')):
        s = t('sdfs').requires_grad_(True)
        loss = O.adaptive_sparsity_ref(list(s.unbind(0)), list(t('ts').unbind(0)), t(dk), float(z['slack']))
        loss.backward()
        _check(loss.detach(), s.grad, z, 'AdaptiveSparsityLoss_' + tag, 'sdfs')


def test_golden_cases_cover_the_edge_cases():
    z, t = _gold(torch.float64)
    assert float(z['HardSparsityLoss_inactive_loss']) == 0 and float(z['HardSparsityLoss_allcrop_loss']) > 0
    assert not z['HardSparsityLoss_allcrop_grad_dens'].any()                 # every cell cropped: no gradient
    crop = z['HardSparsityLoss_crop_grad_dens']
    assert crop.any() and not crop[0].any() and not crop[-2:].any() and not crop[:, :2].any() and not crop[..., -1].any()
    assert np.isnan(z['AdaptiveSparsityLoss_empty_loss']) and not z['AdaptiveSparsityLoss_empty_grad_sdfs'].any()
    mask = t('ts').reshape(2, 12, 16) > (t('depths')[0] + 4.0)[..., None]
    per_ray = mask.sum(-1)
    assert (per_ray == 0).sum() >= 3 and (per_ray > 0).sum() >= 10


def _cfgs():
    return json.load(open(CFGS))


def test_commented_config_blocks_build_through_multiloss():
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss as L
    for name, c in _cfgs().items():
        extra = ([ADAPTIVE_BLOCK] if name == 'nuscenes/nuscenes_occ.py' else []) + [SPARSITY_BLOCK]
        m = LOSSES.build(dict(c, loss_cfgs=c['loss_cfgs'] + extra))
        assert isinstance(m, L.MultiLoss) and m.num_losses == len(c['loss_cfgs']) + len(extra)
        sp = m.losses[-1]
        assert type(sp) is L.SparsityLoss and sp.weight == 0.001 and sp.scale == 0.1
        assert sp.input_dict == {'density': 'uniform_sdf'}
        if extra[0] is ADAPTIVE_BLOCK:
            ad = m.losses[-2]
            assert type(ad) is L.AdaptiveSparsityLoss and ad.weight == 0.001 and ad.slack == 4.0
            assert ad.input_dict == ADAPTIVE_BLOCK['input_dict']
    hard = LOSSES.build(dict(type='HardSparsityLoss', weight=0.01, scale=2.0, thresh=0.1, crop=[[1, 0], [0, 2], [0, 0]],
                             input_dict={'density': 'uniform_sdf'}))
    assert (hard.scale, hard.thresh, hard.crop, hard.weight) == (2.0, 0.1, [[1, 0], [0, 2], [0, 0]], 0.01)
    # the reference's defaults
    d = L.SparsityLoss(), L.HardSparsityLoss(), L.AdaptiveSparsityLoss()
    assert d[0].scale == 1.0 and d[0].input_dict == {'density': 'density'}
    assert (d[1].scale, d[1].thresh, d[1].crop) == (1.0, 0.2, [[0, 0], [0, 0], [0, 0]])
    assert d[2].slack == 4.0 and d[2].weight == 1 and d[2].input_dict == {'sdfs': 'sdfs', 'ts': 'ts', 'ms_depths': 'ms_depths'}


def test_adaptive_sparsity_names_a_missing_key():
    import selfocc_b200.loss as L
    inputs = dict(ts=[torch.zeros(8)], ms_depths=[torch.zeros(1, 1, 2)], sample_sdf=[torch.zeros(8)])
    with pytest.raises(KeyError, match="'sdfs'.*sample_sdf.*return_sample_sdf"):
        L.AdaptiveSparsityLoss()(inputs)
    del inputs['sample_sdf']
    with pytest.raises(KeyError, match="'sample_sdf'"):
        L.AdaptiveSparsityLoss(input_dict=ADAPTIVE_BLOCK['input_dict'])(inputs)


def test_fuse_objective_accepts_the_lattice_terms_and_refuses_the_per_sample_one():
    from selfocc_b200.loss import MultiLoss, fuse_objective
    head = types.SimpleNamespace(two_split=False, return_sample_sdf=False)
    base = _cfgs()['nuscenes/nuscenes_occ.py']['loss_cfgs']
    hard = dict(type='HardSparsityLoss', weight=0.01, crop=[[1, 1], [0, 0], [0, 0]], input_dict={'density': 'uniform_sdf'})
    got = fuse_objective(head, MultiLoss(base + [SPARSITY_BLOCK, hard]))
    assert got == dict(mode='combine', img_size=(768, 1600), eikonal=True) and head.fused_objective is got
    head.fused_objective = None
    with pytest.raises(NotImplementedError, match='AdaptiveSparsityLoss reads per-sample outputs'):
        fuse_objective(head, MultiLoss(base + [ADAPTIVE_BLOCK, SPARSITY_BLOCK]))
    assert head.fused_objective is None


def test_hard_sparsity_leaves_its_input_for_the_next_term(monkeypatch):
    """The reference writes 100 into the crop borders of the caller's uniform_sdf, so SoftSparsityLoss listed after it sees
    the cropped lattice; here the module hands the tensor to the kernel (stood in for by the oracle on the CPU; the GPU
    test runs the kernel) and nothing writes it."""
    import oracle.sparsity as O
    from oracle.losses import soft_sparsity_ref
    from selfocc_b200 import ops
    from selfocc_b200.loss import MultiLoss
    monkeypatch.setattr(ops.HardSparsityFunction, 'apply', lambda x, s, t, c: O.hard_sparsity_ref(x, s, t, c))
    monkeypatch.setattr(ops.SampleMeanFunction, 'apply', lambda x, op: soft_sparsity_ref(x))
    z, t = _gold(torch.float32)
    x = t('dens')
    before = x.clone()
    hard = dict(type='HardSparsityLoss', crop=[[1, 2], [2, 1], [1, 1]], thresh=0.05, input_dict={'density': 'uniform_sdf'})
    soft = dict(type='SoftSparsityLoss', input_dict={'density': 'uniform_sdf'})
    tot, d = MultiLoss([hard, soft])({'uniform_sdf': x})
    assert torch.equal(x, before)
    assert abs(float(d['HardSparsityLoss']) - float(z['HardSparsityLoss_crop_loss'])) <= 1e-6 * float(z['HardSparsityLoss_crop_loss'])
    assert float(d['SoftSparsityLoss']) == float(soft_sparsity_ref(before))


def test_lattice_terms_under_ray_sharding_read_the_replicated_lattice():
    import selfocc_b200.loss as L
    for cls in (L.SparsityLoss, L.HardSparsityLoss):
        assert cls(input_dict={'density': 'uniform_sdf'}).local_payload({}, (0, 2, 10)) == []
        with pytest.raises(NotImplementedError, match='%s under ray sharding takes the replicated uniform_sdf' % cls.__name__):
            cls(input_dict={'density': 'sample_sdf'}).local_payload({}, (0, 2, 10))


# ---- AdaptiveSparsityLoss on two gloo ranks: the kernels are stood in for by torch restatements of their contract (per ray
# (sum, count) in fp64, their ratio); tests/test_gpu_sparsity.py runs the kernels on emulated ranks
N_CAM, R, S = 3, 7 * 5, 8


class _RaysStandIn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, slack, ts, depth, *sdfs):
        m = torch.stack([t.reshape(depth.shape[1], -1) for t in ts]) > (depth + slack)[..., None]
        s = torch.stack([x.reshape(depth.shape[1], -1) for x in sdfs])
        ctx.shapes = [x.shape for x in sdfs]
        ctx.save_for_backward(m, s)
        return torch.stack([(torch.relu(-s) * m).double().sum(-1), m.double().sum(-1)], -1)

    @staticmethod
    def backward(ctx, g):
        m, s = ctx.saved_tensors
        gs = -g[..., 0:1].float() * (m & (s < 0))
        return (None, None, None) + tuple(x.reshape(shp) for x, shp in zip(gs.unbind(0), ctx.shapes))


def _reduce_stand_in(st):
    st = st.reshape(-1, 2)
    return (st[:, 0].sum() / st[:, 1].sum().detach()).float()


def _adaptive_case():
    g = torch.Generator().manual_seed(5)
    ts = (0.5 + 40 * torch.rand(N_CAM, R, S, generator=g)).sort(-1).values
    depths = 1 + 30 * torch.rand(1, N_CAM, R, generator=g)
    sdfs = torch.randn(N_CAM, R, S, generator=g)
    return sdfs, ts, depths


def _adaptive_inputs(sdfs, ts, depths):
    """The head's outputs for the rays given: per camera R * S samples ray-major, depths [1, N, R]."""
    return dict(sample_sdf=[s.reshape(-1) for s in sdfs], ts=[t.reshape(-1) for t in ts], ms_depths=[depths])


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from selfocc_b200 import ops
    from selfocc_b200.dist import ray_slice
    from selfocc_b200.loss import MultiLoss
    ops.AdaptiveSparsityRaysFunction.apply = _RaysStandIn.apply
    ops.AdaptiveSparsityReduceFunction.apply = _reduce_stand_in
    sdfs, ts, depths = _adaptive_case()
    ml = MultiLoss([ADAPTIVE_BLOCK])
    full = sdfs.clone().requires_grad_(True)
    ref, _ = ml(_adaptive_inputs(full, ts, depths))
    g_ref, = torch.autograd.grad(ref, full)
    b, c = ray_slice(R, world, rank)
    own = sdfs[:, b:b + c].clone().requires_grad_(True)
    tot, d = ml(dict(_adaptive_inputs(own, ts[:, b:b + c], depths[:, :, b:b + c]), ray_shard=(rank, world, R)))
    g, = torch.autograd.grad(tot, own)
    ok = torch.equal(tot, ref) and torch.equal(d['AdaptiveSparsityLoss'], ref.detach())
    ok = ok and (g / world - g_ref[:, b:b + c]).abs().max().item() <= 1e-7 * g_ref.abs().max().item()
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_adaptive_sparsity_on_two_gloo_ranks_equals_one_rank():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, 29871, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(60) for p in procs]
    assert res == [(0, True), (1, True)]


def test_sparsity_entry_points_are_exported_and_reject_bad_arguments_without_a_gpu():
    """Null pointers, bad sizes, bad scales, negative crops, mis-aligned pointers: SO_ERR_INVALID_ARG (-1) before any CUDA
    call; empty ray sets are no-ops."""
    import ctypes as C
    import subprocess
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    nm = subprocess.run(['nm', '-D', '--defined-only', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = ('so_sparsity_forward', 'so_sparsity_backward', 'so_hard_sparsity_forward', 'so_hard_sparsity_backward',
             'so_adaptive_sparsity_rays', 'so_adaptive_sparsity_reduce', 'so_adaptive_sparsity_backward')
    hdr = open(os.path.join(HERE, '..', 'include', 'selfocc_b200.h')).read()
    for n in names:
        assert n in nm and n in _lib.SIGNATURES and n + '(' in hdr, n
    N, one, ws = None, C.c_void_p(16), C.c_void_p(64)
    sf, sb = lib.so_sparsity_forward, lib.so_sparsity_backward
    assert sf(N, 8, 0.1, ws, one, N) == -1 and sf(one, 8, 0.1, N, one, N) == -1 and sf(one, 8, 0.1, ws, N, N) == -1
    assert sf(one, 0, 0.1, ws, one, N) == -1 and sb(one, -1, 0.1, one, one, N) == -1
    for bad in (0.0, float('inf'), float('nan')):
        assert sf(one, 8, bad, ws, one, N) == -1 and sb(one, 8, bad, one, one, N) == -1
    assert sf(C.c_void_p(18), 8, 0.1, ws, one, N) == -1 and sf(one, 8, 0.1, C.c_void_p(20), one, N) == -1
    assert sb(one, 8, 0.1, N, one, N) == -1 and sb(one, 8, 0.1, one, C.c_void_p(18), N) == -1
    hf, hb = lib.so_hard_sparsity_forward, lib.so_hard_sparsity_backward
    crop = (C.c_int32 * 6)(0, 0, 0, 0, 0, 0)
    neg = (C.c_int32 * 6)(0, 0, -1, 0, 0, 0)
    assert hf(N, 4, 4, 4, crop, 1.0, 0.2, ws, one, N) == -1
    assert hf(one, 0, 4, 4, crop, 1.0, 0.2, ws, one, N) == -1 and hf(one, 4, 4, -1, crop, 1.0, 0.2, ws, one, N) == -1
    assert hf(one, 2048, 2048, 1024, crop, 1.0, 0.2, ws, one, N) == -1                 # 2^32 cells: 32-bit indices
    assert hf(one, 4, 4, 4, neg, 1.0, 0.2, ws, one, N) == -1
    assert hf(one, 4, 4, 4, crop, float('nan'), 0.2, ws, one, N) == -1 and hf(one, 4, 4, 4, crop, 1.0, float('inf'), ws, one, N) == -1
    assert hf(one, 4, 4, 4, crop, 1.0, 0.2, N, one, N) == -1
    assert hb(one, 4, 4, 4, crop, 1.0, N, one, one, N) == -1 and hb(one, 4, 4, 4, neg, 1.0, one, one, one, N) == -1
    assert hb(one, 4, 4, 4, crop, 1.0, one, one, C.c_void_p(18), N) == -1
    ar, rd, ab = lib.so_adaptive_sparsity_rays, lib.so_adaptive_sparsity_reduce, lib.so_adaptive_sparsity_backward
    assert ar(N, one, one, 4, 16, 4.0, one, N) == -1 and ar(one, one, one, 4, 0, 4.0, one, N) == -1
    assert ar(one, one, one, -1, 16, 4.0, one, N) == -1 and ar(one, one, one, 4, 16, float('nan'), one, N) == -1
    assert ar(one, one, one, 4, 16, 4.0, C.c_void_p(24), N) == -1                       # stats not 16-byte aligned
    assert ar(N, N, N, 0, 16, 4.0, N, N) == 0 and ab(N, N, N, 0, 16, 4.0, N, N, N) == 0   # no rays: nothing to do
    assert rd(N, 4, ws, one, N, N) == -1 and rd(one, 0, ws, one, N, N) == -1 and rd(one, 4, C.c_void_p(72), one, N, N) == -1
    assert rd(one, 4, ws, N, N, N) == -1 and rd(C.c_void_p(24), 4, ws, one, N, N) == -1
    assert ab(one, one, one, 4, 16, 4.0, N, one, N) == -1 and ab(one, one, one, 4, 16, 4.0, one, C.c_void_p(18), N) == -1
    assert lib.so_abi_version() == 10
