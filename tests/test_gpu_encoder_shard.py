"""GPU: the query-sharded training pass of the encoder (TPVFormerEncoder.query_shard, forward_query_sharded: each rank runs
every layer on its own rows of each plane, dist.all_gather_rows rebuilds the planes, its backward reduce-scatters).

Emulated ranks run in lockstep in one process on the small training model of test_gpu_ray_shard (here with two encoder
layers, so the exchange's backward feeds a layer below it): per layer every rank's rows from the same RNG state, then the
emulated gather.  The gather's reduce-scatter is emulated inside ONE autograd graph: rank r's all_gather_rows returns its own
block of the gradient, and the other ranks' rows reach rank r's planes through a zero-valued path (x - x.detach()), so
the gradient of sum_r tot_r at rank s's rows is sum_r g_r there, as the reduce-scatter gives it.  grad(sum_r tot_r) / world
is then what DistributedDataParallel's mean gives.

Real processes: a two-process run on one GPU over gloo with host-staged collectives and an explicit gradient all_reduce,
and a torchrun / NCCL / DDP run on >= 2 GPUs (skipped below 2)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.dist import all_gather_rows, local_rows, pad_rows

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from test_gpu_ray_shard import CFGS, _build, _check_values  # noqa: E402
from test_ray_shard_cpu import emulated_ranks  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def small_training_model(dev, dropout=0.1, num_layers=2):
    """test_gpu_ray_shard.small_training_model with ``num_layers`` encoder layers and the encoder dropout ``dropout``."""
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=num_layers, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=32, ray_number=(48, 100), ray_img_size=(768, 1600),
                                  color_dims=24, return_sem=True, return_max_depth=False, ray_sample_mode='cellular',
                                  render_bkgd='random', dropout=dropout)
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
    model = build_head(cfg)
    model.encoder.init_weights()
    with torch.no_grad():
        model.head.model.field.deviation_network.variance.fill_(0.25)
    model.train().to(dev)
    l2i, i2l = synth.camera_rig()
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6, 768, 1600), generator=torch.Generator().manual_seed(2)).to(torch.uint8).numpy()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(768, 1600), sem=lab,
                  img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))]
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(1, 6, 96, h, w, generator=g).to(dev).requires_grad_(True) for h, w in synth.fpn_level_shapes(768, 1600)]
    imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
    return model, _build(CFGS['nuscenes/nuscenes_occ.py']), feats, metas, imgs


def _objective_inputs(out, imgs, metas):
    return dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas)


def unsharded_step(model, feats, metas, imgs, seed=0):
    """The existing training forward (query_shard None) -> (planes, objective inputs)."""
    torch.manual_seed(seed)
    np.random.seed(seed)
    model.head.ray_shard = None
    model.encoder.query_shard = None
    r = model.lifter(ms_img_feats=feats)
    rep = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)['representation']
    return rep, _objective_inputs(model.head(representation=rep, metas=metas), imgs, metas)


def _rng():
    return torch.get_rng_state(), torch.cuda.get_rng_state(), np.random.get_state()


def _set_rng(s):
    torch.set_rng_state(s[0])
    torch.cuda.set_rng_state(s[1])
    np.random.set_state(s[2])


def _place(local, idx, Q):
    return local.new_zeros(Q, local.shape[1]).index_put((idx,), local)


def lockstep_step(model, feats, metas, imgs, world, ray_shard=True, seed=0):
    """One query-sharded training forward of ``world`` emulated ranks in lockstep -> (per-rank planes, per-rank objective
    inputs, per layer the ranks' CUDA RNG states after the layer, the ranks' CUDA RNG states after the head)."""
    enc = model.encoder
    H, W, Z = enc.tpv_size
    sizes = [H * W, Z * H, W * Z]
    Q = sum(sizes)
    torch.manual_seed(seed)
    np.random.seed(seed)
    s0 = _rng()
    reps, sts = [], []
    for r in range(world):                      # replicated per rank: lifter, positional embedding, A3 / A4 set-up
        _set_rng(s0)
        reps.append(model.lifter(ms_img_feats=feats)['representation'])
        sts.append(enc.shard_state(feats, metas))
    qfull = [torch.cat([p[0] for p in rep], 0) for rep in reps]
    idx = [local_rows(torch.arange(Q, device=qfull[0].device), sizes, r, world) for r in range(world)]
    layer_states = []
    for li in range(len(enc.layers)):
        s = _rng()
        locs, after = [], []
        for r in range(world):
            _set_rng(s)
            locs.append(enc.shard_layer(li, qfull[r], sts[r], r, world))
            after.append(torch.cuda.get_rng_state())
        layer_states.append(after)
        bufs = [pad_rows(l.detach(), sizes, r, world) for r, l in enumerate(locs)]
        C = locs[0].shape[1]
        for r in range(world):
            full = all_gather_rows(locs[r], sizes, r, world, collective=lambda out, buf: torch.cat(bufs, out=out),
                                   reduce_scatter=lambda out, buf, r=r: out.copy_(buf.view(world, -1, C)[r]))
            for s_ in range(world):
                if s_ != r:
                    p = _place(locs[s_], idx[s_], Q)
                    full = full + (p - p.detach())
            qfull[r] = full
    planes = [[t[None] for t in torch.split(q, sizes, 0)] for q in qfull]
    s = _rng()
    inputs, head_states = [], []
    for r in range(world):
        _set_rng(s)
        model.head.ray_shard = (r, world) if ray_shard else None
        inputs.append(_objective_inputs(model.head(representation=planes[r], metas=metas), imgs, metas))
        head_states.append(torch.cuda.get_rng_state())
    model.head.ray_shard = None
    return planes, inputs, layer_states, head_states


def _wrt(model, feats):
    return [p for p in model.parameters() if p.requires_grad] + list(feats)


def _grads(tot, model, feats):
    return torch.autograd.grad(tot, _wrt(model, feats), allow_unused=True)


def _sharded_objective(ml, inputs, world, ray_shard):
    if ray_shard:
        return emulated_ranks(ml, inputs, world)
    return [ml(inp) for inp in inputs]


def _check_grads(got, ref, tol=1e-5):
    assert len(got) == len(ref)
    for i, (g, g1) in enumerate(zip(got, ref)):
        if g1 is None:
            assert g is None or not g.any(), i
            continue
        assert g is not None, i
        assert (g - g1).abs().max().item() <= tol * g1.abs().max().item(), (i, (g - g1).abs().max().item(), g1.abs().max().item())


def _sharded_grads(ml, model, feats, inputs, world, ray_shard):
    res = _sharded_objective(ml, inputs, world, ray_shard)
    tot = sum(t for t, _ in res)
    g = _grads(tot, model, feats)
    return res, [None if x is None else x / world for x in g]


@pytest.mark.parametrize('world', [2, 3])
def test_query_sharded_step_equals_unsharded_without_dropout(world):
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev, dropout=0.0)
    rep1, inp1 = unsharded_step(model, feats, metas, imgs)
    tot1, ref = ml(inp1)
    ref_g = _grads(tot1, model, feats)
    del inp1
    planes, inputs, _, _ = lockstep_step(model, feats, metas, imgs, world)
    for rep in planes:                                   # every row is computed as the unsharded forward computes it
        assert all(torch.equal(a, b) for a, b in zip(rep, rep1))
    assert all(inp['ray_shard'] == (r, world, 4800) for r, inp in enumerate(inputs))
    res, got = _sharded_grads(ml, model, feats, inputs, world, True)
    for _, d in res:
        _check_values(ref, d)
    _check_grads(got, ref_g)


def test_query_sharded_step_without_ray_shard():
    """Every rank renders all rays: each rank's objective is the whole objective, unscaled, and the rule still holds."""
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev, dropout=0.0)
    _, inp1 = unsharded_step(model, feats, metas, imgs)
    tot1, ref = ml(inp1)
    ref_g = _grads(tot1, model, feats)
    del inp1
    _, inputs, _, _ = lockstep_step(model, feats, metas, imgs, 2, ray_shard=False)
    res, got = _sharded_grads(ml, model, feats, inputs, 2, False)
    for _, d in res:
        _check_values(ref, d)
    _check_grads(got, ref_g)


def test_dropout_masks_of_the_row_routine_equal_the_unsharded_forward():
    """At dropout 0.1 the routine at world 1 draws the unsharded forward's masks: the same planes, bit for bit."""
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev, dropout=0.1)
    rep1, _ = unsharded_step(model, feats, metas, imgs)
    s1 = torch.cuda.get_rng_state()
    planes, _, layer_states, head_states = lockstep_step(model, feats, metas, imgs, 1)
    assert all(torch.equal(a, b) for a, b in zip(planes[0], rep1))
    assert torch.equal(head_states[0], s1)


@pytest.mark.parametrize('world', [2, 3])
def test_query_sharded_step_with_dropout_equals_world_one(world):
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev, dropout=0.1)
    planes1, inp1, _, _ = lockstep_step(model, feats, metas, imgs, 1)
    tot1, ref = ml(inp1[0])
    ref_g = _grads(tot1, model, feats)
    del inp1
    planes, inputs, layer_states, head_states = lockstep_step(model, feats, metas, imgs, world)
    for after in layer_states:                           # every rank leaves every layer with the same RNG state
        assert all(torch.equal(s, after[0]) for s in after)
    assert all(torch.equal(s, head_states[0]) for s in head_states)
    for rep in planes:                                   # one well-defined mask: the planes of the world-1 routine
        assert all(torch.equal(a, b) for a, b in zip(rep, planes1[0]))
    # the head draws the same jitter and background on every rank: each rank's rays carry the world-1 values
    res, got = _sharded_grads(ml, model, feats, inputs, world, True)
    for _, d in res:
        _check_values(ref, d)
    _check_grads(got, ref_g)


def test_query_shard_switch():
    dev = _dev()
    model, _, feats, metas, _ = small_training_model(dev, dropout=0.0, num_layers=1)
    enc = model.encoder
    rep = [p.detach() for p in model.lifter(ms_img_feats=feats)['representation']]
    calls = []
    orig = enc.forward_query_sharded

    def spy(*a, **k):
        calls.append(1)
        return orig(*a, **k)
    enc.forward_query_sharded = spy
    try:
        ref = enc(representation=rep, ms_img_feats=feats, metas=metas)['representation']
        for shard in (None, (0, 1)):                       # None and world 1: the existing path
            enc.query_shard = shard
            out = enc(representation=rep, ms_img_feats=feats, metas=metas)['representation']
            assert all(torch.equal(a, b) for a, b in zip(out, ref))
        assert not calls
        enc.query_shard = (0, 2)
        with torch.no_grad():                              # inference keeps its paths
            enc(representation=rep, ms_img_feats=feats, metas=metas)
        enc.eval()
        enc(representation=rep, ms_img_feats=feats, metas=metas)
        enc.train()
        assert not calls
        enc.query_shard_group = None
        smallest = min(enc.tpv_size[0] * enc.tpv_size[1], enc.tpv_size[2] * enc.tpv_size[0], enc.tpv_size[1] * enc.tpv_size[2])
        with pytest.raises(ValueError, match='ranks'):   # one rank more than the smallest plane has rows
            enc.forward_query_sharded(rep, feats, metas, 0, smallest + 1)
    finally:
        enc.query_shard = None
        del enc.forward_query_sharded


GLOO_WORKER = r'''
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, %r); sys.path.insert(0, %r)
from test_gpu_encoder_shard import small_training_model, unsharded_step, _objective_inputs, _wrt
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
model, ml, feats, metas, imgs = small_training_model(dev)
ml.collective = gather
torch.manual_seed(0)
import numpy as np; np.random.seed(0)
model.head.ray_shard = (rank, world)
r = model.lifter(ms_img_feats=feats)
rep = model.encoder.forward_query_sharded(r['representation'], feats, metas, rank, world, gather, reduce_scatter)
tot, d = ml(_objective_inputs(model.head(representation=rep, metas=metas), imgs, metas))
grads = torch.autograd.grad(tot, _wrt(model, feats), allow_unused=True)
ok = True
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
    model1, ml1, feats1, _, _ = small_training_model(dev)
    _, inputs1 = unsharded_step(model1, feats1, metas, imgs)
    tot1, d1 = ml1(inputs1)
    ref = torch.autograd.grad(tot1, _wrt(model1, feats1), allow_unused=True)
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


def test_query_sharded_step_two_processes_one_gpu(tmp_path):
    """The real per-rank autograd path in two processes on one GPU: gloo carries host-staged buffers through the collective
    hooks, the gradients are averaged with an explicit all_reduce, dropout 0.1 as shipped."""
    _dev()
    script = tmp_path / 'gloo_worker.py'
    script.write_text(GLOO_WORKER % (ROOT, HERE))
    env = dict(os.environ, PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), '2', '29781'], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
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
import torch, torch.distributed as dist
sys.path.insert(0, %r); sys.path.insert(0, %r)
from test_gpu_encoder_shard import small_training_model, unsharded_step, _objective_inputs
import numpy as np
rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)
exchange = dist.new_group(backend='nccl')                 # the encoder's exchange on its own communicator
model, ml, feats, metas, imgs = small_training_model(dev)
feats = [f.detach() for f in feats]
net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False)
model.head.ray_shard = (rank, world)
model.encoder.query_shard = (rank, world)
model.encoder.query_shard_group = exchange


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
    model1, ml1, _, _, _ = small_training_model(dev)
    _, inputs1 = unsharded_step(model1, feats, metas, imgs)
    tot1, d1 = ml1(inputs1)
    tot1.backward()
    ok = ok and all(abs(d[k].item() - d1[k].item()) <= 1e-6 * abs(d1[k].item()) for k in d1)
    for g, p in zip(ddp, [p for p in model1.parameters() if p.requires_grad]):
        if p.grad is not None:
            ok = ok and g is not None and (g - p.grad).abs().max().item() <= 1e-5 * p.grad.abs().max().item()
flag = torch.tensor([int(bool(ok))], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print('SHARD_OK' if int(flag) == 1 else 'SHARD_MISMATCH', world)
dist.destroy_process_group()
'''


def test_query_sharded_training_step_over_nccl_with_ddp(tmp_path):
    """Needs >= 2 GPUs: DDP + NCCL with encoder.query_shard and head.ray_shard; every rank reports the same loss values and
    the DDP-averaged gradients equal the unsharded step's computed on rank 0."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    n = 3 if torch.cuda.device_count() >= 3 else 2
    script = tmp_path / 'worker.py'
    script.write_text(NCCL_WORKER % (ROOT, HERE))
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n), '--master-addr',
                        '127.0.0.1', '--master-port', '29791', str(script)], capture_output=True, text=True, timeout=900)
    assert 'SHARD_OK %d' % n in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
