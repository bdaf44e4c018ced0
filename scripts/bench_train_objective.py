"""nuscenes_occ's training objective, forward and backward, on seeded synthetic head outputs at nuScenes_occ sizes
(6 cameras x 48x100 rays x 256 samples, 768x1600 images, 17 semantic classes):
    python scripts/bench_train_objective.py [--iters 10]
Two paths, alternated on the same GPU:
  native     selfocc_b200.loss.MultiLoss built from the config's loss dict (reprojection statistics kernel, the per-sample
             loss-term kernel for EikonalLoss / SecondGradLoss, torch for the per-ray RGB / semantic terms);
  reference  the same five terms composed as the reference does, in fp32 torch (oracle/reproj.py, oracle/losses.py), with
             the reference MultiLoss's `.item()` per term.
Prints one JSON line: ms per step and peak memory above the inputs for each path, kernel-only times of the three
loss-term ops (forward, backward), host syncs per step (torch.cuda sync-debug warnings), the loss and gradient
differences between the paths, and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfocc_b200 import synth, ops  # noqa: E402
from selfocc_b200.registry import LOSSES  # noqa: E402
import selfocc_b200.loss  # noqa: E402,F401

N, RH, RW, S, C = 6, 48, 100, 256, 17
IMG, RR = [768, 1600], [RH, RW]
CFG = [dict(type='ReprojLossMonoMultiNewCombine', weight=1.0, no_ssim=False, img_size=IMG, ray_resize=RR,
            input_dict={k: k for k in ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')}),
       dict(type='RGBLossMS', weight=0.1, img_size=IMG, no_ssim=False, ray_resize=RR,
            input_dict={'ms_colors': 'ms_colors', 'ms_rays': 'ms_rays', 'gt_imgs': 'color_imgs'}),
       dict(type='EikonalLoss', weight=0.1), dict(type='SecondGradLoss', weight=0.01),
       dict(type='SemCELossMS', weight=0.1, img_size=IMG, ray_resize=RR, input_dict={'sem': 'sem', 'metas': 'metas', 'ms_rays': 'ms_rays'})]


def make_inputs(dev):
    g = torch.Generator().manual_seed(0)
    R = RH * RW
    ys, xs = torch.meshgrid(torch.arange(RH), torch.arange(RW), indexing='ij')
    rays = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * IMG[1] / RW,
                        (ys.flatten() + torch.rand(R, generator=g)) * IMG[0] / RH], -1).to(dev)
    prev, nxt = synth.temporal_rig()
    imgs = synth.textured_images(4 * N, *IMG, seed=2).reshape(4, 1, N, 3, *IMG).to(dev)
    lab = torch.randint(0, C, (N, *IMG), generator=g).to(torch.uint8).numpy()
    metas = [dict(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev), sem=lab)]
    gd = torch.Generator(device=dev).manual_seed(1)
    leaves = dict(weights=torch.rand(N, R * S, device=dev, generator=gd) / S,
                  ms_colors=torch.rand(1, N, R, 3, device=dev, generator=gd),
                  sem=torch.softmax(3 * torch.randn(1, N, R, C, device=dev, generator=gd), -1),
                  eik_grad=0.6 * torch.randn(N * R, S, 3, device=dev, generator=gd),
                  second_grad=torch.randn(N * R, S, 3, device=dev, generator=gd))
    leaves = {k: v.requires_grad_(True) for k, v in leaves.items()}
    ts = (0.5 + 40 * torch.rand(N, R * S, device=dev, generator=gd)).sort(-1).values
    inputs = dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas, ms_rays=rays,
                  ray_indices=[torch.arange(R, device=dev).repeat_interleave(S)] * N, ts=list(ts.unbind(0)))
    return inputs, leaves


def with_leaves(inputs, leaves):
    return dict(inputs, weights=list(leaves['weights'].unbind(0)), ms_colors=[leaves['ms_colors']], sem=[leaves['sem']],
                eik_grad=leaves['eik_grad'], second_grad=leaves['second_grad'])


def native_step(ml, inputs, leaves):
    tot, d = ml(with_leaves(inputs, leaves))
    return tot, torch.autograd.grad(tot, list(leaves.values()))


def reference_step(inputs, leaves):
    """The reference's composition in fp32 torch, with its MultiLoss's per-term `.item()`."""
    from oracle.reproj import reproj_loss_ref
    import oracle.losses as O
    x = with_leaves(inputs, leaves)
    m = x['metas'][0]
    lab = torch.from_numpy(m['sem'][None]).to(leaves['sem'].device)
    terms = [reproj_loss_ref('combine', x['curr_imgs'][0], x['prev_imgs'][0], x['next_imgs'][0], x['weights'], x['ts'],
                             m['img2prevImg'], m['img2nextImg'], x['ms_rays'], IMG, RR),
             0.1 * O.rgb_ref(x['ms_colors'], x['ms_rays'], x['color_imgs'], IMG, RR, no_ssim=False),
             0.1 * O.eikonal_ref(x['eik_grad']), 0.01 * O.second_grad_ref(x['second_grad']),
             0.1 * O.sem_ce_ref(x['sem'], lab, x['ms_rays'])]
    tot, loss_dict = 0., {}
    for c, t in zip(CFG, terms):
        tot = tot + t
        loss_dict[c['type']] = t.detach().item()
    return tot, torch.autograd.grad(tot, list(leaves.values()))


def timed(fn, iters):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, out


def syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    # the notice that sync-debug mode is a prototype is not a synchronisation
    return sum(1 for x in w if 'synchroniz' in str(x.message).lower() and 'prototype' not in str(x.message).lower())


def card():
    name, power = torch.cuda.get_device_name(0), None
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
        name, power = q[0], float(q[1])
    except Exception:
        pass
    return name, power


def kernel_ms(x, op, iters):
    """Forward and backward of one loss-term op alone, device-timed."""
    xl = x.detach().requires_grad_(True)
    f = lambda: ops.SampleMeanFunction.apply(xl, op)
    g1 = torch.ones((), device=x.device)
    for _ in range(3):
        torch.autograd.grad(f(), xl, g1)
    fwd, _, loss = timed(f, iters)
    bwd, _, _ = timed(lambda: torch.autograd.grad(loss, xl, g1, retain_graph=True), iters)
    return round(fwd, 4), round(bwd, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    inputs, leaves = make_inputs(dev)
    ml = LOSSES.build(dict(type='MultiLoss', loss_cfgs=CFG))
    nat = lambda: native_step(ml, inputs, leaves)
    ref = lambda: reference_step(inputs, leaves)
    for _ in range(2):
        nat(), ref()
    res = {'native': [], 'reference': []}
    for _ in range(3):                                            # alternated
        for name, fn in (('native', nat), ('reference', ref)):
            res[name].append(timed(fn, args.iters))
    (ln, gn), (lr, gr) = nat(), ref()
    grad_err = {k: (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30) for k, a, b in zip(leaves, gn, gr)}
    name, power = card()
    n_in = sum(v.numel() for v in leaves.values())
    print(json.dumps({
        'workload': 'nuscenes_occ objective (reprojection, RGB+SSIM, eikonal, second-grad, semantic CE), forward + backward, '
                    '6 cams x 48x100 rays x 256 samples, fp32',
        'card': name, 'power_limit_w': power,
        'native_ms': sorted(round(r[0], 3) for r in res['native']),
        'reference_ms': sorted(round(r[0], 3) for r in res['reference']),
        'native_peak_mib_above_inputs': round(max(r[1] for r in res['native']), 1),
        'reference_peak_mib_above_inputs': round(max(r[1] for r in res['reference']), 1),
        'kernel_ms_fwd_bwd': {'eikonal': kernel_ms(leaves['eik_grad'], 'eikonal', args.iters),
                              'abs': kernel_ms(leaves['second_grad'], 'abs', args.iters),
                              'neg_relu': kernel_ms(torch.randn(200, 200, 16, device=dev), 'neg_relu', args.iters)},
        'host_syncs_per_step': {'native': syncs(nat), 'reference': syncs(ref)},
        'loss': {'native': ln.item(), 'reference': lr.item(), 'rel_diff': abs(ln.item() - lr.item()) / abs(lr.item())},
        'grad_rel_max_diff': grad_err, 'input_floats': n_in}))


if __name__ == '__main__':
    main()
