"""SparsityLoss, HardSparsityLoss and AdaptiveSparsityLoss, forward + backward: the native terms (so_sparsity_*,
so_hard_sparsity_*, so_adaptive_sparsity_*) against the reference's torch composition (loss/sparsity_loss.py, restated
below), alternated in one session after warm-up.  Sizes: nuscenes_occ's uniform_sdf lattice (200 x 200 x 16) for the two
lattice terms, nuScenes_occ's rays (6 cameras x 48x100 rays x 256 samples) for the adaptive term.

Reported per term: median CUDA-event time of one forward + backward for each side, host synchronisations per step
(torch.cuda sync-debug warnings) and the relative difference of the two sides' values.  The card's name and power limit are
read in the same run.  Prints one JSON line (and writes it to --out if given).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

LATTICE = (200, 200, 16)
N_CAM, R, S = 6, 48 * 100, 256


# ---- the reference's terms (loss/sparsity_loss.py), fp32 torch
def ref_sparsity(density, scale=0.1):
    return torch.pow(1.0 / torch.cosh(density / (2.0 * scale)), 2).mean()


def ref_hard(density, scale=1.0, thresh=0.2, crop=((2, 2), (2, 2), (1, 1))):
    density = density.clone()          # the reference crops in place; the clone keeps the timed input (and autograd) intact
    (h0, h1), (w0, w1), (d0, d1) = crop
    density[:h0, ...] = 100
    density[-h1:, ...] = 100
    density[:, :w0, :] = 100
    density[:, -w1:, :] = 100
    density[..., :d0] = 100
    density[..., -d1:] = 100
    return torch.relu(torch.sigmoid(-1 * scale * density).mean() - thresh)


def ref_adaptive(sdfs, ts, ms_depths, slack=4.0):
    depths = ms_depths[0]
    bs, num_cams, num_rays = depths.shape
    t = torch.stack(ts, dim=0).reshape(bs, num_cams, num_rays, -1)
    s = torch.stack(sdfs, dim=0).reshape(bs, num_cams, num_rays, -1)
    return torch.relu(-1 * s[t > (depths + slack).unsqueeze(-1)]).mean()


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(',')]
    except Exception:              # noqa: BLE001  the numbers stay usable without the label
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def time_steps(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return sum('synchroniz' in str(x.message) and 'prototype' not in str(x.message) for x in w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50, help='timed steps per side and term (alternated)')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_sparsity measures on the GPU'
    import selfocc_b200.loss as L
    dev = torch.device('cuda:0')
    g = torch.Generator(device=dev).manual_seed(0)
    lat = (torch.randn(*LATTICE, device=dev, generator=g) * 0.5).requires_grad_(True)
    sdf = torch.randn(N_CAM, R * S, device=dev, generator=g).requires_grad_(True)
    ts = (0.5 + 45 * torch.rand(N_CAM, R, S, device=dev, generator=g)).sort(-1).values.reshape(N_CAM, R * S)
    depth = 1 + 40 * torch.rand(1, N_CAM, R, device=dev, generator=g)
    crop = [[2, 2], [2, 2], [1, 1]]
    sp, hard = L.SparsityLoss(scale=0.1), L.HardSparsityLoss(crop=crop)
    ad = L.AdaptiveSparsityLoss(input_dict=dict(sdfs='sample_sdf', ts='ts', ms_depths='ms_depths'))
    adin = dict(sample_sdf=list(sdf.unbind(0)), ts=list(ts.unbind(0)), ms_depths=[depth])
    terms = {
        'SparsityLoss': (lambda: sp({'density': lat}), lambda: ref_sparsity(lat), lat),
        'HardSparsityLoss': (lambda: hard({'density': lat}), lambda: ref_hard(lat, crop=crop), lat),
        'AdaptiveSparsityLoss': (lambda: ad(adin), lambda: ref_adaptive(list(sdf.unbind(0)), list(ts.unbind(0)), [depth]), sdf),
    }
    res = {}
    for name, (nat, ref, leaf) in terms.items():
        def step(f):
            loss = f()
            loss.backward()
            leaf.grad = None
            return loss.detach()
        vn, vr = step(nat), step(ref)
        for _ in range(a.warmup):
            step(nat), step(ref)
        tn, tr = [], []
        for _ in range(a.iters):                       # alternate the two sides
            tn += time_steps(lambda: step(nat), 1)
            tr += time_steps(lambda: step(ref), 1)
        res[name] = dict(native_ms=round(statistics.median(tn), 4), reference_ms=round(statistics.median(tr), 4),
                         speedup=round(statistics.median(tr) / statistics.median(tn), 2),
                         native_syncs=count_syncs(lambda: step(nat)), reference_syncs=count_syncs(lambda: step(ref)),
                         value_rel_diff=abs(vn.item() - vr.item()) / max(abs(vr.item()), 1e-30))
    name, power = card()
    out = dict(bench='sparsity_terms', gpu=name, power_limit=power, lattice=list(LATTICE), rays=[N_CAM, R, S],
               iters=a.iters, terms=res)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
