"""The photometric reprojection loss (ReprojLossMonoMultiNewCombine, the nuScenes configs' objective), forward + backward to
the rendering weights, at nuScenes_occ sizes: 6 cameras x 48x100 rays x 256 samples, 768x1600 fp32 images, SSIM and
automask on.  Two compositions on identical seeded inputs:
  (a) native: selfocc_b200.loss (so_reproj_stats_forward / _backward + the per-ray torch tail);
  (b) reference contract: oracle/reproj.py's restatement in fp32 on the same GPU (per-camera batched matmul, grid_sample,
      index_add over the samples, autograd keeping the per-sample intermediates), the composition the reference runs.
    python scripts/bench_train_loss.py [--iters K] [--warmup W]
The two alternate, two timed windows each, device events.  Also timed: the statistics kernels alone, and a repack of the
three image stacks into a channel-last float4 copy (the alternative gather layout), to size it against the kernels.
Prints one JSON line: ms and peak memory above the inputs per composition, loss and gradient differences, GPU name and
power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from selfocc_b200 import ops                                      # noqa: E402
from selfocc_b200.loss import ReprojLossMonoMultiNewCombine       # noqa: E402
from oracle.reproj import reproj_loss_ref                         # noqa: E402
from test_gpu_reproj_loss import NUSC, make_case, _native         # noqa: E402


def _gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(',')]
    except Exception as e:                 # noqa: BLE001
        return [torch.cuda.get_device_name(), 'unknown (%s)' % type(e).__name__]


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    case = make_case(dev, **NUSC)
    m, w, inputs = _native(ReprojLossMonoMultiNewCombine, case, True, True, False)

    def native():
        w.grad = None
        m(inputs).backward()
        return w.grad

    def reference():
        w.grad = None
        reproj_loss_ref('combine', case['curr'][0], case['prev'][0], case['next'][0], list(w.unbind(0)), list(case['ts'].unbind(0)),
                        case['img2prev'], case['img2next'], case['rays'], case['img_size'], case['ray_resize']).backward()
        return w.grad

    arms = {'native': native, 'reference_contract': reference}
    res = {k: dict(ms=[], peak_mem_mb=[]) for k in arms}
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    for _ in range(2):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            res[k]['ms'].append(timed(fn, args.iters))
            res[k]['peak_mem_mb'].append((torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    gn, gr = native().clone(), reference().clone()
    with torch.no_grad():
        ln = float(m(inputs))
        lr = float(reproj_loss_ref('combine', case['curr'][0], case['prev'][0], case['next'][0], list(w.unbind(0)),
                                   list(case['ts'].unbind(0)), case['img2prev'], case['img2next'], case['rays'], case['img_size'],
                                   case['ray_resize']))

    # the statistics kernels alone, and the channel-last repack they would need per step to gather 16-byte texels
    N, R, S = w.shape[0], case['rays'].shape[0], case['S']
    cfg = dict(mode='combine', shape=(N, R, S), ts=case['ts'], deltas=None, pix=case['rays'], img2prev=case['img2prev'],
               img2next=case['img2next'], images=(case['curr'][0], case['prev'][0], case['next'][0]), img_size=case['img_size'])
    stats, _ = ops.ReprojStatsFunction.apply(cfg, *w.unbind(0))
    g_stats = torch.randn_like(stats)
    fwd = lambda: ops.ReprojStatsFunction.apply(cfg, *w.detach().unbind(0))
    bwd = lambda: torch.autograd.grad(stats, w, g_stats, retain_graph=True)
    fwd(), bwd()
    fwd_ms, bwd_ms = timed(fwd, args.iters), timed(bwd, args.iters)
    hwc = torch.empty(3, N, case['img_size'][0], case['img_size'][1], 4, device=dev)

    def repack():
        for i, im in enumerate((case['curr'], case['prev'], case['next'])):
            hwc[i, ..., :3].copy_(im[0].permute(0, 2, 3, 1))
    repack_ms = timed(repack, args.iters)
    name, power = _gpu()
    print(json.dumps({
        'workload': 'ReprojLossMonoMultiNewCombine fwd+bwd, 6 cams x 48x100 rays x 256 samples, 768x1600 fp32 images, ssim + automask',
        'gpu': name, 'power_limit': power,
        'native_ms': res['native']['ms'], 'reference_contract_ms': res['reference_contract']['ms'],
        'native_peak_mem_mb': res['native']['peak_mem_mb'], 'reference_contract_peak_mem_mb': res['reference_contract']['peak_mem_mb'],
        'stats_forward_kernel_ms': fwd_ms, 'stats_backward_kernel_ms': bwd_ms, 'hwc_float4_repack_ms': repack_ms,
        'loss_native': ln, 'loss_reference_contract': lr, 'loss_rel_diff': abs(ln - lr) / abs(lr),
        'grad_max_abs_diff_over_max': float((gn - gr).abs().max() / gr.abs().max())}))


if __name__ == '__main__':
    main()
