"""One encoder layer's attention cores, forward + backward, at BASELINE configs[4] sizes (fp32), in two compositions on
identical seeded inputs:
  (a) fused: ops.TPVSelfAttnFunction / ops.TPVCrossAttnFunction (the inference kernels + their backward kernels);
  (b) reference contract: torch softmax + location arithmetic + ops.MultiScaleDeformableAttnFunction, and for the image
      cross-attention the per-camera rebatch built from ops.visible_index_lists (one host sync per plane), the padded
      [cams, Lmax, ...] copies and index_add back into the query rows (BEVCrossAttention._rebatch_forward).
Sizes: self-attention over the 257 x 257 x 25 TPV queries (3 levels x 12 points), cross-attention of the three planes
(8 / 48 / 48 pillar points) over 6 cameras x 4 FPN levels of a 768 x 1600 rig; 6 heads x 16 channels.
    python scripts/bench_train_attn.py [--iters K] [--warmup W]
The two compositions alternate; each is timed with device events.  Prints one JSON line: ms and peak memory per
composition and core, the largest differences of outputs and gradients between (a) and (b), the GPU name and power limit."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfocc_b200 import ops, synth                          # noqa: E402
from selfocc_b200.encoder import _pillar_tables, _cross_view_refs   # noqa: E402
from selfocc_b200.mapping import GridMeterMapping            # noqa: E402

MAPPING = dict(synth.NUSC_MAPPING, h_size=[128, 0], h_range=[40.0, 0], w_size=[128, 0], w_range=[40.0, 0], d_size=[24, 0],
               d_range=[-1.0, 5.4, 5.4])
IMG = (768, 1600)
HEADS, DH, P_SELF, P_CROSS = 6, 16, 12, (48, 48, 8)           # num_points_cross = [p_wz, p_zh, p_hw]


def _levels(shapes, dev):
    ss = torch.tensor(shapes, dtype=torch.int64)
    return ss.to(dev), torch.cat([ss.new_zeros(1), ss.prod(1).cumsum(0)[:-1]]).to(dev)


def make_inputs(dev, seed=0, mapping=MAPPING, img=IMG, n_cam=6):
    """Seeded core inputs of one layer: {'self': dict, 'cross': [dict per plane hw, zh, wz]}.  Offsets are a few pixels
    (some samples leave the feature maps), logits O(1), incoming gradients N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    m = GridMeterMapping(**mapping)
    H, W, Z = m.size_h, m.size_w, m.size_d
    C = HEADS * DH
    s_shapes = [(H, W), (Z, H), (W, Z)]
    Qs = H * W + Z * H + W * Z
    ss, lsi = _levels(s_shapes, dev)
    slf = dict(value=torch.randn(Qs, HEADS, DH, generator=g), offsets=2.0 * torch.randn(Qs, HEADS, 3, P_SELF, 2, generator=g),
               logits=torch.randn(Qs, HEADS, 3, P_SELF, generator=g), ref=_cross_view_refs(H, W, Z, P_SELF),
               grad=torch.randn(Qs, C, generator=g))
    slf = {k: v.to(dev).contiguous() for k, v in slf.items()}
    slf.update(ss=ss, lsi=lsi)
    f_shapes = synth.fpn_level_shapes(*img)
    Nv = sum(h * w for h, w in f_shapes)
    fss, flsi = _levels(f_shapes, dev)
    l2i, _ = synth.camera_rig()
    l2i = torch.tensor(l2i, dtype=torch.float32, device=dev)
    cross = []
    for r3 in _pillar_tables(m, list(P_CROSS)):
        D, Q = r3.shape[:2]
        uv, mask, vis = ops.point_sampling(r3.contiguous().to(dev), l2i, img)
        t = dict(value=torch.randn(n_cam, Nv, HEADS, DH, generator=g), offsets=2.0 * torch.randn(Q, HEADS, 4, D, 2, generator=g),
                 logits=torch.randn(Q, HEADS, 4, D, generator=g), grad=torch.randn(Q, C, generator=g))
        t = {k: v.to(dev).contiguous() for k, v in t.items()}
        t.update(uv=uv, mask=mask, vis=vis, ss=fss, lsi=flsi)
        cross.append(t)
    return {'self': slf, 'cross': cross}


def _leaves(t):
    return [t[k].detach().clone().requires_grad_(True) for k in ('value', 'offsets', 'logits')]


def _normalizer(ss, dtype):
    return torch.stack([ss[..., 1], ss[..., 0]], -1).to(dtype)


def self_fused(t):
    v, o, lg = _leaves(t)
    out = ops.TPVSelfAttnFunction.apply(v, t['ss'], t['lsi'], o, lg, t['ref'])
    out.backward(t['grad'])
    return out.detach(), v.grad, o.grad, lg.grad


def self_reference(t):
    """cross_view_hybrid_attention.py:88-116 at the core: softmax, ref + offsets / (w, h), mmcv-contract op."""
    v, o, lg = _leaves(t)
    Q, Hd, L, P, _ = o.shape
    aw = lg.view(1, Q, Hd, L * P).softmax(-1).view(1, Q, Hd, L, P)
    loc = t['ref'][None, :, None] + o[None] / _normalizer(t['ss'], o.dtype)[None, None, None, :, None, :]
    out = ops.MultiScaleDeformableAttnFunction.apply(v[None], t['ss'], t['lsi'], loc, aw, 64)[0]
    out.backward(t['grad'])
    return out.detach(), v.grad, o.grad, lg.grad


def cross_fused(t):
    v, o, lg = _leaves(t)
    out = ops.TPVCrossAttnFunction.apply(v, t['ss'], t['lsi'], o, lg, t['uv'], t['vis'])
    out.backward(t['grad'])
    return out.detach(), v.grad, o.grad, lg.grad


def cross_reference(t):
    """image_cross_attention.py:84-136, 313-345 at the core: visible-query lists, padded per-camera rebatch of the
    query-side operands, softmax, ref + offsets / (w, h), mmcv-contract op, index_add back, divide by the count."""
    v, o, lg = _leaves(t)
    Q, Hd, L, D, _ = o.shape
    N = v.shape[0]
    lists, lens = ops.visible_index_lists(t['mask'])
    lens = lens.tolist()                                                   # the host sync of the reference formulation
    lmax = max(max(lens), 1)
    idx = [lists[i, :lens[i]] for i in range(N)]
    o_re = o.new_zeros(N, lmax, Hd, L, D, 2)
    lg_re = lg.new_zeros(N, lmax, Hd, L, D)
    r_re = t['uv'].new_zeros(N, lmax, D, 2)
    for i in range(N):
        o_re[i, :lens[i]] = o[idx[i]]
        lg_re[i, :lens[i]] = lg[idx[i]]
        r_re[i, :lens[i]] = t['uv'][i, idx[i]]
    aw = lg_re.view(N, lmax, Hd, L * D).softmax(-1).view(N, lmax, Hd, L, D)
    loc = r_re[:, :, None, None] + o_re / _normalizer(t['ss'], o.dtype)[None, None, None, :, None, :]
    res = ops.MultiScaleDeformableAttnFunction.apply(v, t['ss'], t['lsi'], loc, aw, 64)
    slots = v.new_zeros(Q, Hd * v.shape[-1])
    for i in range(N):
        slots = slots.index_add(0, idx[i], res[i, :lens[i]])
    count = (t['mask'].sum(-1) > 0).sum(0).clamp(min=1)
    out = slots / count[:, None]
    out.backward(t['grad'])
    return out.detach(), v.grad, o.grad, lg.grad


def diffs(a, b):
    """max |a - b| and max |a - b| / max |b| for outputs and each gradient."""
    res = {}
    for name, x, y in zip(('out', 'grad_value', 'grad_offsets', 'grad_logits'), a, b):
        d = (x - y).abs().max().item()
        res[name] = {'max_abs': d, 'max_rel': d / max(y.abs().max().item(), 1e-30)}
    return res


def _gpu_info():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl or 'unknown'


def _timed(fn, t, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a.record()
    for _ in range(iters):
        fn(t)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def main():
    iters = int(sys.argv[sys.argv.index('--iters') + 1]) if '--iters' in sys.argv else 10
    warmup = int(sys.argv[sys.argv.index('--warmup') + 1]) if '--warmup' in sys.argv else 3
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_attn.py measures on a CUDA device; none is visible')
    dev = torch.device('cuda')
    inp = make_inputs(dev)
    cores = [('self', inp['self'], self_fused, self_reference)] + \
            [('cross_' + n, t, cross_fused, cross_reference) for n, t in zip(('hw', 'zh', 'wz'), inp['cross'])]
    result = {'workload': 'one encoder layer attention, fwd + bwd, TPV 257x257x25, 6 cams x 4 FPN levels of 768x1600, '
                          '6 heads x 16 ch, fp32', 'iters': iters, 'warmup': warmup, 'cores': {}}
    tot = {'fused': 0.0, 'reference': 0.0}
    for name, t, fa, fb in cores:
        for _ in range(warmup):
            fa(t); fb(t)
        ms = {'fused': [], 'reference': []}
        mem = {'fused': 0.0, 'reference': 0.0}
        for _ in range(2):                                       # alternate (a) and (b)
            for key, fn in (('fused', fa), ('reference', fb)):
                m, pk = _timed(fn, t, iters)
                ms[key].append(m)
                mem[key] = max(mem[key], pk)
        entry = {'ms_fused': ms['fused'], 'ms_reference': ms['reference'], 'peak_extra_gb_fused': mem['fused'],
                 'peak_extra_gb_reference': mem['reference'], 'diff': diffs(fa(t), fb(t))}
        if name.startswith('cross'):
            entry['queries'], entry['pillar_points'] = t['offsets'].shape[0], t['offsets'].shape[3]
        result['cores'][name] = entry
        tot['fused'] += min(ms['fused'])
        tot['reference'] += min(ms['reference'])
    result['ms_layer_fused'], result['ms_layer_reference'] = tot['fused'], tot['reference']
    result['gpu'], result['power_limit'] = _gpu_info()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
