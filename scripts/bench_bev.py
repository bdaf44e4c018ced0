"""BEV-only model (config/nuscenes/nuscenes_occ_bev.py) on the GPU: the BEV decode against the fp32 torch composition of
bev_nerf.py:74-81 plus the copy into the volume layout, alternated in one session with their outputs compared, then a BEV
inference frame (lift + decode + render at the eval ray grid) and a BEV training step through the config's objective.

    python scripts/bench_bev.py [--rounds 10] [--iters 20] [--out DIR]

Prints one JSON line per measurement (and writes them to DIR/bench_bev.json), with the card's name and power limit."""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from selfocc_b200 import ops, synth                      # noqa: E402
from selfocc_b200.mapping import GridMeterMapping        # noqa: E402
from selfocc_b200.registry import build_head, LOSSES     # noqa: E402
import selfocc_b200.segmentor  # noqa: E402,F401
import selfocc_b200.loss  # noqa: E402,F401

HBM_TBS, TF32_TFLOPS = 3.35, 495.0                       # H100 SXM data sheet (dense TF32), for the floors only


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def bench_decode(cfg, rounds, iters):
    dev = torch.device('cuda:0')
    f = GridMeterMapping(**cfg['head']['mapping_args'])
    n_feat = cfg['head']['color_dims']
    desc = f.volume_desc(n_feat)
    H, W, Z, Cf, Cc = desc.H, desc.W, desc.Z, 1 + n_feat, cfg['head']['embed_dims']
    g = torch.Generator().manual_seed(0)
    bev = (0.7 * torch.randn(H * W, Cc, generator=g)).to(dev)
    w1, b1 = (torch.randn(Cc, Cc, generator=g) / Cc ** 0.5).to(dev), (0.1 * torch.randn(Cc, generator=g)).to(dev)
    w2, b2 = (torch.randn(Z * Cf, Cc, generator=g) / Cc ** 0.5).to(dev), (0.1 * torch.randn(Z * Cf, generator=g)).to(dev)
    vs_t = torch.zeros(H, W, desc.zpitch, device=dev)
    vf_t = torch.zeros(H, W, Z, desc.feat_pitch, device=dev)

    def kernel():
        return ops.bev_decode(bev, w1, b1, w2, b2, desc)

    def composition():
        out = F.linear(F.softplus(F.linear(F.softplus(bev), w1, b1)), w2, b2).view(H, W, Z, Cf)
        vs_t[..., :Z] = out[..., 0]
        vf_t[..., :n_feat] = out[..., 1:]
        return vs_t, vf_t

    assert not torch.backends.cuda.matmul.allow_tf32          # the composition is the fp32 reference formulation
    for fn in (kernel, composition):
        timed(fn, 3)
    tk, tc = [], []
    for _ in range(rounds):                                     # alternate: both see the same clocks and neighbours
        tk.append(timed(kernel, iters))
        tc.append(timed(composition, iters))
    vs, vf = kernel()
    composition()
    diff_s = (vs[..., :Z] - vs_t[..., :Z]).abs().max().item()
    diff_f = (vf[..., :n_feat] - vf_t[..., :n_feat]).abs().max().item()
    bytes_out = H * W * (desc.zpitch + Z * desc.feat_pitch) * 4
    flop = 3 * 2 * H * W * (Cc * Cc + Cc * Z * Cf)
    floor_us = max(bytes_out / (HBM_TBS * 1e12), flop / (TF32_TFLOPS * 1e12)) * 1e6
    return dict(name='bev_decode', H=H, W=W, Z=Z, Cf=Cf, C=Cc, kernel_us=1e3 * median(tk), torch_composition_us=1e3 * median(tc),
                kernel_us_spread=[1e3 * min(tk), 1e3 * max(tk)], speedup=median(tc) / median(tk), max_abs_diff_sdf=diff_s,
                max_abs_diff_feat=diff_f, bytes_written=bytes_out, flop_3xtf32=flop, floor_us=floor_us,
                floor_share=floor_us / (1e3 * median(tk)))


def build_model(cfg, dev):
    torch.manual_seed(0)
    model = build_head(dict(type='TPVHotPath', **cfg)).to(dev)
    with torch.no_grad():
        model.head.model.field.deviation_network.variance.fill_(0.25)
    return model


def frame_inputs(cfg, dev, training):
    img = tuple(cfg['head']['ray_img_size'])
    l2i, i2l = synth.camera_rig()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), temImg2lidar=list(i2l), img_shape=img)]
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(1, 6, cfg['encoder']['embed_dims'], h, w, generator=g).to(dev) for h, w in synth.fpn_level_shapes(*img)]
    extra = {}
    if training:
        prev, nxt = synth.temporal_rig()
        metas[0].update(sem=torch.randint(0, 17, (6,) + img, generator=g).to(torch.uint8).numpy(),
                        img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                        img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))
        imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
        extra = dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3])
    return metas, feats, extra


def bench_frame(cfg, rounds, iters):
    dev = torch.device('cuda:0')
    model = build_model(cfg, dev).eval()
    metas, feats, _ = frame_inputs(cfg, dev, False)
    os.environ['eval'] = 'true'                                 # the head's eval ray grid

    def frame():
        with torch.no_grad():
            model(ms_img_feats=feats, metas=metas, prepare=True)
            return model.head.render(metas=metas)
    timed(frame, 2)
    ts = [timed(frame, iters) for _ in range(rounds)]
    out = frame()
    os.environ.pop('eval')
    return dict(name='bev_frame', rays=out['ms_depths'][0].numel(), samples=model.head.num_samples, ms=median(ts),
                ms_spread=[min(ts), max(ts)], depth_finite=bool(torch.isfinite(out['ms_depths'][0]).all()))


def bench_train_step(cfg, rounds, iters):
    dev = torch.device('cuda:0')
    c = copy.deepcopy(cfg)
    c['head']['second_grad_assumption'] = True
    model = build_model(c, dev).train()
    metas, feats, extra = frame_inputs(c, dev, True)
    cfgs = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_multiloss_cfgs.json')))
    loss = LOSSES.build(cfgs['nuscenes/nuscenes_occ_bev.py'])
    state = {}

    def step():
        model.zero_grad(set_to_none=True)
        out = model(ms_img_feats=feats, metas=metas)
        tot, _ = loss(dict(out, metas=metas, **extra))
        tot.backward()
        state['loss'] = tot
    timed(step, 2)
    ts = [timed(step, iters) for _ in range(rounds)]
    return dict(name='bev_train_step', ms=median(ts), ms_spread=[min(ts), max(ts)], loss=state['loss'].item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_bev.py measures on the GPU: no CUDA device')
    cfg = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_model_cfgs_bev.json')))['nuscenes/nuscenes_occ_bev.py']
    gpu = card()
    res = [bench_decode(cfg, args.rounds, args.iters), bench_frame(cfg, args.rounds, max(1, args.iters // 4)),
           bench_train_step(cfg, max(2, args.rounds // 3), max(1, args.iters // 10))]
    lines = [json.dumps(dict(r, gpu=gpu)) for r in res]
    print('\n'.join(lines))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, 'bench_bev.json'), 'w').write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
