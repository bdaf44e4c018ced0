"""Device timing of so_linear_3xtf32 for the 12 projection launches of one encoder layer of the flagship frame
(6 x 900 x 1600, cfg 3), each with the epilogue the layer uses.  Per shape: ms per launch, achieved GB/s over the
algorithmic bytes (X + W hi/lo + Y + residual), TFLOP/s of tensor work (the three split products) and the share of
the larger of the two data-sheet floors (H100 SXM: 3.35 TB/s HBM3, 495 TFLOP/s dense TF32).

    python scripts/bench_gemm.py [--iters 20] [--json OUT]
"""
import argparse, json, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfocc_b200 import ops

HBM_GBS, TF32_TFLOPS = 3350.0, 495.0
# name, M, N, K, epilogue ('bias', 'relu' or 'ln': + residual, then LayerNorm over the row)
SHAPES = [('self value_proj', 81983, 96, 96, 'bias'), ('self offsets+logits', 81983, 648, 96, 'bias'),
          ('self output_proj+res+LN', 81983, 96, 96, 'ln'), ('img value_proj x3', 153000, 288, 96, 'bias'),
          ('hw offsets+logits', 66049, 576, 96, 'bias'), ('zh offsets+logits', 7967, 3456, 96, 'bias'),
          ('wz offsets+logits', 7967, 3456, 96, 'bias'), ('hw output_proj+res+LN', 66049, 96, 96, 'ln'),
          ('zh output_proj+res+LN', 7967, 96, 96, 'ln'), ('wz output_proj+res+LN', 7967, 96, 96, 'ln'),
          ('ffn1 relu', 81983, 192, 96, 'relu'), ('ffn2+res+LN', 81983, 96, 192, 'ln')]


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return 'unknown (%r)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--json', help='also write the result list to this file')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    g = torch.Generator(device=dev).manual_seed(0)
    res, tot_ms, tot_floor = [], 0.0, 0.0
    for name, M, N, K, epi in SHAPES:
        x = torch.randn(M, K, device=dev, generator=g)
        w = torch.randn(N, K, device=dev, generator=g) * 0.1
        b = torch.randn(N, device=dev, generator=g)
        r = torch.randn(M, N, device=dev, generator=g) if epi == 'ln' else None
        ln = (1 + 0.1 * torch.randn(N, device=dev, generator=g), torch.randn(N, device=dev, generator=g), 1e-5) if epi == 'ln' else None
        y = torch.empty(M, N, device=dev)
        hi, lo = ops.split_tf32(w)

        def fn():
            ops.linear_3xtf32(x, hi, lo, b, relu=epi == 'relu', residual=r, out=y, ln=ln)
        for _ in range(3):
            fn()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(e) / args.iters
        nbytes = (M * K + 2 * N * K + M * N + (M * N if r is not None else 0)) * 4
        flop = 3 * 2 * M * N * K
        floor_ms = max(nbytes / (HBM_GBS * 1e9), flop / (TF32_TFLOPS * 1e12)) * 1e3
        bound = 'hbm' if nbytes / HBM_GBS > flop / TF32_TFLOPS / 1e3 else 'tf32'
        tot_ms += ms
        tot_floor += floor_ms
        res.append(dict(name=name, M=M, N=N, K=K, epilogue=epi, ms=round(ms, 4), GBps=round(nbytes / (ms * 1e-3) / 1e9, 1),
                        TFLOPs=round(flop / (ms * 1e-3) / 1e12, 1), floor_ms=round(floor_ms, 4), bound=bound,
                        frac_of_floor=round(floor_ms / ms, 3)))
        print(json.dumps(res[-1]))
        del x, w, b, r, y, hi, lo
    summary = dict(gpu=gpu_info(), layer_ms=round(tot_ms, 4), layer_floor_ms=round(tot_floor, 4),
                   frame_ms_4_layers=round(4 * tot_ms, 3), frame_floor_ms_4_layers=round(4 * tot_floor, 3))
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(shapes=res, summary=summary), f, indent=1)


if __name__ == '__main__':
    main()
