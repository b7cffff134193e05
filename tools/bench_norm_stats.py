"""Times the GroupNorm statistics paths: gn_stats + gn_apply (ops.groupnorm) at the VAE decoder's full-resolution
shapes, and the tap-GEMM with fused statistics (ops.gemm(..., stats=)) at the decoder's and the UNet's level-0 shapes,
with CUDA events over many launches after a warm-up.  Prints one JSON line per shape and the card's name and power
limit.  Run it from two trees, alternating, to compare builds.

    python tools/bench_norm_stats.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TAPS_3X3 = [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from vista_b200 import lib, ops
    lib.load()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}))
    g = torch.Generator(device=dev).manual_seed(0)
    res = []
    # decoder GroupNorms at full resolution, statistics over one frame (spatial) and over a 14-frame chunk (temporal)
    for T, H, W, C, fps in ((14, 576, 1024, 128, 1), (14, 288, 512, 256, 1), (14, 144, 256, 512, 1),
                            (14, 576, 1024, 128, 14)):
        x = (torch.randn(T * H * W, C, generator=g, device=dev) + 3).half()
        y = torch.empty_like(x)
        gamma = torch.ones(C, device=dev)
        beta = torch.zeros(C, device=dev)
        ws = ops.GNWorkspace(dev)
        ms = timed(lambda: ops.groupnorm(x, y, T, H * W, gamma, beta, 1e-6, True, frames_per_stat=fps, ws=ws), args.reps)
        res.append({"op": "groupnorm", "shape": [T, H, W, C], "fps": fps, "ms": round(ms, 4),
                    "GB/s": round(2 * x.numel() * 2 * 1e-6 / ms, 1)})
        del x, y
    # STATS tap-GEMMs: decoder 3x3 conv 128 -> 128 at 576 x 1024, 256 -> 256 at 288 x 512; UNet level 0 3x3 320 -> 320
    for NB, H, W, Cin, C in ((2, 576, 1024, 128, 128), (4, 288, 512, 256, 256), (50, 72, 128, 320, 320)):
        a = torch.randn(NB * H * W, Cin, generator=g, device=dev).half()
        w = (torch.randn(C, 9 * Cin, generator=g, device=dev) * (9 * Cin) ** -0.5).half()
        bias = torch.randn(C, generator=g, device=dev)
        out = torch.empty(NB * H * W, C, dtype=torch.float16, device=dev)
        part = torch.empty(NB * H * W // 32, C, 2, dtype=torch.float32, device=dev)
        ms = timed(lambda: ops.gemm(a, w, out, taps=TAPS_3X3, geom=(W, H, NB), bias=bias, stats=part), args.reps)
        res.append({"op": "gemm_stats", "shape": [NB, H, W, Cin, C], "ms": round(ms, 4),
                    "TFLOP/s": round(2 * NB * H * W * 9 * Cin * C * 1e-9 / ms, 1)})
        del a, out, part
    for r in res:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
