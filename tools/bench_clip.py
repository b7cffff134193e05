"""CUDA-event time of the conditioner's CLIP image embedder on one GPU: the native tower (vista_b200.clip) against the
torch-eager fp16 tower (transformers' CLIPVisionModelWithProjection holding the same weights, preprocess in torch fp32 as
the kornia restatement of oracle/clip_oracle.py) on the same frames.  Default: the conditioning call of do_sample, 25 rows
of one 576 x 1024 frame (get_batch repeats it, sample_utils.py:243-244), ViT-H/14 with synthetic weights.

    python tools/bench_clip.py [--rows 25] [--reps 10] [--preset vit_h_14]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_oracle as co  # noqa: E402
from oracle.make_golden_clip import clip_frames, clip_weights, hf_vision_from_open_clip  # noqa: E402
from vista_b200 import lib  # noqa: E402
from vista_b200.clip import FrozenOpenCLIPImagePredictionEmbedder  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=25)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--preset", default="vit_h_14")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    cfg, sd = clip_weights(args.preset, 12)
    frame = torch.from_numpy(clip_frames(12, "bench", 1, args.height, args.width))
    x = frame.expand(args.rows, -1, -1, -1).contiguous().to(dev)

    emb = FrozenOpenCLIPImagePredictionEmbedder(
        {"target": "vista_b200.clip.FrozenOpenCLIPImageEmbedder", "params": {"arch": cfg}}, n_cond_frames=1, n_copies=1)
    emb.load_state_dict({"open_clip.model.visual." + k: torch.from_numpy(v) for k, v in sd.items()})
    emb = emb.to(dev)
    native_ms, z = timed(lambda: emb(x), args.reps)
    z = z.float().clone()

    hf = hf_vision_from_open_clip(cfg, sd).to(dev).half()

    @torch.no_grad()
    def eager():
        return hf(pixel_values=co.preprocess(x, True).half()).image_embeds

    eager_ms, ze = timed(eager, args.reps)
    rel = float((z.reshape(ze.shape) - ze.float()).norm() / ze.float().norm())
    flops = 2.0 * args.rows * cfg.tokens * (12 * cfg.width ** 2) * cfg.layers \
        + 4.0 * args.rows * cfg.heads * cfg.tokens ** 2 * cfg.head_width * cfg.layers
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps(dict(device=torch.cuda.get_device_name(dev), power_limit=power, preset=args.preset, rows=args.rows,
                          frame=[args.height, args.width], native_ms=round(native_ms, 3), eager_fp16_ms=round(eager_ms, 3),
                          speedup=round(eager_ms / native_ms, 3), native_tflops=round(flops / native_ms / 1e9, 1),
                          rel_l2_native_vs_eager=rel)))


if __name__ == "__main__":
    main()
