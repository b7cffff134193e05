"""Scoring candidate actions from a rollout session, on one GPU: the engine of tools/bench_session.py
(configs/inference/vista_b200_native.yaml with the vista UNet and decoder, the ViT-H/14 CLIP tower and the vista encoder,
seeded synthetic weights) on a --height x --width clip, sample.py's uc_keys.  ``RolloutSession.score`` rates --candidates
trajectory actions with an ensemble of --ensemble members of --steps EDM steps each (reward.py's defaults: 5 members,
10 steps), at round 0 and, after one session round of the engine's 50 steps, at round 1.

Reported per round: the wall time of every score call (host clock, ended by a device synchronise) and the median per
candidate; the peak allocated memory over the score calls, with the session and the engine resident; and whether the
repeated calls returned bit-identical rewards.  Also the peak of the session step between the two rounds.  One untimed
score (one candidate, two members) comes first: it packs the weights and captures the --steps-step CUDA graph.

    python tools/bench_score.py [--candidates 2] [--ensemble 5] [--steps 10] [--reps 2] [--height 576] [--width 1024]
                                [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_session import TRAJECTORY, UC_KEYS, build_engine  # noqa: E402
from oracle.make_golden_clip import clip_frames  # noqa: E402
from vista_b200 import lib, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--candidates", type=int, default=2)
    ap.add_argument("--ensemble", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10, help="EDM steps of every ensemble member")
    ap.add_argument("--reps", type=int, default=2, help="timed score calls per round")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_score", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "bench_score.z", (T, 4, h, w), std=0.9)).to(dev)
    noise = torch.from_numpy(synth.normal(7, "bench_score.noise0", (T, 4, h, w))).to(dev)
    # candidate k adds 0.5 k, 1.0 k, 1.5 k and 2.0 k to the trajectory's four lateral offsets
    candidates = []
    for k in range(args.candidates):
        t = TRAJECTORY.clone()
        t[0::2] += 0.5 * k * torch.arange(1, 5, dtype=t.dtype)
        candidates.append({"trajectory": t})

    sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
    sess.score(candidates[:1], ensemble_size=2, num_steps=args.steps)          # warm-up
    torch.cuda.synchronize()

    def timed_scores():
        torch.cuda.reset_peak_memory_stats(dev)
        secs, rewards = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r, _ = sess.score(candidates, ensemble_size=args.ensemble, num_steps=args.steps)
            torch.cuda.synchronize()
            secs.append(time.perf_counter() - t0)
            rewards.append(r.cpu())
        return dict(score_s=[round(s, 3) for s in secs],
                    s_per_candidate_median=round(float(np.median(secs)) / args.candidates, 3),
                    rewards=[round(float(v), 6) for v in rewards[0]],
                    repeat_bit_identical=all(torch.equal(r, rewards[0]) for r in rewards),
                    score_peak_allocated_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))

    rounds = {"0": timed_scores()}
    torch.cuda.reset_peak_memory_stats(dev)
    sess.step(candidates[0], noise=noise)
    torch.cuda.synchronize()
    step_peak = torch.cuda.max_memory_allocated(dev)
    rounds["1"] = timed_scores()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  candidates=args.candidates, ensemble=args.ensemble, steps=args.steps, session_steps=eng.sampler.num_steps,
                  rounds=rounds, step_peak_allocated_gib=round(step_peak / 2 ** 30, 2))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
