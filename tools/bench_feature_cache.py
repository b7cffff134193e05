"""Feature caching (the samplers' ``cache_interval`` / ``cache_branch``) on one GPU, at --height x --width (default
Vista's 576 x 1024) with the native-YAML engine of tools/bench_session.py (the vista UNet, seeded synthetic weights), a
trajectory action and sample.py's uc_keys.

Reported:
- the card and its power limit / max SM clock, read in the same run;
- the step time of a full step and of a cached step of branches 0 and 1, for Euler and 2M under the engine's guider:
  every step of an n-step schedule replayed from that kind of step's CUDA graph and timed with CUDA events, the variants
  alternating, as medians;
- the wall time of one session round, from ``step()`` to its uint8 frames on the host, at 50 Euler steps and at 25 2M
  steps, for cache_interval 1, 2, 3 and 5 (branch --branch), alternating;
- the time of one ``score`` call at its defaults (2 candidates x 5 members x 10 steps) for cache_interval 1 and 2;
- the final-latent rel-L2 of each cached round against the uncached one.  The weights are synthetic: this shows how far
  caching moves the sample, not what it does to frames from the real checkpoint;
- the peak allocated memory over the whole run.

    python tools/bench_feature_cache.py [--pairs 3] [--rounds 2] [--branch 0] [--height 576] [--width 1024] [--out r.json]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_session import TRAJECTORY, UC_KEYS, build_engine  # noqa: E402
from oracle.make_golden_clip import clip_frames  # noqa: E402
from vista_b200 import lib, synth  # noqa: E402
from vista_b200.diffusion import B200Denoiser, DPMPP2MSampler, EulerEDMSampler  # noqa: E402

INTERVALS = (1, 2, 3, 5)


def sampler(eng, multistep, steps, interval=1, branch=0):
    """Euler or 2M with the engine's discretisation and guider, ``steps`` steps, caching at ``interval``."""
    cls = DPMPP2MSampler if multistep else EulerEDMSampler
    s = cls(discretization_config={"target": "vista_b200.diffusion.EDMDiscretization"}, num_steps=steps,
            guider_config={"target": "vista_b200.diffusion.IdentityGuider"}, device=eng.sampler.device,
            cache_interval=interval, cache_branch=branch)
    s.discretization, s.guider = eng.sampler.discretization, eng.sampler.guider
    return s


def step_times(eng, den, inputs, n, pairs):
    """Every step of an n-step schedule replayed from one kind of step's graph, timed with events.  A cached sample of
    each branch first fills the loop state and captures the full and the cached graphs; replays start from its final
    state (the step time does not depend on the values)."""
    x, cond, uc, z, mask = inputs
    variants = []
    for ms in (False, True):
        for branch in (0, 1):
            sampler(eng, ms, n, 2, branch)(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask)
        tag = "2m" if ms else "euler"
        variants += [(f"{tag}_full", ms, False, 0), (f"{tag}_cached_b0", ms, True, 0), (f"{tag}_cached_b1", ms, True, 1)]
    rt = eng.model._rt_get(eng.model.diffusion_model, eng.num_frames, x.device)
    st = rt._loop_states[(x.shape[0], x.shape[2], x.shape[3])]
    out = {v[0]: [] for v in variants}
    for _ in range(pairs):
        for name, ms, cached, branch in variants:
            run = st.runner(rt, n, ms, False, True, cached, branch)
            st.step.zero_()
            for _ in range(n):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                out[name].append(e0.elapsed_time(e1))
    return {k: round(float(np.median(v)), 2) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3, help="the step-time variants alternated this many times")
    ap.add_argument("--rounds", type=int, default=2, help="timed session rounds per configuration")
    ap.add_argument("--branch", type=int, default=0, help="cache_branch of the session rounds and score calls")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--step-schedule", type=int, default=10, help="steps per timed schedule for the step time")
    ap.add_argument("--no-score", action="store_true", help="skip the score timing")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_feature_cache", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    act = {"trajectory": TRAJECTORY}
    z = torch.from_numpy(synth.normal(7, "bench_feature_cache.z", (T, 4, h, w), std=0.9)).to(dev)
    noise = torch.from_numpy(synth.normal(7, "bench_feature_cache.noise", (T, 4, h, w))).to(dev)
    den = B200Denoiser(eng.denoiser, eng.model)
    torch.cuda.reset_peak_memory_stats(dev)
    base = eng.sampler
    with torch.no_grad():
        cond, uc = eng.condition({**vd, **act}, T, UC_KEYS)
        mask = torch.zeros(T, device=dev)
        mask[0] = 1.0
        steps_ms = step_times(eng, den, (noise, cond, uc, z, mask), args.step_schedule, args.pairs)

        def session_round():
            sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sess.step(act, noise=noise).cpu()
            return time.perf_counter() - t0, sess.samples_z.double().clone()

        rounds, spread = {}, {}
        for ms, n in ((False, 50), (True, 25)):
            label = f"{'2m' if ms else 'euler'}_{n}"
            smps = {f"interval_{k}": sampler(eng, ms, n, k, args.branch) for k in INTERVALS}
            times, finals = {k: [] for k in smps}, {}
            for k, smp in smps.items():                   # warm-up (graph capture, decoder buffers)
                eng.sampler = smp
                session_round()
            for _ in range(args.rounds):
                for k, smp in smps.items():
                    eng.sampler = smp
                    t, finals[k] = session_round()
                    times[k].append(t)
            rounds[label] = {k: dict(runs=[round(t, 3) for t in v], median=round(float(np.median(v)), 3))
                             for k, v in times.items()}
            spread[label] = {k: float((finals[k] - finals["interval_1"]).norm() / finals["interval_1"].norm())
                             for k in smps if k != "interval_1"}
        score_s = {}
        if not args.no_score:
            eng.sampler = sampler(eng, False, 25)
            sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
            cands = [act, None]
            smps = {f"interval_{k}": sampler(eng, False, 10, k, args.branch) for k in (1, 2)}
            for smp in smps.values():                     # warm-up
                sess.score(cands, sampler=smp)
            for k, smp in smps.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rewards, _ = sess.score(cands, sampler=smp)
                rewards = rewards.cpu()
                score_s[k] = dict(seconds=round(time.perf_counter() - t0, 3), rewards=[float(r) for r in rewards])
        eng.sampler = base
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  branch=args.branch, step_ms_median=steps_ms, session_round_s=rounds, score_defaults_euler_s=score_s,
                  final_latent_rel_l2_vs_uncached_synthetic_weights=spread, peak_allocated_gib=round(peak / 2 ** 30, 2))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
