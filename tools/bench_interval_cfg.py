"""Interval guidance (vista_b200.diffusion.IntervalCFG) on one GPU, at --height x --width (default Vista's 576 x 1024)
with the native-YAML engine of tools/bench_session.py (the vista UNet, seeded synthetic weights), a trajectory action and
sample.py's uc_keys.

Reported:
- the card and its power limit / max SM clock, read in the same run;
- the step time of a guided step and of a conditional-only step, for Euler and 2M, wrapping the engine's guider
  (VanillaCFG-style per-frame guidance) and wrapping ActionCFG over it: every step of an n-step schedule replayed from
  that kind of step's CUDA graph and timed with CUDA events, the variants alternating, as medians;
- the wall time of one session round, from ``step()`` to its uint8 frames on the host, at 50 Euler steps and at 25 2M
  steps, for full guidance, for the interval (0.28, 5.42] and for an empty interval, the three alternating;
- the final-latent rel-L2 of the interval and empty-interval rounds against full guidance.  The weights are synthetic:
  this shows how far the schedule moves the sample, not what it does to frames from the real checkpoint;
- the peak allocated memory over the whole run.

    python tools/bench_interval_cfg.py [--pairs 3] [--rounds 2] [--height 576] [--width 1024] [--out result.json]
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
from vista_b200.diffusion import (ActionCFG, B200Denoiser, DPMPP2MSampler, EulerEDMSampler, IdentityGuider,  # noqa: E402
                                  IntervalCFG)

PAPER_INTERVAL = (0.28, 5.42)        # Kynkaanniemi et al. 2024's example interval for EDM


def sampler(eng, multistep, guider, steps):
    """Euler or 2M with the engine's discretisation and ``guider`` (an instance), ``steps`` steps."""
    cls = DPMPP2MSampler if multistep else EulerEDMSampler
    s = cls(discretization_config={"target": "vista_b200.diffusion.EDMDiscretization"}, num_steps=steps,
            guider_config={"target": "vista_b200.diffusion.IdentityGuider"}, device=eng.sampler.device)
    s.discretization, s.guider = eng.sampler.discretization, guider
    return s


def interval(lo, hi, inner):
    """IntervalCFG(lo, hi) around an already-built guider instance."""
    g = IntervalCFG(lo, hi, {"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 1.0}})
    g.guider = inner
    g.additional_cond_keys = list(inner.additional_cond_keys)
    return g


def action(eng, scale=2.5):
    g = ActionCFG(scale, {"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 1.0}})
    g.image_guider = eng.sampler.guider
    return g


def step_times(eng, den, inputs, n, pairs):
    """Every step of an n-step schedule replayed from one kind of step's graph, timed with events; the loop state is
    filled by a sample whose interval guides half the steps, so both kinds of graph are captured."""
    x, cond, uc, z, mask = inputs
    sig = [float(v) for v in eng.sampler.discretization(n, device="cpu").to(torch.float32)]
    mid = (sig[n // 2 - 1] * sig[n // 2]) ** 0.5
    variants = []
    for inner_name, inner in (("vanilla", eng.sampler.guider), ("action", action(eng))):
        for ms in (False, True):
            smp = sampler(eng, ms, interval(mid, 2 * sig[0], inner), n)
            for guided in (True, False):
                name = f"{inner_name}_{'2m' if ms else 'euler'}_{'guided' if guided else 'cond_only'}"
                variants.append((name, smp, ms, inner_name == "action", guided))
    for _, smp, *_ in variants[::2]:                                # warm-up: captures every graph
        smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask)
    rt = eng.model._rt_get(eng.model.diffusion_model, eng.num_frames, x.device)
    st = rt._loop_states[(x.shape[0], x.shape[2], x.shape[3])]
    out = {v[0]: [] for v in variants}
    for _ in range(pairs):
        for name, smp, ms, act, guided in variants:
            smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask)            # this variant's inputs
            run = st.runner(rt, n, ms, act, guided)
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
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--step-schedule", type=int, default=10, help="steps per timed schedule for the step time")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_interval_cfg", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    act = {"trajectory": TRAJECTORY}
    z = torch.from_numpy(synth.normal(7, "bench_interval_cfg.z", (T, 4, h, w), std=0.9)).to(dev)
    noise = torch.from_numpy(synth.normal(7, "bench_interval_cfg.noise", (T, 4, h, w))).to(dev)
    den = B200Denoiser(eng.denoiser, eng.model)
    torch.cuda.reset_peak_memory_stats(dev)
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

        base = eng.sampler
        rounds, spread, guided_steps = {}, {}, {}
        for ms, n in ((False, 50), (True, 25)):
            label = f"{'2m' if ms else 'euler'}_{n}"
            sig = [float(v) for v in base.discretization(n, device="cpu").to(torch.float32)]
            configs = {"full": base.guider, "interval_0.28_5.42": interval(*PAPER_INTERVAL, base.guider),
                       "empty": interval(4 * sig[0], 8 * sig[0], base.guider)}
            smps = {k: sampler(eng, ms, g, n) for k, g in configs.items()}
            guided_steps[label] = {k: sum(1 for s in sig[:n] if not isinstance(g, IdentityGuider)
                                          and (not isinstance(g, IntervalCFG) or g.guided(s))) for k, g in configs.items()}
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
            spread[label] = {k: float((finals[k] - finals["full"]).norm() / finals["full"].norm())
                             for k in ("interval_0.28_5.42", "empty")}
        eng.sampler = base
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  step_ms_median=steps_ms, guided_steps=guided_steps, session_round_s=rounds,
                  final_latent_rel_l2_vs_full_synthetic_weights=spread, peak_allocated_gib=round(peak / 2 ** 30, 2))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
