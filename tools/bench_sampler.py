"""Euler against DPM-Solver++(2M) on one GPU, at --height x --width (default Vista's 576 x 1024) with the native-YAML
engine of tools/bench_session.py (the vista UNet, seeded synthetic weights), a trajectory action and sample.py's uc_keys.

Reported:
- the card and its power limit / max SM clock;
- the step time of each sampler: every step of an n-step schedule replayed from the loop's CUDA graph and timed with CUDA
  events, the two samplers alternating, as medians;
- the time of the 2M update kernel (and of the Euler one beside it) at the production layout, CUDA events over many
  back-to-back launches;
- the final-latent rel-L2 of Euler and 2M at 10 / 25 / 50 steps against a 200-step 2M solution.  The weights are
  synthetic: this is the ODE-solver error on a random network, not a statement about frames from the real checkpoint;
- the wall time of one session round, from ``step()`` to its uint8 frames on the host, at 25 steps of 2M and at 50 steps
  of Euler, alternating.

    python tools/bench_sampler.py [--pairs 3] [--height 576] [--width 1024] [--out result.json]
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
from vista_b200 import lib, ops, synth  # noqa: E402
from vista_b200.diffusion import B200Denoiser, DPMPP2MSampler, EulerEDMSampler, dpmpp2m_coefficients  # noqa: E402


def samplers(eng):
    """(Euler, 2M) with the engine's discretisation and guider."""
    base = eng.sampler
    dpm = DPMPP2MSampler(discretization_config={"target": "vista_b200.diffusion.EDMDiscretization"},
                         num_steps=base.num_steps, guider_config={"target": "vista_b200.diffusion.IdentityGuider"},
                         device=base.device)
    dpm.discretization, dpm.guider = base.discretization, base.guider
    assert isinstance(base, EulerEDMSampler)
    return base, dpm


def step_times(eng, den, inputs, euler, dpm, n, pairs):
    """Every step of an n-step schedule, replayed from the loop state's graph (one per sampler), timed with events."""
    x, cond, uc, z, mask = inputs
    out = {"euler": [], "2m": []}
    for smp in (euler, dpm):                          # warm-up: captures both graphs
        smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=n)
    rt = eng.model._rt_get(eng.model.diffusion_model, eng.num_frames, x.device)
    st = rt._loop_states[(x.shape[0], x.shape[2], x.shape[3])]
    for _ in range(pairs):
        for name, smp, multistep in (("euler", euler, False), ("2m", dpm, True)):
            smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=n)    # the state holds this schedule
            run = st.runner(rt, n, multistep)
            st.step.zero_()
            for _ in range(n):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                out[name].append(e0.elapsed_time(e1))
    return {k: round(float(np.median(v)), 2) for k, v in out.items()}


def update_kernel_times(T, h, w, dev, launches=1000):
    """Back-to-back launches of each update at (T, 4, h, w), net_out rows of 8; the step index walks a 1000-step table."""
    from vista_b200.diffusion import EDMDiscretization
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(T, 4, h, w, generator=g, device=dev)
    net = torch.randn(2 * T * h * w, 8, generator=g, device=dev)
    sig = EDMDiscretization(0.002, 700.0, 7.0)(launches).to(torch.float32)
    sigmas = torch.zeros(1024, device=dev)
    sigmas[:launches + 1] = sig.to(dev)
    coefs = torch.zeros(1024, 4, device=dev)
    coefs[:launches] = dpmpp2m_coefficients(sig).to(torch.float32).to(dev)
    d_prev, scales, step = torch.empty_like(x), torch.full((T,), 2.5, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    calls = {"euler": lambda: ops.sampler_update(x, net, None, None, scales, sigmas, step, launches, T, h, w),
             "2m": lambda: ops.sampler_update_2m(x, net, None, None, scales, coefs, d_prev, sigmas, step, launches, T, h, w)}
    res = {}
    for name, call in calls.items():
        x0 = x.clone()
        step.zero_()
        call()
        torch.cuda.synchronize()
        step.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            call()
        e1.record()
        e1.synchronize()
        res[name] = round(e0.elapsed_time(e1) * 1000 / launches, 2)      # us per update (kernel + step increment)
        x.copy_(x0)
    return res


def errors(eng, den, inputs, euler, dpm):
    x, cond, uc, z, mask = inputs
    run = lambda smp, n: smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=n).double()
    ref = run(dpm, 200)
    rel = lambda a: float((a - ref).norm() / ref.norm())
    return {name: {n: rel(run(smp, n)) for n in (10, 25, 50)} for name, smp in (("euler", euler), ("2m", dpm))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3, help="Euler / 2M runs alternated this many times")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--step-schedule", type=int, default=20, help="steps per timed schedule for the step time")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_sampler", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    action = {"trajectory": TRAJECTORY}
    z = torch.from_numpy(synth.normal(7, "bench_sampler.z", (T, 4, h, w), std=0.9)).to(dev)
    noise = torch.from_numpy(synth.normal(7, "bench_sampler.noise", (T, 4, h, w))).to(dev)
    euler, dpm = samplers(eng)
    den = B200Denoiser(eng.denoiser, eng.model)
    with torch.no_grad():
        cond, uc = eng.condition({**vd, **action}, T, UC_KEYS)
        mask = torch.zeros(T, device=dev)
        mask[0] = 1.0
        inputs = (noise, cond, uc, z, mask)
        steps_ms = step_times(eng, den, inputs, euler, dpm, args.step_schedule, args.pairs)
        kernel_us = update_kernel_times(T, h, w, dev)
        rel = errors(eng, den, inputs, euler, dpm)

        def session_round(smp, n):
            eng.sampler = smp
            smp.num_steps = n
            sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sess.step(action, noise=noise).cpu()
            return time.perf_counter() - t0

        session_round(dpm, 25)            # warm-up at both schedules (graph capture, decoder buffers)
        session_round(euler, 50)
        rounds = {"2m_25": [], "euler_50": []}
        for _ in range(args.pairs):
            rounds["2m_25"].append(session_round(dpm, 25))
            rounds["euler_50"].append(session_round(euler, 50))
        eng.sampler = euler
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  step_ms_median=steps_ms, update_us_per_launch=kernel_us,
                  final_latent_rel_l2_vs_200_step_2m_synthetic_weights=rel,
                  session_round_s=dict(runs={k: [round(t, 3) for t in v] for k, v in rounds.items()},
                                       median={k: round(float(np.median(v)), 3) for k, v in rounds.items()}))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
