"""Action guidance (vista_b200.diffusion.ActionCFG) on one GPU, at --height x --width (default Vista's 576 x 1024) with
the native-YAML engine of tools/bench_session.py (the vista UNet, seeded synthetic weights whose action adapters are
non-zero), a trajectory action and sample.py's uc_keys.

Reported:
- the card and its power limit / max SM clock;
- the step time of Vanilla (the engine's Triangle guider alone) and of ActionCFG over it, for Euler and 2M: every step of
  an n-step schedule replayed from the loop's CUDA graph and timed with CUDA events, the four alternating, as medians;
- the update kernel plus its step increment per back-to-back launch from Python, for each of the four variants;
- the UNet runtime's buffer bytes, summed from the buffers' shapes: the 2T-row set every sample uses, and the T-row set
  the image branch adds;
- the wall time of one session round, from ``step()`` to its uint8 frames on the host, at 25 steps of 2M with ActionCFG;
- the peak allocated memory over the whole run;
- how far the action moves the final latent: the rel-L2 between two actions' final latents (same noise, 25 steps of 2M)
  at s_act = 1, 2.5 and 5, and with the image guider alone.  The weights are synthetic: this shows the knob acts, not
  what it does to frames from the real checkpoint.

    python tools/bench_action_cfg.py [--pairs 3] [--height 576] [--width 1024] [--out result.json]
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


def sampler(eng, multistep, action_scale=None):
    """Euler or 2M with the engine's discretisation, guided by the engine's guider, or by ActionCFG over it."""
    base = eng.sampler
    g = {"target": "vista_b200.diffusion.IdentityGuider"}
    cls = DPMPP2MSampler if multistep else EulerEDMSampler
    s = cls(discretization_config={"target": "vista_b200.diffusion.EDMDiscretization"}, num_steps=base.num_steps,
            guider_config=g, device=base.device)
    s.discretization = base.discretization
    if action_scale is None:
        s.guider = base.guider
    else:
        from vista_b200.diffusion import ActionCFG
        s.guider = ActionCFG(action_scale, g)
        s.guider.image_guider = base.guider
    return s


VARIANTS = (("vanilla_euler", False, None), ("action_euler", False, 2.5), ("vanilla_2m", True, None),
            ("action_2m", True, 2.5))


def step_times(eng, den, inputs, n, pairs):
    """Every step of an n-step schedule, replayed from the loop state's graph (one per variant), timed with events."""
    x, cond, uc, z, mask = inputs
    smps = {name: sampler(eng, ms, a) for name, ms, a in VARIANTS}
    for smp in smps.values():                                   # warm-up: captures every graph
        smp(den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=n)
    rt = eng.model._rt_get(eng.model.diffusion_model, eng.num_frames, x.device)
    st = rt._loop_states[(x.shape[0], x.shape[2], x.shape[3])]
    out = {name: [] for name, _, _ in VARIANTS}
    for _ in range(pairs):
        for name, ms, a in VARIANTS:
            smps[name](den, x.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=n)   # this variant's inputs
            run = st.runner(rt, n, ms, a is not None)
            st.step.zero_()
            for _ in range(n):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                out[name].append(e0.elapsed_time(e1))
    return {k: round(float(np.median(v)), 2) for k, v in out.items()}


def buffer_bytes(rt, keys):
    return sum(t.numel() * t.element_size() for k, t in rt._bufs.items() if k in keys)


def update_kernel_times(T, h, w, dev, launches=1000):
    """Back-to-back launches of each update at (T, 4, h, w), net_out rows of 8, net_img rows of 8; the step index walks
    a 1000-step table."""
    from vista_b200.diffusion import EDMDiscretization
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(T, 4, h, w, generator=g, device=dev)
    net = torch.randn(2 * T * h * w, 8, generator=g, device=dev)
    net_img = torch.randn(T * h * w, 8, generator=g, device=dev)
    sig = EDMDiscretization(0.002, 700.0, 7.0)(launches).to(torch.float32)
    sigmas = torch.zeros(1024, device=dev)
    sigmas[:launches + 1] = sig.to(dev)
    coefs = torch.zeros(1024, 4, device=dev)
    coefs[:launches] = dpmpp2m_coefficients(sig).to(torch.float32).to(dev)
    d_prev, step = torch.empty_like(x), torch.zeros(1, dtype=torch.int32, device=dev)
    scales, a_scales = torch.full((T,), 2.5, device=dev), torch.full((T,), 5.0, device=dev)
    calls = {"vanilla_euler": lambda: ops.sampler_update(x, net, None, None, scales, sigmas, step, launches, T, h, w),
             "action_euler": lambda: ops.sampler_update_action(x, net, net_img, None, None, scales, a_scales, None, None,
                                                               sigmas, step, launches, T, h, w),
             "vanilla_2m": lambda: ops.sampler_update_2m(x, net, None, None, scales, coefs, d_prev, sigmas, step, launches,
                                                         T, h, w),
             "action_2m": lambda: ops.sampler_update_action(x, net, net_img, None, None, scales, a_scales, coefs, d_prev,
                                                            sigmas, step, launches, T, h, w)}
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3, help="the four variants alternated this many times")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--step-schedule", type=int, default=20, help="steps per timed schedule for the step time")
    ap.add_argument("--rounds", type=int, default=3, help="timed session rounds")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_action_cfg", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    actions = [{"trajectory": TRAJECTORY}, {"trajectory": -TRAJECTORY}]
    z = torch.from_numpy(synth.normal(7, "bench_action_cfg.z", (T, 4, h, w), std=0.9)).to(dev)
    noise = torch.from_numpy(synth.normal(7, "bench_action_cfg.noise", (T, 4, h, w))).to(dev)
    den = B200Denoiser(eng.denoiser, eng.model)
    rt = eng.model._rt_get(eng.model.diffusion_model, T, dev)
    torch.cuda.reset_peak_memory_stats(dev)
    with torch.no_grad():
        cond, uc = eng.condition({**vd, **actions[0]}, T, UC_KEYS)
        mask = torch.zeros(T, device=dev)
        mask[0] = 1.0
        inputs = (noise, cond, uc, z, mask)
        sampler(eng, False)(den, noise.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=3)
        keys_2t = set(rt._bufs)
        sampler(eng, False, 2.5)(den, noise.clone(), cond, uc=uc, cond_frame=z, cond_mask=mask, num_steps=3)
        keys_t = set(rt._bufs) - keys_2t
        buffers = {"2T_rows_set": buffer_bytes(rt, keys_2t), "T_rows_set_added": buffer_bytes(rt, keys_t)}
        steps_ms = step_times(eng, den, inputs, args.step_schedule, args.pairs)
        kernel_us = update_kernel_times(T, h, w, dev)

        # how far the action moves the final latent, per s_act (same noise, 25 steps of 2M)
        conds = [eng.condition({**vd, **a}, T, UC_KEYS) for a in actions]
        spread = {}
        for a_s in (None, 1.0, 2.5, 5.0):
            smp = sampler(eng, True, a_s)
            outs = [smp(den, noise.clone(), c, uc=u, cond_frame=z, cond_mask=mask, num_steps=25).double() for c, u in conds]
            spread["image_guider_only" if a_s is None else f"s_act={a_s}"] = float((outs[0] - outs[1]).norm() / outs[1].norm())

        def session_round():
            sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sess.step(actions[0], noise=noise).cpu()
            return time.perf_counter() - t0

        base = eng.sampler
        eng.sampler = sampler(eng, True, 2.5)
        eng.sampler.num_steps = 25
        session_round()                                    # warm-up (graph capture, decoder buffers)
        rounds = [session_round() for _ in range(args.rounds)]
        eng.sampler = base
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  step_ms_median=steps_ms, update_us_per_launch=kernel_us, unet_buffer_bytes=buffers,
                  session_round_s_2m_25_action=dict(runs=[round(t, 3) for t in rounds],
                                                    median=round(float(np.median(rounds)), 3)),
                  peak_allocated_gib=round(peak / 2 ** 30, 2),
                  action_spread_rel_l2_synthetic_weights=spread)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
