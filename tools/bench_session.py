"""A closed-loop rollout session against the batch rollout, on one GPU: configs/inference/vista_b200_native.yaml with the
vista UNet and decoder, the ViT-H/14 CLIP tower and the vista encoder (seeded synthetic weights), a --height x --width clip,
4 rounds of 50 EDM steps, a trajectory action, sample.py's uc_keys.  Session and batch runs alternate in one job after one
untimed warm-up round, with the same injected noise.

Reported per session run: the time of every round from the ``step()`` call to its uint8 frames on the host, and the
decode time (CUDA events) of every round; per batch run (``engine.rollout(..., recondition=conditioner_recondition(...),
u8=True)``, frames copied to the host): the total and its decode time (the tail decodes between rounds plus the final
decode); for both, how many chunks the decoder ran; and whether the two paths' bytes and latents are equal.

    python tools/bench_session.py [--rounds 4] [--pairs 2] [--height 576] [--width 1024] [--out result.json]

A smaller frame (--height / --width, multiples of 64) runs the same code.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_problem  # noqa: E402
from oracle.make_golden_clip import clip_frames  # noqa: E402
from vista_b200 import lib, spec, synth, vae  # noqa: E402
from vista_b200.diffusion import instantiate_from_config  # noqa: E402
from vista_b200.rollout import conditioner_recondition  # noqa: E402

UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]
TRAJECTORY = torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])


def build_engine(dev):
    """The native-YAML engine at full size with seeded synthetic weights under the reference checkpoint's key names."""
    ucfg, dcfg, _, _, rand_sd = make_problem("full", dev)
    cfg = yaml.safe_load(open(os.path.join(ROOT, "configs", "inference", "vista_b200_native.yaml")))["model"]
    eng = instantiate_from_config(cfg)
    ck = {"model.diffusion_model." + k: v for k, v in rand_sd(spec.unet_param_specs(ucfg)).items()}
    ck.update({"first_stage_model.decoder." + k: v for k, v in rand_sd(spec.decoder_param_specs(dcfg)).items()})
    ck.update({"conditioner.embedders.0.open_clip.model.visual." + k: v
               for k, v in rand_sd(spec.clip_param_specs(spec.clip_preset("vit_h_14"))).items()})
    enc = rand_sd(spec.encoder_param_specs(spec.encoder_preset("vista")))
    ck.update({"conditioner.embedders.3.encoder.encoder." + k: v for k, v in enc.items()})
    ck.update({"first_stage_model.encoder." + k: v for k, v in enc.items()})
    ck["conditioner.embedders.3.encoder.quant_conv.weight"] = torch.eye(8, device=dev).reshape(8, 8, 1, 1)
    ck["conditioner.embedders.3.encoder.quant_conv.bias"] = torch.zeros(8, device=dev)
    missing, unexpected = eng.load_state_dict(ck, strict=False)
    assert not unexpected and not missing, (missing[:3], unexpected[:3])
    return eng.to(dev)


class DecodeTimer:
    """CUDA events around every call of the wrapped methods; ``ms()`` sums them (after a synchronize)."""

    def __init__(self):
        self.pairs = []

    def wrap(self, obj, name):
        fn = getattr(obj, name)

        def timed(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            self.pairs.append((e0, e1))
            return out
        setattr(obj, name, timed)

    def ms(self):
        torch.cuda.synchronize()
        t = sum(e0.elapsed_time(e1) for e0, e1 in self.pairs)
        self.pairs.clear()
        return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--pairs", type=int, default=2, help="session / batch runs alternated this many times")
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    T, H, W = eng.num_frames, args.height, args.width
    h, w = H // 8, W // 8
    frame = torch.from_numpy(clip_frames(12, "bench_session", 1, H, W)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    action = {"trajectory": TRAJECTORY}
    z = torch.from_numpy(synth.normal(7, "bench_session.z", (T, 4, h, w), std=0.9)).to(dev)
    noises = [torch.from_numpy(synth.normal(7, f"bench_session.noise{i}", (T, 4, h, w))).to(dev) for i in range(args.rounds)]

    chunks = [0]
    forward = vae.DecoderRuntime.forward

    def counted(self, *a, **k):
        chunks[0] += 1
        return forward(self, *a, **k)
    vae.DecoderRuntime.forward = counted
    timer = DecodeTimer()
    timer.wrap(eng, "decode_first_stage")
    timer.wrap(eng, "decode_first_stage_u8")

    def session_run(rounds):
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
        timer.wrap(sess, "_decode")
        chunks[0] = 0
        frames, round_s, decode_ms = [], [], []
        t_start = time.perf_counter()
        for r in range(rounds):
            t0 = time.perf_counter()
            frames.append(sess.step(action if r == 0 else None, noise=noises[r]).cpu())
            round_s.append(time.perf_counter() - t0)
            decode_ms.append(timer.ms())
        frames.append(sess.close().cpu())
        total = time.perf_counter() - t_start
        return torch.cat(frames), sess.samples_z.cpu(), dict(total_s=round(total, 3), round_s=[round(t, 3) for t in round_s],
                                                              decode_ms=[round(t, 1) for t in decode_ms], chunks=chunks[0])

    def batch_run(rounds):
        chunks[0] = 0
        t0 = time.perf_counter()
        c, uc = eng.condition({**vd, **action}, T, UC_KEYS)
        frames, samples_z = eng.rollout(c, uc, z, rounds, noises=noises,
                                        recondition=conditioner_recondition(eng, {**vd, **action}, UC_KEYS), u8=True)
        frames = frames.cpu()
        total = time.perf_counter() - t0
        return frames, samples_z.cpu(), dict(total_s=round(total, 3), decode_ms=round(timer.ms(), 1), chunks=chunks[0])

    session_run(1)                      # warm-up: weight packing, CUDA-graph capture, decoder buffers
    timer.ms()
    runs = []
    for _ in range(args.pairs):
        sf, sz, s = session_run(args.rounds)
        bf, bz, b = batch_run(args.rounds)
        s["bytes_equal"], s["latents_equal"] = bool(torch.equal(sf, bf)), bool(torch.equal(sz, bz))
        runs.append(dict(session=s, batch=b))
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    med = lambda v: float(np.median(v))
    result = dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power, frames=[H, W],
                  rounds=args.rounds, steps=eng.sampler.num_steps, runs=runs,
                  peak_allocated_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                  session_total_s_median=med([r["session"]["total_s"] for r in runs]),
                  batch_total_s_median=med([r["batch"]["total_s"] for r in runs]),
                  session_decode_ms_per_round_median=med([t for r in runs for t in r["session"]["decode_ms"]]),
                  all_equal=all(r["session"]["bytes_equal"] and r["session"]["latents_equal"] for r in runs))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
