"""CUDA-event time of ``engine.condition`` on one GPU at do_sample's conditioning inputs: one 576 x 1024 frame repeated over
the 25 rows (get_batch, sample_utils.py:243-244), the ViT-H/14 CLIP tower and the vista VAE encoder of
configs/inference/vista_b200_native.yaml with synthetic weights, a trajectory action and sample.py:243's uc_keys.
In the same run it times the reference's work — the same embedders run directly on all 2 x 25 rows of c and uc — and
reports how many CLIP rows and encoder frames each path computed.

    python tools/bench_conditioner.py [--reps 5] [--height 576] [--width 1024]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden_clip import clip_frames  # noqa: E402
from vista_b200 import lib, spec, synth  # noqa: E402
from vista_b200.diffusion import instantiate_from_config  # noqa: E402

UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]


def build_engine(dev):
    """The native-YAML engine with a tiny UNet / decoder (condition() does not touch them) and the full-size conditioner,
    whose CLIP tower and encoder get seeded synthetic weights under the reference checkpoint's key names."""
    cfg = yaml.safe_load(open(os.path.join(ROOT, "configs", "inference", "vista_b200_native.yaml")))["model"]
    p = cfg["params"]
    u, d = spec.unet_preset("tiny"), spec.decoder_preset("tiny")
    p["network_config"]["params"].update(model_channels=u.model_channels, channel_mult=list(u.channel_mult),
                                         num_res_blocks=u.num_res_blocks, attention_resolutions=list(u.attention_resolutions))
    p["first_stage_config"]["params"]["decoder_config"]["params"].update(ch=d.ch, ch_mult=list(d.ch_mult),
                                                                         num_res_blocks=d.num_res_blocks)
    eng = instantiate_from_config(cfg)
    ck = {f"conditioner.embedders.0.open_clip.model.visual.{k}": torch.from_numpy(v)
          for k, v in synth.synth_state_dict(spec.clip_param_specs(spec.clip_preset("vit_h_14")), seed=12).items()}
    ecfg = spec.encoder_preset("vista")
    ck.update({f"conditioner.embedders.3.encoder.encoder.{k}": torch.from_numpy(v)
               for k, v in synth.synth_state_dict(spec.encoder_param_specs(ecfg), seed=3).items()})
    ck["conditioner.embedders.3.encoder.quant_conv.weight"] = torch.eye(8).reshape(8, 8, 1, 1)
    ck["conditioner.embedders.3.encoder.quant_conv.bias"] = torch.zeros(8)
    missing, unexpected = eng.load_state_dict(ck, strict=False)
    assert not unexpected and not [m for m in missing if m.startswith("_conditioner.")], (missing[:3], unexpected[:3])
    return eng.to(dev)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2], times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=25)
    args = ap.parse_args()
    lib.load()
    dev = torch.device("cuda:0")
    eng = build_engine(dev)
    cond = eng.conditioner
    T = args.frames
    frame = torch.from_numpy(clip_frames(12, "bench_cond", 1, args.height, args.width)).to(dev)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame,
          "trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}

    def native():
        return eng.condition(vd, T, UC_KEYS)

    native_ms, native_all = timed(native, args.reps)
    cond.rows_embedded.clear()
    native()
    torch.cuda.synchronize()
    counts = dict(cond.rows_embedded)

    rows = frame.expand(T, -1, -1, -1).contiguous()

    @torch.no_grad()
    def reference_work():
        n = {"cond_frames_without_noise": 0, "cond_frames": 0}
        for _ in range(2):                          # c, then uc: the reference embeds before zeroing
            cond.embedders[0](rows)
            cond.embedders[3](rows)
            n["cond_frames_without_noise"] += T
            n["cond_frames"] += T
        return n

    ref_ms, ref_all = timed(reference_work, args.reps)
    ref_counts = reference_work()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps(dict(device=torch.cuda.get_device_name(dev), power_limit_and_max_sm_clock=power,
                          frame=[args.height, args.width], rows=T, condition_ms=round(native_ms, 3),
                          condition_ms_all=[round(t, 3) for t in native_all], reference_work_ms=round(ref_ms, 3),
                          reference_work_ms_all=[round(t, 3) for t in ref_all], speedup=round(ref_ms / native_ms, 2),
                          clip_rows_computed=counts.get("cond_frames_without_noise", 0),
                          encoder_frames_computed=counts.get("cond_frames", 0),
                          reference_clip_rows=ref_counts["cond_frames_without_noise"],
                          reference_encoder_frames=ref_counts["cond_frames"])))


if __name__ == "__main__":
    main()
