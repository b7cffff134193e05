"""Camera frames in: sample.py's host path against ``engine.frames_from_u8`` and ``engine.rollout_session_from_frames``,
on one GPU.  Three comparisons, each after a warm-up, as the median of --runs (--session-runs) runs:

1. host path: 25 seeded 1600 x 900 uint8 frames through load_img's body (crop, PIL LANCZOS, ToTensor, * 2 - 1),
   stacked, and the pinned H2D copy of the fp32 result — host clock, ending in a synchronize;
2. device path: the same frames' pinned uint8 H2D copy plus the kernel (CUDA events), and the kernel alone, with the
   bytes it moves over its time against the H100 SXM's 3.35 TB/s of HBM3;
3. session start, each arm in a process of its own: ``rollout_session_from_frames`` until its first ``step()`` has
   returned (frames on the device, synchronized), against the session sample.py's recipe builds by hand: host load_img of the 25 frames, H2D,
   ``encode_first_stage`` of all 25, the value dict and ``rollout_session``, timed to a ready session (its first
   ``step()`` is the same work as the other arm's, so its time to the first frames adds that arm's step).  The engine is
   tools/bench_session.py's (native YAML, seeded synthetic weights) at 576 x 1024.

    python tools/bench_ingest.py [--runs 5] [--session-runs 2] [--out result.json]

Prints one JSON line; --out also writes it.
"""
import argparse
import hashlib
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image
from torchvision import transforms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vista_b200 import ingest, lib  # noqa: E402

HBM_TBS = 3.35          # NVIDIA H100 SXM data sheet, HBM3
T, SRC_H, SRC_W, H, W = 25, 900, 1600, 576, 1024


def load_img_body(rgb: np.ndarray, target_height: int, target_width: int) -> torch.Tensor:
    """sample.py:174-201 (load_img) after the file is decoded to RGB."""
    image = Image.fromarray(rgb)
    ori_w, ori_h = image.size
    if ori_w / ori_h > target_width / target_height:
        tmp_w = int(target_width / target_height * ori_h)
        image = image.crop(((ori_w - tmp_w) // 2, 0, (ori_w + tmp_w) // 2, ori_h))
    elif ori_w / ori_h < target_width / target_height:
        tmp_h = int(target_height / target_width * ori_w)
        image = image.crop((0, (ori_h - tmp_h) // 2, ori_w, (ori_h + tmp_h) // 2))
    image = image.resize((target_width, target_height), resample=Image.LANCZOS)
    return transforms.Compose([transforms.ToTensor(), transforms.Lambda(lambda x: x * 2.0 - 1.0)])(image)


def host_path(rgb, dev, pinned_out):
    torch.stack([load_img_body(f, H, W) for f in rgb], out=pinned_out)
    out = pinned_out.to(dev, non_blocking=True)
    torch.cuda.synchronize()
    return out


def frames():
    """The 25 seeded 1600 x 900 frames."""
    return np.random.default_rng(2026).integers(0, 256, size=(T, SRC_H, SRC_W, 3), dtype=np.uint8)


def kernel_bytes(n_frames):
    """Bytes the two passes move: the crop read, the intermediate rows written and read, the fp32 output written."""
    left, top, right, bottom = ingest.crop_box(SRC_W, SRC_H, W, H)
    rows = bottom - top
    if rows != H:
        b = ingest.lanczos_tables(rows, H).bounds
        rows = int(b[-1, 0] + b[-1, 1] - b[0, 0])
    mid = n_frames * rows * W * 3 if right - left != W else 0
    return n_frames * (bottom - top) * (right - left) * 3 + 2 * mid + n_frames * 3 * H * W * 4


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="timed runs of comparisons 1 and 2")
    ap.add_argument("--session-runs", type=int, default=2, help="timed pairs of comparison 3 (0 skips it)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--session-arm", choices=["from_frames", "hand_built"], default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    lib.load()
    if args.session_arm:
        return session_arm(args.session_arm, args.session_runs)
    dev = torch.device("cuda:0")
    med = lambda v: float(np.median(v))
    rgb = frames()
    result = dict(device=torch.cuda.get_device_name(dev), host_cores=os.cpu_count(), frames=[T, SRC_H, SRC_W], out=[H, W])
    try:
        result["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        result["power_limit_and_max_sm_clock"] = "unknown"

    # 1. host path
    pinned_out = torch.empty(T, 3, H, W, dtype=torch.float32).pin_memory()
    want = host_path(rgb, dev, pinned_out).clone()
    host_s = []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        host_path(rgb, dev, pinned_out)
        host_s.append(time.perf_counter() - t0)
    result["host_path_ms"] = round(med(host_s) * 1e3, 1)

    # 2. device path
    pinned_u8 = torch.from_numpy(rgb).pin_memory()
    frames_dev = pinned_u8.to(dev)
    got = ingest.frames_u8_resize(frames_dev, H, W)
    result["device_equals_host"] = bool(torch.equal(got, want))
    h2d_kernel = [events_ms(lambda: ingest.frames_u8_resize(pinned_u8.to(dev, non_blocking=True), H, W), 5)
                  for _ in range(args.runs)]
    kernel = [events_ms(lambda: ingest.frames_u8_resize(frames_dev, H, W), 20) for _ in range(args.runs)]
    nbytes = kernel_bytes(T)
    result.update(device_h2d_plus_kernel_ms=round(med(h2d_kernel), 3), kernel_ms=round(med(kernel), 3),
                  kernel_bytes=nbytes, kernel_gbs=round(nbytes / (med(kernel) * 1e-3) / 1e9, 1),
                  kernel_share_of_hbm=round(nbytes / (med(kernel) * 1e-3) / (HBM_TBS * 1e12), 3),
                  host_over_device=round(result["host_path_ms"] / med(h2d_kernel), 1))

    # 3. session start: one process per arm.  On one 80 GB H100 the hand-built arm's 25-frame encode (its encoder
    # buffers for a 14-frame chunk at 576 x 1024) does not fit beside a session that has stepped (sampler graph, decoder
    # arena), so the two arms do not share a process, and that arm releases those buffers after each encode.
    if args.session_runs > 0:
        arms = {}
        for arm in ("from_frames", "hand_built"):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--session-arm", arm, "--session-runs",
                                str(args.session_runs)], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"session arm {arm} failed:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
            arms[arm] = json.loads(r.stdout.strip().splitlines()[-1])
        ff, hb = arms["from_frames"], arms["hand_built"]
        step_s = ff["first_step_s_median"] - ff["ready_s_median"]
        result.update(session=arms, first_step_frames_equal=ff["sha256"] == hb["sha256"], step_s=round(step_s, 3),
                      from_frames_ready_s=ff["ready_s_median"], hand_built_ready_s=hb["ready_s_median"],
                      from_frames_first_step_s=ff["first_step_s_median"],
                      hand_built_first_step_s_estimate=round(hb["ready_s_median"] + step_s, 3))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


def session_arm(arm: str, runs: int):
    """One arm of comparison 3 in this process: a warm-up (weight packing, graph capture, decoder buffers), then ``runs``
    timed session starts -> JSON line with the median seconds to a ready session and to the first step's frames."""
    dev = torch.device("cuda:0")
    spec_ = importlib.util.spec_from_file_location("bench_session", os.path.join(ROOT, "tools", "bench_session.py"))
    bs = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(bs)
    eng = bs.build_engine(dev)
    rgb = frames()
    action = {"trajectory": bs.TRAJECTORY}
    g = torch.Generator().manual_seed(3)
    cond_aug_noise = torch.randn(1, 3, H, W, generator=g).to(dev)
    encode_noise = torch.randn(T, 4, H // 8, W // 8, generator=g).to(dev)
    noise = torch.randn(T, 4, H // 8, W // 8, generator=g).to(dev)
    pinned_out = torch.empty(T, 3, H, W, dtype=torch.float32).pin_memory()

    def start():
        if arm == "from_frames":
            return eng.rollout_session_from_frames(torch.from_numpy(rgb), n_conds=1, cond_aug=0.02, action=action,
                                                   force_uc_zero_embeddings=bs.UC_KEYS, cond_aug_noise=cond_aug_noise,
                                                   encode_noise=encode_noise)
        images = host_path(rgb, dev, pinned_out)          # sample.py:222-253 and the head of do_sample, by hand
        vd = ingest.embedder_options({e.input_key for e in eng.conditioner.embedders})
        cond_img = images[0][None]
        vd.update(cond_frames_without_noise=cond_img, cond_aug=0.02, cond_frames=cond_img + 0.02 * cond_aug_noise, **action)
        z = eng.encode_first_stage(images, noise=encode_noise)
        # do_sample unloads the first stage after the encode (sample_utils.py:306-308); here the encoder's activation
        # buffers for a 14-frame chunk are released, or the session's step does not fit beside them on 80 GB
        eng.first_stage_model.encoder.runtime(dev)._bufs.clear()
        torch.cuda.empty_cache()
        return eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS, initial_cond_indices=[0])

    def run():
        t0 = time.perf_counter()
        sess = start()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        x = sess.step(None, noise=noise)
        torch.cuda.synchronize()
        return t1 - t0, time.perf_counter() - t0, x

    ready, first = [], []
    if arm == "from_frames":
        _, _, x = run()
        for _ in range(runs):
            a, b, x = run()
            ready.append(a)
            first.append(b)
    else:
        # after a session has stepped, the next 25-frame encode no longer fits on 80 GB (its sampler graph and decoder
        # arena stay resident): this arm times the session start alone, then steps once for the frames' checksum
        for i in range(runs + 1):
            t0 = time.perf_counter()
            sess = start()
            torch.cuda.synchronize()
            if i:
                ready.append(time.perf_counter() - t0)
        x = sess.step(None, noise=noise)
        torch.cuda.synchronize()
    print(json.dumps(dict(arm=arm, steps=eng.sampler.num_steps, ready_s=[round(v, 3) for v in ready],
                          first_step_s=[round(v, 3) for v in first], ready_s_median=round(float(np.median(ready)), 3),
                          first_step_s_median=round(float(np.median(first)), 3) if first else None,
                          sha256=hashlib.sha256(x.cpu().numpy().tobytes()).hexdigest(),
                          peak_allocated_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))))


if __name__ == "__main__":
    main()
