"""Golden fixtures of the whole conditioner (tests/golden/cond_vista_tiny.npz, seam_rollout_cond.npz).

Runs the REAL ``vwm.modules.GeneralConditioner`` built from vista.yaml's ``emb_models`` list — its own
``ConcatTimestepEmbedderND`` sinusoids, ``FrozenOpenCLIPImagePredictionEmbedder`` and ``VideoPredictionEmbedderWithEncoder``
over the REAL ``AutoencoderKLModeOnly`` — on the CPU in fp32, at the tiny CLIP preset (open_clip / kornia replaced by the
stand-ins of oracle/make_golden_clip.py) and the tiny encoder preset:

  cond_vista_tiny     c / uc of ``sample_utils.get_condition`` for five value_dicts (free, traj, cmd, steer, goal; inputs
                      as sample.py:228-235 and sample_utils.init_embedder_options build them, uc with sample.py:243's
                      uc_keys) and one re-conditioning call with ``skip_encode`` set (sample_utils.py:342-351).  Every
                      row of a result is the same, so row 0 of each is stored.
  seam_rollout_cond   the UNMODIFIED ``sample_utils.do_sample``, 2 rounds with a trajectory action, on the all-reference
                      DiffusionEngine holding this conditioner, with the seeded sampler noise of tests/seam_fakes.py.

    python -m oracle.make_golden_cond [--only cond_vista_tiny]
"""
from __future__ import annotations

import argparse
import contextlib
import copy
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_golden_clip  # noqa: E402
from vista_b200 import spec, synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
T, H, W = 25, 32, 64                  # rows of a conditioning batch; conditioning frame size (seam clip size)
CLIP_SEED, ENC_SEED = 13, 3
UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]   # sample.py:243
CASES = ("free", "traj", "cmd", "steer", "goal")
ROLLOUT_ROUNDS, ROLLOUT_STEPS = 2, 2


def cond_weights():
    """(clip cfg, clip state dict, encoder cfg, encoder state dict, quant_conv weight, quant_conv bias), numpy."""
    ccfg, csd = make_golden_clip.clip_weights("tiny", CLIP_SEED)
    ecfg = spec.encoder_preset("tiny")
    esd = synth.synth_state_dict(spec.encoder_param_specs(ecfg), seed=ENC_SEED)
    qw = synth.normal(ENC_SEED, "cond.qw", (2 * ecfg.z_channels, 2 * ecfg.z_channels, 1, 1), std=0.35)
    qb = synth.normal(ENC_SEED, "cond.qb", (2 * ecfg.z_channels,), std=0.05)
    return ccfg, csd, ecfg, esd, qw, qb


def conditioner_checkpoint(prefix: str = "conditioner.") -> dict:
    """The conditioner's part of a reference checkpoint: embedder 0's CLIP tower and embedder 3's encoder + quant_conv."""
    _, csd, _, esd, qw, qb = cond_weights()
    ck = {f"{prefix}embedders.0.open_clip.model.visual.{k}": torch.from_numpy(v) for k, v in csd.items()}
    ck.update({f"{prefix}embedders.3.encoder.encoder.{k}": torch.from_numpy(v) for k, v in esd.items()})
    ck[f"{prefix}embedders.3.encoder.quant_conv.weight"] = torch.from_numpy(qw)
    ck[f"{prefix}embedders.3.encoder.quant_conv.bias"] = torch.from_numpy(qb)
    return ck


def tiny_emb_models(emb_models: list, clip_arch=None) -> list:
    """vista.yaml's emb_models list at the tiny encoder preset; ``clip_arch`` replaces the CLIP ``arch`` when given."""
    ecfg = spec.encoder_preset("tiny")
    em = copy.deepcopy(emb_models)
    em[3]["params"]["encoder_config"]["params"]["ddconfig"].update(ch=ecfg.ch, ch_mult=list(ecfg.ch_mult),
                                                                   num_res_blocks=ecfg.num_res_blocks)
    if clip_arch is not None:
        em[0]["params"]["open_clip_embedding_config"]["params"]["arch"] = clip_arch
    return em


def cond_image(tag: str) -> torch.Tensor:
    return torch.from_numpy(make_golden_clip.clip_frames(CLIP_SEED, f"cond.{tag}", 1, H, W))


def value_dict(case: str) -> dict:
    """sample.py:228-235: init_embedder_options (fps 10 / fps_id 9, motion_bucket_id 127), the clean conditioning frame, a
    noise-augmented copy for cond_frames, and the action of ``case`` (sample.py:146-166 for its tensor types)."""
    img = cond_image("frame")
    cond_aug = 0.02
    vd = {"fps": 10, "fps_id": 9, "motion_bucket_id": 127, "cond_frames_without_noise": img, "cond_aug": cond_aug,
          "cond_frames": img + cond_aug * torch.from_numpy(synth.normal(CLIP_SEED, "cond.aug", (1, 3, H, W), std=1.0))}
    if case == "traj":
        vd["trajectory"] = torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])
    elif case == "cmd":
        vd["command"] = torch.tensor(2)
    elif case == "steer":
        vd["speed"] = torch.tensor([5.41, 5.62, 5.80, 6.03])
        vd["angle"] = torch.tensor([-12.0, -8.5, -3.25, 1.5]) / 780
    elif case == "goal":
        vd["goal"] = torch.tensor([1012 / 1600, 507 / 900])
    elif case != "free":
        raise KeyError(case)
    return vd


def recondition_value_dict() -> dict:
    """The value_dict of a re-conditioning call (sample_utils.py:342-343): a decoded frame and a latent / scale_factor."""
    vd = value_dict("traj")
    vd["cond_frames_without_noise"] = cond_image("decoded")
    vd["cond_frames"] = torch.from_numpy(synth.normal(CLIP_SEED, "cond.latent", (1, 4, H // 2, W // 2), std=1.0)) / 0.18215
    return vd


_REF = []


def _reference():
    """(sample_utils, GeneralConditioner class, seam_fakes) with the CLIP stand-ins installed before anything imports vwm
    (once per process: a second install would re-import the embedder classes under the conditioner's feet)."""
    if not _REF:
        ccfg, csd, *_ = cond_weights()
        make_golden_clip.install_stand_ins(ccfg, csd)
        from oracle import make_golden
        sf, su, _, _ = make_golden._seam_setup()
        # get_condition calls get_batch without a device, whose default is "cuda" (sample_utils.py:232,257-261)
        get_batch = su.get_batch
        su.get_batch = lambda keys, value_dict, N, device="cpu": get_batch(keys, value_dict, N, device="cpu")
        from vwm.modules import GeneralConditioner
        _REF.extend([su, GeneralConditioner, sf])
    return tuple(_REF)


def _load_encoder(conditioner):
    _, _, _, esd, qw, qb = cond_weights()
    missing, unexpected = conditioner.embedders[3].encoder.load_state_dict(
        {**{"encoder." + k: torch.from_numpy(v) for k, v in esd.items()}, "quant_conv.weight": torch.from_numpy(qw),
         "quant_conv.bias": torch.from_numpy(qb)}, strict=False)
    assert not unexpected and all(k.startswith(("decoder.", "post_quant_conv.")) for k in missing), (missing, unexpected)


def _condition(su, conditioner, vd, force_uc):
    model = type("M", (), {"conditioner": conditioner})()
    return su.get_condition(model, vd, T, force_uc, "cpu")


def make_cond():
    from oracle import ref_loader
    su, GeneralConditioner, _ = _reference()
    em = tiny_emb_models(ref_loader.vista_yaml()["model"]["params"]["conditioner_config"]["params"]["emb_models"])
    em[0]["params"]["open_clip_embedding_config"]["params"]["device"] = "cpu"
    with contextlib.redirect_stdout(io.StringIO()):
        cond = GeneralConditioner(em).eval()
    _load_encoder(cond)
    out = {"rows": np.int64(T), "uc_keys": np.array(UC_KEYS)}
    runs = [(case, value_dict(case), False) for case in CASES] + [("recond", recondition_value_dict(), True)]
    with torch.no_grad():
        for case, vd, skip in runs:
            for e in cond.embedders:
                if hasattr(e, "skip_encode"):
                    e.skip_encode = skip
            c, uc = _condition(su, cond, vd, UC_KEYS)
            for tag, d in (("c", c), ("uc", uc)):
                for k, v in d.items():
                    assert v.shape[0] == T and torch.equal(v, v[:1].expand_as(v)), (case, tag, k)
                    out[f"{case}_{tag}_{k}"] = v[:1].float().numpy()
            print(f"cond_vista_tiny/{case}: " + ", ".join(f"{k} {tuple(v.shape)}" for k, v in c.items()))
    path = os.path.join(GOLDEN, "cond_vista_tiny.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


def make_seam_rollout():
    """sample_utils.do_sample, 2 rounds x 2 steps (TrianglePredictionGuider), trajectory action, on the all-reference engine
    whose conditioner is the real one: the clip it encoded and strided samples / block means of the latents and frames."""
    from oracle import make_golden, ref_loader
    su, _, sf = _reference()
    from vwm.models.diffusion import DiffusionEngine
    ucfg, dcfg, ecfg = cfgs = sf.presets()
    p = copy.deepcopy(ref_loader.vista_yaml()["model"]["params"])
    p["network_config"]["params"].update(model_channels=ucfg.model_channels, num_res_blocks=ucfg.num_res_blocks,
                                         attention_resolutions=list(ucfg.attention_resolutions),
                                         channel_mult=list(ucfg.channel_mult))
    cp = p["conditioner_config"]["params"]
    cp["emb_models"] = tiny_emb_models(cp["emb_models"])
    cp["emb_models"][0]["params"]["open_clip_embedding_config"]["params"]["device"] = "cpu"
    f = p["first_stage_config"]["params"]
    f["encoder_config"]["params"].update(ch=ecfg.ch, ch_mult=list(ecfg.ch_mult), num_res_blocks=ecfg.num_res_blocks)
    f["decoder_config"]["params"].update(ch=dcfg.ch, ch_mult=list(dcfg.ch_mult), num_res_blocks=dcfg.num_res_blocks)
    with contextlib.redirect_stdout(io.StringIO()):
        eng = DiffusionEngine(**p).eval()
    missing, unexpected = eng.load_state_dict(sf.checkpoint(cfgs), strict=False)
    assert not unexpected and all(m.startswith("conditioner.") for m in missing), (missing[:3], unexpected[:3])
    _load_encoder(eng.conditioner)
    images, _ = sf.clip_inputs()
    vd = rollout_value_dict(sf)
    zs, real_encode = [], eng.encode_first_stage
    eng.encode_first_stage = lambda x: (zs.append(real_encode(x)), zs[-1])[1]
    sampler = su.init_sampling(guider="TrianglePredictionGuider", steps=ROLLOUT_STEPS, cfg_scale=2.5, num_frames=T)
    sampler.device = "cpu"
    torch.manual_seed(1234)
    with make_golden._seeded_sampler_noise(sf, "rollout_cond") as count, torch.no_grad(), \
            contextlib.redirect_stderr(io.StringIO()):
        x, z_all, _ = su.do_sample(images, eng, sampler, dict(vd), num_rounds=ROLLOUT_ROUNDS, num_frames=T,
                                   force_uc_zero_embeddings=UC_KEYS, initial_cond_indices=[0], device="cpu")
    assert count[0] == ROLLOUT_ROUNDS and len(zs) == 1
    print(f"seam_rollout_cond: latents {tuple(z_all.shape)} frames {tuple(x.shape)}")
    path = os.path.join(GOLDEN, "seam_rollout_cond.npz")
    np.savez_compressed(path, z=zs[0].numpy(), rounds=ROLLOUT_ROUNDS, steps=ROLLOUT_STEPS,
                        **make_golden.sampled(z_all, 2, 4, "lat_"), **make_golden.sampled(x, 4, 8, "frames_"))
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


def rollout_value_dict(sf) -> dict:
    """The seam clip's conditioning frames (tests/seam_fakes.clip_inputs) with the trajectory case's other inputs."""
    _, frames = sf.clip_inputs()
    vd = value_dict("traj")
    vd.update(frames)
    return vd


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, choices=["cond_vista_tiny", "seam_rollout_cond"])
    args = ap.parse_args()
    torch.set_num_threads(os.cpu_count() or 1)
    if args.only in (None, "cond_vista_tiny"):
        make_cond()
    if args.only in (None, "seam_rollout_cond"):
        make_seam_rollout()
