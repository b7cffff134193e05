"""Production-shape conformance: the full-size engine (configs/inference/vista_b200_native.yaml, seeded synthetic
weights) run eagerly at 576 x 1024, T = 25, under the shadow harness of tests/shadow.py, so that every distinct launch
configuration of the single-GPU path is held to fp64 on the inputs it really received: the sampler step under each
guider and solver, the uint8 decode of a 25-frame clip, the conditioner (CLIP ViT-H/14, the embedders, the VAE
encoder) and the rollout session's glue.  Each test also runs under torch.profiler: every vb:: kernel it launches must
belong to an entry point with at least one checked configuration.

Each test prints the census (keys per op, worst error / bound per op), its wall time and its peak memory."""
import re
import time

import pytest
import torch

from shadow import Shadow, gemm_field

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
T, H, W = 25, 576, 1024
UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]
ACTION = {"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}

# the kernels behind each entry point (the profiler's vb:: names)
OP_KERNELS = {
    "gemm": {"tapgemm_kernel"}, "groupnorm": {"gn_stats_kernel", "gn_apply_kernel"},
    "groupnorm_from_partials": {"gn_from_partials_kernel"}, "groupnorm_apply": {"gn_apply_kernel"},
    "layernorm": {"layernorm_kernel", "layernorm40_kernel"}, "attention_spatial": {"attn_spatial_kernel"},
    "attention_temporal": {"attn_temporal_kernel"}, "attention_d80": {"attn_d80_kernel"},
    "softmax_rows": {"softmax_rows_kernel"}, "conv3x3_small_cin": {"conv3x3_small_cin_kernel"},
    "im2col_s2": {"im2col_s2_kernel"}, "im2col_s2_asym": {"im2col_s2_asym_kernel"}, "upsample2x": {"upsample2x_kernel"},
    "nchw_to_tokens": {"nchw_to_tokens_kernel"}, "tokens_to_nchw": {"tokens_to_nchw_kernel"},
    "time_mix_small": {"time_mix_small_kernel"}, "time_mix_small_u8": {"time_mix_small_u8_kernel"},
    "sampler_prepare": {"sampler_prepare_kernel"}, "sampler_update": {"sampler_update_kernel"},
    "sampler_update_2m": {"sampler_update_kernel"}, "sampler_update_action": {"sampler_update_kernel"},
    "rollout_advance": {"rollout_advance_kernel"}, "ensemble_reward": {"ensemble_reward_kernel"},
    "timestep_embedding": {"timestep_embedding_kernel"}, "blend_emb": {"blend_emb_kernel"},
    "sinusoid_embed": {"sinusoid_embed_kernel"}, "clip_preprocess": {"clip_preprocess_kernel"},
}


@pytest.fixture(scope="module")
def eng():
    from tools.bench_session import build_engine
    from vista_b200 import lib
    lib.load()
    return build_engine(DEV)


@pytest.fixture(scope="module")
def problem(eng):
    from oracle.make_golden_clip import clip_frames
    from vista_b200 import synth
    frame = torch.from_numpy(clip_frames(12, "production_conformance", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "production_conformance.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "production_conformance.noise", (T, 4, H // 8, W // 8))).to(DEV)
    with torch.no_grad():
        c, uc = eng.condition({**vd, **ACTION}, T, UC_KEYS)
    return vd, z, noise, c, uc


@pytest.fixture(autouse=True)
def eager(monkeypatch):
    from vista_b200 import fused
    monkeypatch.setattr(fused, "USE_GRAPH", False)


def shadow_run(name, fn, random_rows=2048):
    """fn() under the shadow harness and torch.profiler; prints the census, wall time and peak memory, then holds every
    key and the coverage of every launched vb:: kernel."""
    from torch.profiler import ProfilerActivity, profile
    from test_conformance_small_cpu import LAUNCHED_NOT_HELD
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    with profile(activities=[ProfilerActivity.CUDA]) as prof, torch.no_grad(), Shadow(random_rows=random_rows) as sh:
        fn()
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(DEV) / 2 ** 30
    launched = set()
    for e in prof.events():
        m = re.search(r"\bvb::(\w+)", e.name)
        if m:
            launched.add(m.group(1))
    print(f"\n[{name}] {torch.cuda.get_device_name(DEV)}: wall {wall:.1f} s, peak allocated {peak:.2f} GiB")
    print(sh.report())
    sh.assert_ok()
    held = set().union(*(OP_KERNELS[op] for op in sh.checked_ops()))
    unheld = launched - held - LAUNCHED_NOT_HELD
    assert not unheld, f"{name}: kernels launched without a checked configuration: {sorted(unheld)}"
    return sh


def sampler(eng, kind, steps):
    from test_action_cfg_cpu import action_cfg, triangle_cfg, vanilla_cfg, with_guider
    guider = {"euler_vanilla": vanilla_cfg(), "euler_triangle": triangle_cfg(T), "dpm2m": vanilla_cfg(),
              "action": action_cfg(5.0, triangle_cfg(T))}[kind]
    return with_guider(eng.sampler, "dpm" if kind == "dpm2m" else "euler", guider, steps)


@pytest.mark.parametrize("kind", ["euler_vanilla", "euler_triangle", "dpm2m", "action"])
def test_sampler_step_production(eng, problem, kind, monkeypatch):
    """Sampler steps at 576 x 1024, T = 25 through the full-size UNet: Euler under VanillaCFG and the triangle guider, 2M
    over 3 steps (step 1 is a second-order row that reads D_prev), and action guidance (the extra T-row forward has
    its own GEMM and attention keys).  Every key passes."""
    vd, z, noise, c, uc = problem
    monkeypatch.setattr(eng, "sampler", sampler(eng, kind, 3 if kind == "dpm2m" else 1))
    sh = shadow_run(f"sampler {kind}", lambda: eng.sample(c, uc=uc, N=T, shape=tuple(z.shape[1:]), noise=noise.clone(),
                                                         cond_frame=z))
    fams = sh.families()
    upd = {"euler_vanilla": "sampler_update", "euler_triangle": "sampler_update", "dpm2m": "sampler_update_2m",
           "action": "sampler_update_action"}[kind]
    assert {"gemm", "attention_spatial", "attention_temporal", "layernorm", "sampler_prepare", upd} <= set(fams)
    if kind == "dpm2m":
        assert fams[upd][0] >= 2, "the first- and second-order rows of the 2M update"


def test_decode_production(eng, problem):
    """decode_first_stage_u8 of a 25-frame latent clip: two 14-frame chunks with the 3-frame overlap.  The upsampling
    tap-GEMM with fused statistics at all three transitions, GroupNorm up to 14 x 589824 tokens, the mid-attention's
    softmax_rows, the time mix's blend and skip at full resolution."""
    vd, z, noise, c, uc = problem
    lat = noise * 0.9
    sh = shadow_run("decode", lambda: eng.decode_first_stage_u8(lat))
    ups = [k for k in sh.census if k[0] == "gemm" and gemm_field(k, "a_mode") == 2]
    assert len({gemm_field(k, "geom") for k in ups}) >= 3, "the upsampling GEMM at every transition"
    assert {"softmax_rows", "time_mix_small_u8", "groupnorm_apply", "groupnorm_from_partials"} <= set(sh.families())


def test_condition_and_encode_production(eng, problem):
    """engine.condition on 576 x 1024 frames with a trajectory: the ViT-H/14 tower (clip_preprocess with antialiasing,
    the erf-GELU GEMM, attn_d80 at 257 tokens x 16 heads, LayerNorms), the sinusoid embedders, the VAE encoder
    (conv3x3_small_cin, im2col_s2_asym, GroupNorm)."""
    vd = problem[0]
    sh = shadow_run("condition", lambda: eng.condition({**vd, **ACTION}, T, UC_KEYS))
    assert {"clip_preprocess", "attention_d80", "layernorm", "sinusoid_embed", "conv3x3_small_cin", "im2col_s2_asym",
            "groupnorm"} <= set(sh.families())


def test_session_production(eng, problem, monkeypatch):
    """One RolloutSession.step at one sampler step and one score with ensemble_size 2: rollout_advance and
    ensemble_reward at the production element count."""
    vd, z, noise, c, uc = problem
    monkeypatch.setattr(eng, "sampler", sampler(eng, "euler_triangle", 1))

    def run():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
        sess.step(ACTION, noise=noise.clone())
        sess.score([None], ensemble_size=2, num_steps=1)
    sh = shadow_run("session", run)
    assert {"rollout_advance", "ensemble_reward"} <= set(sh.families())
