"""Trajectory conformance at 576 x 1024, T = 25: whole samples of the full-size engine (configs/inference/
vista_b200_native.yaml, seeded synthetic weights) through ``engine.sample``, recorded after every step (tests/trajectory.py).

Per case: the CUDA-graph arm (the product's path) bit-equal to the eager arm at every step; the conditioning frames
exact; the final latent within rel-L2 5e-3 of the fp32 oracle over the clip and 1e-2 per frame (or 4x the fp16-autocast
yardstick's error where that is above 5e-3).  Case A also decodes both final latents.  A session sequence holds graph
replay to the eager launches across schedule lengths and solvers on one loop state, and the planted defects of
tests/trajectory.py are measured against case A's bound.

| case | sampler | guider                                      | cond frames | steps            |
|------|---------|---------------------------------------------|-------------|------------------|
| A    | Euler   | VanillaCFG 2.5 (BASELINE config 2)          | 1           | 50               |
| B    | Euler   | TrianglePredictionGuider 2.5                | 3           | TRAJ_STEPS["B"]  |
| C    | 2M      | ActionCFG s_act 5 over the triangle guider  | 1           | TRAJ_STEPS["C"]  |

The oracle arms run after the engine's packed runtimes are released (they are repacked on the next use): the fp32
oracle at B = 50 does not fit beside them.  TF32 is off for the oracle (cuDNN would default to it)."""
import gc
import os

import pytest
import torch
import yaml

import trajectory as tj
from test_action_cfg_cpu import action_cfg, triangle_cfg, vanilla_cfg, with_guider

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
T, H, W = 25, 576, 1024
UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]
ACTION = {"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}
TRAJ_STEPS = {"A": 50, "B": 15, "C": 15}      # B and C shortened so that the file stays near 10 minutes on one H100
CASES = {"A": ("euler", vanilla_cfg(2.5), 1), "B": ("euler", triangle_cfg(T), 3),
         "C": ("dpm", action_cfg(5.0, triangle_cfg(T)), 1)}


@pytest.fixture(scope="module")
def built():
    """The engine of tools/bench_session.build_engine, composed here so that its UNet and decoder state dicts stay at
    hand for the oracle."""
    from bench import make_problem
    from vista_b200 import lib, spec
    from vista_b200.diffusion import instantiate_from_config
    lib.load()
    ucfg, dcfg, _, _, rand_sd = make_problem("full", DEV)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.safe_load(open(os.path.join(root, "configs", "inference", "vista_b200_native.yaml")))["model"]
    eng = instantiate_from_config(cfg)
    usd = rand_sd(spec.unet_param_specs(ucfg))
    dsd = rand_sd(spec.decoder_param_specs(dcfg))
    ck = {"model.diffusion_model." + k: v for k, v in usd.items()}
    ck.update({"first_stage_model.decoder." + k: v for k, v in dsd.items()})
    ck.update({"conditioner.embedders.0.open_clip.model.visual." + k: v
               for k, v in rand_sd(spec.clip_param_specs(spec.clip_preset("vit_h_14"))).items()})
    enc = rand_sd(spec.encoder_param_specs(spec.encoder_preset("vista")))
    ck.update({"conditioner.embedders.3.encoder.encoder." + k: v for k, v in enc.items()})
    ck.update({"first_stage_model.encoder." + k: v for k, v in enc.items()})
    ck["conditioner.embedders.3.encoder.quant_conv.weight"] = torch.eye(8, device=DEV).reshape(8, 8, 1, 1)
    ck["conditioner.embedders.3.encoder.quant_conv.bias"] = torch.zeros(8, device=DEV)
    missing, unexpected = eng.load_state_dict(ck, strict=False)
    assert not unexpected and not missing, (missing[:3], unexpected[:3])
    del ck, enc
    return eng.to(DEV), ucfg, usd, dcfg, dsd


@pytest.fixture(scope="module")
def inputs(built):
    """(value dict, c, uc, z, noise): c / uc from one engine.condition call, as tests/test_production_conformance_gpu.py
    builds them; every arm gets the same fp32 tensors."""
    from oracle.make_golden_clip import clip_frames
    from vista_b200 import synth
    eng = built[0]
    frame = torch.from_numpy(clip_frames(12, "trajectory_production", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "trajectory_production.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "trajectory_production.noise", (T, 4, H // 8, W // 8))).to(DEV)
    with torch.no_grad():
        c, uc = eng.condition({**vd, **ACTION}, T, UC_KEYS)
    return vd, c, uc, z, noise


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def release(eng):
    """Drops every packed runtime of the engine (and with the UNet's, its loop states and captured graphs)."""
    for m in eng.modules():
        if hasattr(m, "_rt_invalidate"):
            m._rt_invalidate()
        elif "_runtime" in vars(m):
            m._runtime = None
    gc.collect()
    torch.cuda.synchronize(DEV)
    torch.cuda.empty_cache()


def sampler(eng, case):
    kind, guider, _ = CASES[case]
    return with_guider(eng.sampler, kind, guider, TRAJ_STEPS[case])


def problem(inputs, case):
    vd, c, uc, z, noise = inputs
    return tj.Problem(c, uc, z, noise, CASES[case][2])


def our_arms(eng, case, p):
    smp = sampler(eng, case)
    graph = tj.timed(lambda: tj.run_ours(eng, smp, p, graph=True), DEV)
    eager = tj.timed(lambda: tj.run_ours(eng, smp, p, graph=False), DEV)
    tj.assert_graph_equals_eager(f"case {case}", graph, eager)
    print(f"\n[case {case}] graph replay == eager launches at all {len(graph.states)} steps")
    assert torch.equal(graph.out[:p.n_cond], p.z[:p.n_cond].cpu())
    return smp, graph


def reference_arms(built, smp, p):
    eng, ucfg, usd = built[:3]
    release(eng)
    ref = tj.timed(lambda: tj.run_reference(usd, ucfg, smp, p, torch.float32), DEV)
    yard = tj.timed(lambda: tj.run_reference(usd, ucfg, smp, p, torch.float32, autocast=torch.float16), DEV)
    return ref, yard


def test_trajectory_case_a_decode_and_planted_defects(built, inputs):
    """Case A, then its decode: ours with engine.decode_first_stage against the oracle's fp32 decode of the oracle's
    latent, per frame <= 1e-2; decode_first_stage_u8 of our latent equal to the reference's clamp / scale / truncate of
    our own fp32 frames.  Then each planted defect's case-A sample (eager) against the same fp32 trajectory."""
    from oracle import vista_oracle as vo
    from vista_b200 import ops
    eng, ucfg, usd, dcfg, dsd = built
    p = problem(inputs, "A")
    smp, ours = our_arms(eng, "A", p)
    lat = ours.out.to(DEV)
    with torch.no_grad():
        frames = eng.decode_first_stage(lat)
        u8 = eng.decode_first_stage_u8(lat)
    want8 = (255.0 * torch.clamp((frames + 1.0) / 2.0, 0.0, 1.0)).to(torch.uint8).permute(0, 2, 3, 1)
    assert torch.equal(u8, want8)
    frames = frames.cpu()
    del u8, want8
    planted = {}
    for defect in tj.DEFECTS:
        with tj.planted(defect, ops, eng.model):
            planted[defect] = tj.timed(lambda: tj.run_ours(eng, smp, p, graph=False), DEV)

    ref, yard = reference_arms(built, smp, p)
    r = tj.report("case A, 50 steps", p, ours, ref, yard)
    bound = tj.check_final("case A", r, p.n_cond)
    for defect, arm in planted.items():
        e = tj.rel_l2(arm.out, ref.out)
        print(f"[case A, planted {defect}] final latent {e:.3e} = {e / bound:.2f} x the bound "
              f"(fails by {tj.SENSITIVITY}x: {e >= tj.SENSITIVITY * bound}), {tj.rel_l2(arm.out, ours.out):.3e} "
              f"from the clean sample")
        assert not torch.equal(arm.out, ours.out), f"planted {defect}: the defect did not reach the sample"

    del planted
    sdd = {k: v.float() for k, v in dsd.items()}
    torch.cuda.reset_peak_memory_stats(DEV)
    with torch.no_grad(), torch.device(DEV):
        want = vo.decode_first_stage(sdd, dcfg, ref.out.to(DEV), n_samples=14, overlap=3).cpu()
    errs = tj.frame_errors(frames, want)
    print(f"[case A decode] per-frame rel-L2 against the fp32 oracle decode (peak {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.1f}"
          f" GiB): " + " ".join(f"{e:.1e}" for e in errs))
    assert max(errs) <= tj.FRAME_BOUND


@pytest.mark.parametrize("case", ["B", "C"])
def test_trajectory(built, inputs, case):
    p = problem(inputs, case)
    smp, ours = our_arms(built[0], case, p)
    ref, yard = reference_arms(built, smp, p)
    r = tj.report(f"case {case}, {TRAJ_STEPS[case]} steps", p, ours, ref, yard)
    tj.check_final(f"case {case}", r, p.n_cond)


def test_session_sequence_graph_equals_eager(built, inputs):
    """A session step (Euler, 4 steps), a 2M score (2 candidates x 2 members x 3 steps: three, so that the score's steps
    after the first replay a captured graph too), and another step, on one loop state: the graph arm bit for bit the
    eager arm in samples_z, uint8 frames and rewards."""
    from vista_b200 import fused
    eng = built[0]
    vd, c, uc, z, noise = inputs
    other = {"trajectory": torch.tensor([-0.35, 2.41, -1.02, 4.66, -1.93, 6.74, -3.05, 8.62])}
    dpm = with_guider(eng.sampler, "dpm", triangle_cfg(T), 3)

    def run(graph):
        with tj.engine_setting(eng, with_guider(eng.sampler, "euler", triangle_cfg(T), 4), 0, graph), torch.no_grad():
            sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=UC_KEYS)
            f0 = sess.step(ACTION, noise=noise).cpu()
            rewards, members = sess.score([None, other], ensemble_size=2, num_steps=3, seed=1, sampler=dpm)
            f1 = sess.step(None, noise=noise.flip(0)).cpu()
            return f0, rewards.cpu(), members.cpu(), f1, sess.samples_z.cpu()
    assert fused.USE_GRAPH
    g = run(True)
    e = run(False)
    for name, a, b in zip(("round 0 frames", "rewards", "members", "round 1 frames", "samples_z"), g, e):
        assert torch.equal(a, b), f"session sequence: {name} differ between graph replay and eager launches"
    print(f"\n[session] graph == eager: frames, rewards {g[1].tolist()}, members, samples_z")
