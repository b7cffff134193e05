"""The DPM-Solver++(2M) sampler on the H100: the sampler_update_kernel<true> instantiation against the fp64 reference of
tests/test_dpmpp2m_cpu.py (production layout, NULL mask / cond_frame, first, second, middle and final steps, NaN D_prev
on first-order rows, a 50-step trajectory, CUDA-graph replay), the order of convergence of the fused loop on the
closed-form denoiser, the tiny-preset fused 2M sample against the oracle restatement, and a 576 x 1024 2M session step
and score that repeat bit for bit."""
import pytest
import torch

import test_dpmpp2m_cpu as tdc
from test_conformance_small_cpu import NUM_STEPS, SAMPLER_CASES, sampler_case_id, trajectory_inputs
from test_fullres_gpu import _bench_session
from helpers import rel_l2, to_t
from vista_b200 import synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as _ops
    lib.load()
    return _ops


@pytest.mark.parametrize("step", [0, 1, 24, NUM_STEPS - 1])
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=sampler_case_id)
def test_update_2m(ops, case, step):
    """Every layout of the Euler conformance table, 25 x 4 x 72 x 128 with ld_net 8 among them, and the NULL mask /
    cond_frame variants; the twin runs the same case on the CPU."""
    tdc.check_update_2m(case, step, ops.sampler_update_2m, DEV)
    if case[1] * case[2] <= 128:
        import dpm_fake_ops
        tdc.check_update_2m(case, step, dpm_fake_ops.sampler_update_2m, torch.device("cpu"))


def test_trajectory_2m_and_graph_replay(ops):
    """50 prepare -> 2M update steps at 25 x 72 x 128 against the fp64 trajectory, then the same steps replayed from one
    captured CUDA graph: bit-equal to the eager launches."""
    d = trajectory_inputs(25, 72, 128, DEV)
    coefs = tdc.coef_table(DEV)
    x, idx = tdc.run_trajectory_2m(d, ops.sampler_prepare, ops.sampler_update_2m, coefs, NUM_STEPS)
    torch.cuda.synchronize()
    ref = tdc.trajectory_2m_reference(d, coefs, NUM_STEPS)
    rel = rel_l2(x, ref)
    print(f"2M 50-step trajectory rel-L2 {rel:.3e}")
    assert int(idx[0]) == NUM_STEPS and rel <= tdc.TRAJ_REL
    T, h, w = d["T"], d["h"], d["w"]
    xg = d["x"].clone()
    d_prev = torch.full_like(xg, float("nan"))
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.sampler_prepare(xg, d["cond_frame"], d["mask"], d["concat_u"], d["concat_c"], d["sigmas"], step, d["unet_in"],
                            d["c_noise"], T, h, w)
        ops.sampler_update_2m(xg, d["net"], d["cond_frame"], d["mask"], d["scales"], coefs, d_prev, d["sigmas"], step,
                              NUM_STEPS, T, h, w)
    assert int(step[0]) == 0, "capture must not run the kernels"
    for _ in range(NUM_STEPS):
        g.replay()
    torch.cuda.synchronize()
    assert int(step[0]) == NUM_STEPS
    assert torch.equal(xg, x), "graph replay differs from the eager launches"


def test_update_2m_rejects_misaligned_coefs(ops):
    d = trajectory_inputs(1, 2, 2, DEV)
    coefs = tdc.coef_table(DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="aligned"):
        ops.sampler_update_2m(d["x"], d["net"], None, None, d["scales"], coefs.flatten()[1:], d["x"].clone(), d["sigmas"],
                              step, NUM_STEPS, 1, 2, 2)


def test_order_of_convergence_fused_loop_on_device(ops):
    """The closed-form denoiser through the fused loop on the kernels, steps replayed from CUDA graphs."""
    an = tdc.Analytic(3, 4, 6, DEV)
    tdc.check_order(tdc.fused_errors("euler", an), tdc.fused_errors("dpm", an), "fused loop (H100)")


def test_tiny_fused_2m_against_oracle_and_interleaved(ops):
    """The fused 2M sample on the tiny UNet within the Euler bar (rel-L2 <= 5e-3) of the oracle restatement; two seeded
    runs are bit-identical; Euler and 2M at the same num_steps, interleaved on one loop state (one captured graph each),
    equal their first runs."""
    from dpm_oracle import dpmpp2m_sample
    cfg, sd, net, den, bden = tdc.tiny_network("cuda")
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, DEV)
    dpm, euler = tdc.make_sampler("dpm", 4, "cuda"), tdc.make_sampler("euler", 4, "cuda")
    run = lambda smp: smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    with torch.no_grad():
        first = run(dpm)
        cpu = lambda dd: {k: v.cpu() for k, v in dd.items()}
        ref = dpmpp2m_sample(to_t(sd), cfg, noise.cpu(), cpu(c), cpu(uc), z.cpu(), mask.cpu(), 4, 25)
        e1, d2, e2, d3 = run(euler), run(dpm), run(euler), run(dpm)
    torch.cuda.synchronize()
    r = rel_l2(first.cpu(), ref)
    print(f"tiny fused 2M, 4 steps: rel-L2 {r:.3e} from the oracle")
    assert r <= 5e-3 and torch.equal(first[:1], z[:1])
    assert torch.equal(first, d2) and torch.equal(first, d3) and torch.equal(e1, e2) and not torch.equal(e1, first)
    st = next(iter(net._rt_get(net.diffusion_model, 25, DEV)._loop_states.values()))
    assert set(st.graphs) == {(4, False), (4, True)}


def test_session_step_and_score_at_576x1024_repeat():
    """The native YAML engine at Vista's resolution with a 2M engine.sampler: a 3-step session round, then a 3-step 2M
    score of two members; both repeat bit for bit."""
    from oracle.make_golden_clip import clip_frames
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    eng.sampler = tdc.as_dpm(eng.sampler, steps=3)
    T, H, W = eng.num_frames, 576, 1024
    frame = torch.from_numpy(clip_frames(12, "dpm_fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "dpm_fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "dpm_fullres.noise", (T, 4, H // 8, W // 8))).to(DEV)
    action = {"trajectory": bs.TRAJECTORY}

    def run():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
        frames = sess.step(action, noise=noise)
        rewards, members = sess.score([action], ensemble_size=2, num_steps=3, seed=1)
        return frames, sess.samples_z.clone(), rewards, members

    with torch.no_grad():
        f1, z1, r1, m1 = run()
        f2, z2, r2, m2 = run()
    torch.cuda.synchronize()
    print(f"576 x 1024 2M: reward {r1.tolist()}")
    assert f1.shape == (T - 3, H, W, 3) and torch.isfinite(m1).all()
    assert torch.equal(f1, f2) and torch.equal(z1, z2) and torch.equal(r1, r2) and torch.equal(m1, m2)
