"""Action guidance on the H100: the sampler_update_kernel<*, true> instantiations against the fp64 reference of
tests/test_action_cfg_cpu.py (every layout of the sampler-step table, net_img with its own leading dimension, first,
middle and final steps, NaN D_prev on 2M's first-order rows, per-frame s_img with s_act 0, equal to s_img and above it),
the update's linearity in s_act, the UNet's T-row forward of the conditional half against the 2T-row forward, the fused
loop against the torch loop, graph replay against eager launches, back-to-back and interleaved samples, the engine paths,
and a 576 x 1024 session round and score that repeat bit for bit."""
import pytest
import torch

import test_action_cfg_cpu as tac
import test_dpmpp2m_cpu as tdc
from helpers import rel_l2, to_t, unet_weights
from test_conformance_small_cpu import NUM_STEPS, SAMPLER_CASES, sampler_case_id
from test_fullres_gpu import _bench_session
from test_session_gpu import gpu_engine
from vista_b200 import synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GIB = 2 ** 30


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as _ops
    lib.load()
    return _ops


@pytest.mark.parametrize("multistep", [False, True], ids=["euler", "2m"])
@pytest.mark.parametrize("s_act", tac.S_ACT_KINDS)
@pytest.mark.parametrize("step", [0, 24, NUM_STEPS - 1])
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=sampler_case_id)
def test_update_action(ops, case, step, s_act, multistep):
    """Every layout of the Euler conformance table (25 x 4 x 72 x 128 with ld_net 8 among them, NULL mask / cond_frame),
    net_img with ld_img 12."""
    tac.check_update_action(case, step, s_act, multistep, ops.sampler_update_action, DEV)


@pytest.mark.parametrize("multistep", [False, True], ids=["euler", "2m"])
def test_update_linear_in_s_act(ops, multistep):
    diff = tac.check_linear_in_s_act(ops.sampler_update_action, DEV, multistep)
    print(f"{'2M' if multistep else 'Euler'}: max |update difference| at s_act 0.5 / 1 / 2: "
          f"{[float(diff[a].abs().max()) for a in (0.5, 1.0, 2.0)]}")


def test_update_action_rejects_bad_arguments(ops):
    d = tac.action_inputs((1, 2, 2, "none", False, False, "const"), DEV, 1, "same")
    coefs = tdc.coef_table(DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    call = lambda net_img, c, dp: ops.sampler_update_action(d["x"], d["net"], net_img, None, None, d["scales"],
                                                            d["action_scales"], c, dp, d["sigmas"], step, NUM_STEPS, 1, 2, 2)
    with pytest.raises(RuntimeError, match="both NULL"):
        call(d["net_img"], coefs, None)
    with pytest.raises(RuntimeError, match="both NULL"):
        call(d["net_img"], None, d["x"].clone())
    with pytest.raises(RuntimeError, match="aligned"):
        call(d["net_img"], coefs.flatten()[1:], d["x"].clone())
    with pytest.raises(RuntimeError, match="ld_img"):
        call(torch.zeros(4, 6, device=DEV), None, None)
    assert int(step[0]) == 0


@pytest.mark.parametrize("hw", [(8, 16), (72, 128)], ids=["8x16", "72x128"])
def test_t_row_forward_equals_conditional_half(ops, hw):
    """The image branch's T-row forward reads the conditional half of the prepared batch; under the conditional rows'
    own conditioning it is bit for bit rows [T, 2T) of the 2T-row forward (tiny UNet weights, Vista's layer plan)."""
    from vista_b200.unet import UNetRuntime, padded_input_rows
    h, w = hw
    cfg, sd = unet_weights("tiny")
    rt = UNetRuntime(cfg, to_t(sd, DEV), DEV, 25)
    T = 25
    c, uc = synth.synth_conditioning(3, T, h, w, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
    c, uc = to_t(c, DEV), to_t(uc, DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    unet_in = padded_input_rows(2 * T * h * w, DEV)
    unet_in.copy_(torch.randn(2 * T * h * w, 8, generator=g, device=DEV).half())
    c_noise = torch.full((2 * T,), 0.7, device=DEV)
    mask2 = torch.zeros(2 * T, device=DEV)
    mask2[0] = mask2[T] = 1.0
    with torch.no_grad():
        rt.set_conditioning(torch.cat((uc["crossattn"], c["crossattn"])), torch.cat((uc["vector"], c["vector"])))
        rt.set_conditioning(c["crossattn"], c["vector"])
        full = rt.forward(unet_in, c_noise, mask2, h, w).clone()
        half = rt.forward(unet_in[T * h * w:], c_noise[T:], mask2[T:], h, w).clone()
        full2 = rt.forward(unet_in, c_noise, mask2, h, w)          # the 2T conditioning was not replaced by the T-row one
    torch.cuda.synchronize()
    assert torch.equal(full2, full)
    rows = full[T * h * w:, :4]
    print(f"{h}x{w}: T-row forward vs rows [T, 2T): max |diff| {float((half[:, :4] - rows).abs().max()):.3e}")
    assert torch.equal(half[:, :4], rows)


@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network("cuda")


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_fused_against_torch_loop_and_graph_replay(tiny, kind, monkeypatch):
    """The fused loop (steps replayed from CUDA graphs) against the torch loop on the tiny UNet, and against the same
    fused loop launched eagerly: bit-equal."""
    from vista_b200 import fused as fused_mod
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, DEV)
    smp = tac.make_sampler(kind, 4, 5.0, tac.triangle_cfg(), "cuda")
    run = lambda d: smp(d, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    with torch.no_grad():
        graphed = run(bden)
        generic = run(lambda x, s, cc, m: den(net, x, s, cc, m))
        monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
        eager = run(bden)
        image_only = tac.with_guider(smp, kind, tac.triangle_cfg())(bden, noise.clone(), c, uc=uc, cond_frame=z,
                                                                    cond_mask=mask)
    torch.cuda.synchronize()
    r = rel_l2(graphed, generic)
    print(f"tiny {kind} + ActionCFG(5.0), 4 steps: fused vs torch loop rel-L2 {r:.3e}; "
          f"against the image guider alone {rel_l2(graphed, image_only):.3e}")
    assert torch.equal(graphed, eager)
    assert r < tac.FUSED_REL and torch.equal(graphed[:1], z[:1])
    assert rel_l2(graphed, image_only) > 10 * r
    st = next(iter(net._rt_get(net.diffusion_model, 25, DEV)._loop_states.values()))
    assert (4, kind == "dpm", True) in st.graphs


def test_interleaved_and_back_to_back_calls(tiny):
    """Vanilla then ActionCFG, two ActionCFG samples with different action_scale (one captured graph, the scale read on
    the device), Euler and 2M: each equals its standalone run on a fresh loop state."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, DEV)
    tri = tac.triangle_cfg()
    samplers = [tdc.make_sampler("euler", 4, "cuda", guider=tri), tac.make_sampler("euler", 4, 5.0, tri, "cuda"),
                tac.make_sampler("euler", 4, 1.0, tri, "cuda"), tac.make_sampler("dpm", 4, 5.0, tri, "cuda"),
                tac.make_sampler("dpm", 4, 2.0, tri, "cuda"), tdc.make_sampler("dpm", 4, "cuda", guider=tri)]

    def fresh():
        net._rt_get(net.diffusion_model, 25, DEV).__dict__.pop("_loop_states", None)

    run = lambda smp: smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    with torch.no_grad():
        alone = []
        for smp in samplers:
            fresh()
            alone.append(run(smp))
        fresh()
        seq = [run(smp) for smp in samplers + samplers[::-1]]
    torch.cuda.synchronize()
    for i, (got, want) in enumerate(zip(seq, alone + alone[::-1])):
        assert torch.equal(got, want), i
    assert not torch.equal(alone[1], alone[2]) and not torch.equal(alone[3], alone[4])
    st = next(iter(net._rt_get(net.diffusion_model, 25, DEV)._loop_states.values()))
    assert set(st.graphs) == {(4, False), (4, False, True), (4, True, True), (4, True)}


# ------------------------------------------------------------------------------------------------------------------
# engine paths, tiny presets of the native YAML
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


def test_action_free_equals_forced_zero_actions(eng):
    tac.check_action_free_equals_forced_zero_actions(eng, DEV)


def test_engine_sample(eng, monkeypatch):
    tac.check_engine_sample(eng, DEV, monkeypatch)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_session_equals_batch_rollout_and_repeats(eng, monkeypatch, kind):
    tac.check_session_equals_batch_rollout(eng, DEV, monkeypatch, kind)


def test_score_leaves_the_session_untouched(eng, monkeypatch):
    tac.check_score_leaves_the_session_untouched(eng, DEV, monkeypatch)


def test_session_round_and_score_at_576x1024_repeat_and_fit():
    """The native YAML engine at Vista's resolution with a 2M ActionCFG engine.sampler: one 2-step session round, then a
    score of 2 candidates x 2 members x 2 steps; both repeat bit for bit, and the peak allocation is reported and held
    within 72 GiB (the decoder's scratch stays allocated once the session has stepped)."""
    from oracle.make_golden_clip import clip_frames
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    eng.sampler = tac.with_guider(eng.sampler, "dpm", tac.action_cfg(5.0, tac.triangle_cfg(eng.num_frames)), steps=2)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    T, H, W = eng.num_frames, 576, 1024
    frame = torch.from_numpy(clip_frames(12, "action_fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "action_fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "action_fullres.noise", (T, 4, H // 8, W // 8))).to(DEV)
    candidates = [{"trajectory": bs.TRAJECTORY}, {"trajectory": bs.TRAJECTORY * 0.5}]

    def run():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
        frames = sess.step(candidates[0], noise=noise)
        rewards, members = sess.score(candidates, ensemble_size=2, num_steps=2, seed=1)
        return frames, sess.samples_z.clone(), rewards, members

    with torch.no_grad():
        f1, z1, r1, m1 = run()
        f2, z2, r2, m2 = run()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV)
    print(f"576 x 1024 ActionCFG(5.0) 2M: a 2-step round, then a score (K = 2, E = 2, 2 steps): rewards {r1.tolist()}, "
          f"peak allocated {peak / GIB:.2f} GiB")
    assert f1.shape == (T - 3, H, W, 3) and m1.shape == (2, 2, T, 4, H // 8, W // 8) and torch.isfinite(m1).all()
    assert torch.equal(f1, f2) and torch.equal(z1, z2) and torch.equal(r1, r2) and torch.equal(m1, m2)
    assert not torch.equal(m1[0], m1[1])
    assert peak <= 72 * GIB
