"""Interval guidance on the H100: the unguided update (the sampler_update_kernel<kMultistep> overload behind
b200v_sampler_update_cond) against the fp64 reference of tests/test_interval_cfg_cpu.py on every layout of the
sampler-step table at the first, middle and final steps, Euler and 2M with NaN D_prev on first-order rows; the tiny
preset's equalities of the CPU file on the device loops, graph replay against eager launches, and a 576 x 1024 2M
session round guided on two of its four steps that repeats bit for bit."""
import pytest
import torch

import test_action_cfg_cpu as tac
import test_dpmpp2m_cpu as tdc
import test_interval_cfg_cpu as tic
from helpers import rel_l2
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
@pytest.mark.parametrize("step", [0, 24, NUM_STEPS - 1])
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=sampler_case_id)
def test_update_cond(ops, case, step, multistep):
    """Every layout of the Euler conformance table (25 x 4 x 72 x 128 with ld_net 8 among them, NULL mask / cond_frame)."""
    tic.check_update_cond(case, step, multistep, ops._sampler_update_cond, DEV)


def test_update_cond_rejects_bad_arguments(ops):
    from test_conformance_small_cpu import make_sampler_inputs
    d = make_sampler_inputs((1, 2, 2, "none", False, False, "const"), DEV, 1)
    coefs = tdc.coef_table(DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    call = lambda net, c, dp: ops._sampler_update_cond(d["x"], net, None, None, c, dp, d["sigmas"], step, NUM_STEPS, 1, 2, 2)
    with pytest.raises(RuntimeError, match="both NULL"):
        call(d["net"], coefs, None)
    with pytest.raises(RuntimeError, match="both NULL"):
        call(d["net"], None, d["x"].clone())
    with pytest.raises(RuntimeError, match="aligned"):
        call(d["net"], coefs.flatten()[1:], d["x"].clone())
    with pytest.raises(RuntimeError, match="ld_net"):
        call(torch.zeros(4, 6, device=DEV), None, None)
    assert int(step[0]) == 0


# ------------------------------------------------------------------------------------------------------------------
# the tiny preset on the device loops
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network("cuda")


@pytest.mark.parametrize("kind", ["euler", "dpm"])
@pytest.mark.parametrize("inner", ["vanilla", "action"])
def test_interval_ends(tiny, kind, inner):
    with torch.no_grad():
        tic.check_interval_ends(tiny, "cuda", kind, inner)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_boundary_rule(tiny, kind, monkeypatch):
    with torch.no_grad():
        tic.check_boundary_rule(tiny, "cuda", kind, monkeypatch)


@pytest.mark.parametrize("inner", ["vanilla", "triangle", "action"])
@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_mixed_interval_and_graph_replay(tiny, kind, inner, monkeypatch):
    """The mixed interval of the CPU file launched eagerly, and the same sample with its later steps replayed from CUDA
    graphs (one per kind of step): bit-equal."""
    from vista_b200 import fused as fused_mod
    with torch.no_grad():
        eager = tic.check_mixed(tiny, "cuda", kind, inner, monkeypatch)
        monkeypatch.setattr(fused_mod, "USE_GRAPH", True)
        cfg, sd, net, den, bden = tiny
        c, uc, noise, z, mask = tdc.tiny_inputs(cfg, DEV)
        smp = tic.make(kind, tic.interval_over(tic.STEPS, *tic.MIXED, tic.wrapped(inner)), device="cuda")
        graphed = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
        st = next(iter(tic.runtime(net, "cuda")._loop_states.values()))
        assert (tic.STEPS, kind == "dpm", "cond") in st.graphs
    torch.cuda.synchronize()
    assert torch.equal(graphed, eager)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_empty_interval_allocates_no_2t_buffers(kind):
    with torch.no_grad():
        tic.check_no_2t_buffers("cuda", kind)


def test_interleaved_and_back_to_back_calls(tiny):
    with torch.no_grad():
        st = tic.check_interleaved(tiny, "cuda")
    torch.cuda.synchronize()
    assert {(4, False, "cond"), (4, True, "cond"), (4, False), (4, True), (4, True, True)} <= set(st.graphs)


# ------------------------------------------------------------------------------------------------------------------
# engine paths, tiny presets of the native YAML
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_session_equals_batch_rollout_and_repeats(eng, monkeypatch, kind):
    tic.check_session_equals_batch_rollout(eng, DEV, monkeypatch, kind)


def test_score_leaves_the_session_untouched(eng, monkeypatch):
    tic.check_score_leaves_the_session_untouched(eng, DEV, monkeypatch)


def test_session_round_at_576x1024_repeats():
    """The native YAML engine at Vista's resolution with a 4-step 2M engine.sampler guided (VanillaCFG) on steps 1 and 2
    only: one session round repeats bit for bit, and its peak allocation is reported."""
    from oracle.make_golden_clip import clip_frames
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    n = 4
    s = [float(v) for v in eng.sampler.discretization(n, device="cpu").to(torch.float32)]
    g = tic.interval_cfg((s[2] * s[3]) ** 0.5, (s[0] * s[1]) ** 0.5, tac.vanilla_cfg())
    eng.sampler = tac.with_guider(eng.sampler, "dpm", g, steps=n)
    assert [eng.sampler.guider.guided(v) for v in s[:n]] == [False, True, True, False]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    T, H, W = eng.num_frames, 576, 1024
    frame = torch.from_numpy(clip_frames(12, "interval_fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "interval_fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "interval_fullres.noise", (T, 4, H // 8, W // 8))).to(DEV)

    def run():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
        frames = sess.step({"trajectory": bs.TRAJECTORY}, noise=noise)
        return frames, sess.samples_z.clone()

    with torch.no_grad():
        f1, z1 = run()
        f2, z2 = run()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV)
    print(f"576 x 1024 IntervalCFG(VanillaCFG) 2M, 4 steps guided on steps 1-2: peak allocated {peak / GIB:.2f} GiB")
    assert f1.shape == (T - 3, H, W, 3) and torch.isfinite(z1).all()
    assert torch.equal(f1, f2) and torch.equal(z1, z2)
    assert peak <= 72 * GIB
