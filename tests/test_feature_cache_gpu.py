"""Feature caching on the H100: the checks of tests/test_feature_cache_cpu.py on the device kernels and loops.

- A full forward then a cached forward of every branch on the same x, sigma and conditioning are torch.equal, for the
  2T rows, the T rows and the T rows of the "cond" slot, at the tiny and small presets and at 576 x 1024: the cached
  path reads the feature and GroupNorm partials the full forward left.
- A cached forward on new inputs against the fp32 reference (the real VideoUNet's fixture at tiny and small, the oracle
  on the GPU with TF32 off at 576 x 1024), rel-L2 <= 5e-3.
- Tiny fused samples against the oracle loop with the same schedule, Euler and 2M over VanillaCFG, Triangle, ActionCFG
  and IntervalCFG; graph replay bit-equal to eager launches; cache_interval 1 equal to a sampler without the keyword.
- Isolation: interleaved samples, a session against engine.rollout, a score that leaves the session unchanged.
- A 576 x 1024 2M session round with interval 2 over 4 steps repeats bit for bit, at a peak no higher than uncached."""
import gc

import pytest
import torch

import cache_oracle as co
import test_action_cfg_cpu as tac
import test_dpmpp2m_cpu as tdc
import test_feature_cache_cpu as tfc
import test_interval_cfg_cpu as tic
from helpers import golden, rel_l2, unet_weights
from test_fullres_gpu import _bench_session
from test_session_gpu import gpu_engine
from vista_b200 import synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GIB = 2 ** 30
T = tfc.T


@pytest.fixture(scope="module", autouse=True)
def loaded():
    from vista_b200 import lib
    lib.load()


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------------------------
# forwards at tiny and small
# ------------------------------------------------------------------------------------------------------------------
PRESETS = {"tiny": (8, 16, (0, 1, 3)), "small": (16, 32, (0, 1, 11))}


@pytest.mark.parametrize("preset", list(PRESETS))
def test_cached_forward(preset, monkeypatch):
    h, w, branches = PRESETS[preset]
    cfg, sd = unet_weights(preset)
    rt = tfc.runtime(cfg, sd, DEV)
    problem = tfc.forward_problem(cfg, h, w, DEV)
    g = golden(f"unet_cached_{preset}")
    with torch.no_grad():
        tfc.check_same_input_equality(rt, problem, h, w, branches)
        tfc.check_cached_against(rt, problem, h, w, list(g["branches"]), lambda b: torch.from_numpy(g[f"cached_b{b}"]))
        if preset == "tiny":
            tfc.check_cached_launches(rt, problem, h, w, monkeypatch)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# forwards at 576 x 1024
# ------------------------------------------------------------------------------------------------------------------
def test_cached_forward_576x1024():
    """Same-input equality for branches 0, 1 and 11 on the three row sets, then a cached forward of the T conditional
    rows at x1 after a full one at x0 against the fp32 oracle on the GPU (computed after the runtime is released)."""
    from bench import make_problem
    from vista_b200 import spec
    from vista_b200.unet import UNetRuntime
    ucfg, _, _, _, rand_sd = make_problem("full", DEV)
    usd = rand_sd(spec.unet_param_specs(ucfg))
    h, w, branches = 72, 128, (0, 1, 11)
    problem = tfc.forward_problem(ucfg, h, w, DEV)
    (x0, t0), (x1, t1), ctx, y, mask = problem
    rows = slice(T, 2 * T)
    ours = {}
    with torch.no_grad():
        rt = UNetRuntime(ucfg, usd, DEV, T)
        tfc.check_same_input_equality(rt, problem, h, w, branches)
        rt.set_conditioning(ctx[rows], y[rows])
        for b in branches:
            tfc.rt_forward(rt, x0[rows], t0[rows], mask[rows], h, w)
            ours[b] = tfc.rt_forward(rt, x1[rows], t1[rows], mask[rows], h, w, cached=True, cache_branch=b).cpu()
        del rt
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        with torch.device(DEV):
            for b in branches:
                cache = {"branch": b}
                co.unet_forward(usd, ucfg, x0[rows], t0[rows], ctx[rows], y[rows], mask[rows], T, cache)
                ref = co.unet_forward(usd, ucfg, x1[rows], t1[rows], ctx[rows], y[rows], mask[rows], T, cache).cpu()
                del cache
                r = rel_l2(ours[b], ref)
                print(f"576 x 1024 cached forward, branch {b}: {r:.2e} rel-L2 from the fp32 oracle")
                assert r <= tfc.FORWARD_REL, (b, r)


# ------------------------------------------------------------------------------------------------------------------
# tiny samples on the device loops
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network("cuda")


@pytest.mark.parametrize("name,branch", tfc.CASES, ids=[f"{n}-b{b}" for n, b in tfc.CASES])
@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_cached_sample_and_graph_replay(tiny, kind, name, branch, monkeypatch):
    """The cached sample against the oracle loop, launched eagerly; the same sample with its later steps replayed from
    CUDA graphs (one per kind of step, cached steps their own): bit-equal."""
    from vista_b200 import fused as fused_mod
    with torch.no_grad():
        eager = tfc.check_cached_sample(tiny, "cuda", kind, name, branch, monkeypatch)
        monkeypatch.setattr(fused_mod, "USE_GRAPH", True)
        cfg, sd, net, den, bden = tiny
        c, uc, noise, z, mask = tdc.tiny_inputs(cfg, DEV)
        graphed = tfc.make(kind, tfc.guider(name), 2, branch, device="cuda")(bden, noise.clone(), c, uc=uc, cond_frame=z,
                                                                             cond_mask=mask)
        st = next(iter(tic.runtime(net, "cuda")._loop_states.values()))
        if name != "interval":       # there every cached step is the first of its kind, so it runs eagerly
            key = (tfc.STEPS, kind == "dpm") + ((True,) if name == "action" else ()) + ("cached", branch)
            assert key in st.graphs, list(st.graphs)
    torch.cuda.synchronize()
    assert torch.equal(graphed, eager)


def test_interval_one_is_uncached(tiny):
    with torch.no_grad():
        tfc.check_interval_one_is_uncached(tiny, "cuda")


def test_interleaved_and_back_to_back_calls(tiny):
    with torch.no_grad():
        st = tfc.check_interleaved(tiny, "cuda")
    torch.cuda.synchronize()
    assert {(4, False), (4, False, "cached", 1), (4, False, "cached", 3), (4, True, True, "cached", 2)} <= set(st.graphs), \
        list(st.graphs)


# ------------------------------------------------------------------------------------------------------------------
# engine paths, tiny presets of the native YAML
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_session_equals_batch_rollout_and_repeats(eng, monkeypatch, kind):
    tfc.check_session_equals_batch_rollout(eng, DEV, monkeypatch, kind)


def test_score_leaves_the_session_untouched(eng, monkeypatch):
    tfc.check_score_leaves_the_session_untouched(eng, DEV, monkeypatch)


def test_session_round_at_576x1024_repeats_within_the_uncached_peak():
    """The native YAML engine at Vista's resolution with a 4-step 2M sampler (VanillaCFG): the round with cache_interval
    2 (branch 0) repeats bit for bit, and its peak allocation is no higher than the uncached round's, both measured
    after a first round of each (which builds what stays allocated between rounds)."""
    from oracle.make_golden_clip import clip_frames
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    n = 4
    plain = tac.with_guider(eng.sampler, "dpm", tac.vanilla_cfg(), steps=n)
    cached = tac.with_guider(eng.sampler, "dpm", tac.vanilla_cfg(), steps=n)
    cached.cache_interval, cached.cache_branch = 2, 0
    H, W = 576, 1024
    frame = torch.from_numpy(clip_frames(12, "cache_fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "cache_fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "cache_fullres.noise", (T, 4, H // 8, W // 8))).to(DEV)

    def run(smp):
        eng.sampler = smp
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
        frames = sess.step({"trajectory": bs.TRAJECTORY}, noise=noise)
        return frames.cpu(), sess.samples_z.cpu()        # no round's result stays on the device during another's peak

    def peak(smp):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        out = run(smp)
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated(DEV)

    with torch.no_grad():
        run(plain)                  # first rounds: the runtimes, the decoder's arena and every step graph are built
        held = torch.cuda.memory_allocated(DEV)
        run(cached)
        held_cached = torch.cuda.memory_allocated(DEV) - held
        (f0, z0), peak_plain = peak(plain)
        (f1, z1), peak_cached = peak(cached)
        f2, z2 = run(cached)
    print(f"576 x 1024 2M, 4 steps, cache_interval 2: peak allocated {peak_cached / GIB:.2f} GiB, uncached "
          f"{peak_plain / GIB:.2f} GiB; the first cached round kept {held_cached / 2 ** 20:.1f} MiB more allocated; "
          f"final latent {rel_l2(z1, z0):.3e} rel-L2 from uncached (synthetic weights)")
    assert f1.shape == (T - 3, H, W, 3) and torch.isfinite(z1).all()
    assert torch.equal(f1, f2) and torch.equal(z1, z2)
    assert not torch.equal(z1, z0)
    assert peak_cached <= peak_plain
