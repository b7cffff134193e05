"""Interval guidance (vista_b200.diffusion.IntervalCFG) without a GPU: the guider's construction rules and per-call
semantics, the torch loop and the fused loop (on the CPU twins of the kernels, tests/interval_fake_ops.py) at the two
ends of the interval (every step guided: the wrapped guider; none: IdentityGuider), the boundary rule on a hand-built
sigma table, a mixed interval in the fused loop against the torch loop, the forward-row counts and the 2T buffers the
schedule needs, interleaved samples, the engine paths above the sampler, and the fp64 reference of the unguided update
(the kernel is held to it in tests/test_interval_cfg_gpu.py, its twin here)."""
import math

import pytest
import torch

import seam_fakes as sf
import test_action_cfg_cpu as tac
import test_dpmpp2m_cpu as tdc
from helpers import rel_l2
from interval_fake_ops import patched_interval_ops
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs

IDENTITY = {"target": "vista_b200.diffusion.IdentityGuider"}
STEPS = 4


def interval_cfg(sigma_lo, sigma_hi, guider_config):
    return {"target": "vista_b200.diffusion.IntervalCFG",
            "params": {"sigma_lo": float(sigma_lo), "sigma_hi": float(sigma_hi), "guider_config": guider_config}}


def wrapped(name, T=25):
    """The guider configs IntervalCFG is tested over."""
    return {"vanilla": tac.vanilla_cfg(), "triangle": tac.triangle_cfg(T),
            "action": tac.action_cfg(5.0, tac.triangle_cfg(T))}[name]


def table(n):
    """The fp32 sigma table of tdc.DISC the fused loop reads for n steps (n + 1 values, the last 0)."""
    from vista_b200.diffusion import instantiate_from_config
    return instantiate_from_config(tdc.DISC)(n, device="cpu").to(torch.float32)


def interval_over(n, first, last, guider_config):
    """IntervalCFG guiding steps first..last of n (none when first > last): each end at the geometric mean of two table
    values, so that the loops' sigma tables (computed on the host or on the device) agree on every step."""
    s = [float(v) for v in table(n)]
    mid = lambda i: math.sqrt(s[i] * s[i + 1]) if s[i + 1] > 0 else s[i] / 2
    if first > last:
        return interval_cfg(4 * s[0], 8 * s[0], guider_config)          # above every step
    return interval_cfg(mid(last), 2 * s[0] if first == 0 else mid(first - 1), guider_config)


class TableDiscretization:
    """A fixed fp32 sigma table (n + 1 values, the last 0), as EDMDiscretization is called by the samplers."""

    def __init__(self, sigmas):
        self.sigmas = torch.as_tensor(sigmas, dtype=torch.float32)

    def __call__(self, n, do_append_zero=True, device="cpu", flip=False):
        assert n + 1 == self.sigmas.numel() and do_append_zero and not flip
        return self.sigmas.to(device)


def make(kind, guider_config, steps=STEPS, device="cpu"):
    return tdc.make_sampler(kind, steps, device, guider=guider_config)


def guided_steps(guider, sigmas, n):
    from vista_b200.diffusion import IntervalCFG
    if not isinstance(guider, IntervalCFG):
        return [type(guider).__name__ != "IdentityGuider"] * n
    return [guider.guided(sigmas[i]) for i in range(n)]


# ------------------------------------------------------------------------------------------------------------------
# the guider
# ------------------------------------------------------------------------------------------------------------------
def test_construction_rules():
    from vista_b200.diffusion import ActionCFG, IntervalCFG, instantiate_from_config
    for inner in ("vanilla", "triangle", "action"):
        g = instantiate_from_config(interval_cfg(0.28, 5.42, wrapped(inner)))
        assert isinstance(g, IntervalCFG) and g.sigma_lo == 0.28 and g.sigma_hi == 5.42
    linear = {"target": "vista_b200.diffusion.LinearPredictionGuider", "params": {"num_frames": 25}}
    IntervalCFG(0.1, 1.0, linear)
    with pytest.raises(ValueError, match="below"):
        IntervalCFG(5.42, 5.42, tac.vanilla_cfg())
    with pytest.raises(ValueError, match="below"):
        IntervalCFG(6.0, 5.42, tac.vanilla_cfg())
    for bad in (IDENTITY, interval_cfg(0.1, 1.0, tac.vanilla_cfg()), tac.action_cfg(2.0, IDENTITY)):
        with pytest.raises(ValueError, match="wraps"):
            IntervalCFG(0.1, 1.0, bad)
    with pytest.raises(ValueError, match="outermost"):
        ActionCFG(2.0, interval_cfg(0.1, 1.0, tac.vanilla_cfg()))


def test_per_call_semantics():
    """Inside (sigma_lo, sigma_hi] prepare_inputs and __call__ are the wrapped guider's; outside, (x, s, c, cond_mask)
    pass through and the output is the identity.  The ends: sigma_lo excluded, sigma_hi included."""
    from vista_b200.diffusion import IntervalCFG, VanillaCFG
    lo, hi = 0.5, 4.0
    g, v = IntervalCFG(lo, hi, tac.vanilla_cfg()), VanillaCFG(2.5)
    T = 2
    c = {"crossattn": torch.randn(T, 1, 5), "vector": torch.randn(T, 7), "concat": torch.randn(T, 4, 2, 2)}
    uc = {k: torch.randn_like(t) for k, t in c.items()}
    x, m = torch.randn(T, 4, 2, 2), torch.tensor([1.0, 0.0])
    out2 = torch.randn(2 * T, 4, 2, 2)
    for sig, inside in ((hi, True), (lo, False), (1.0, True), (hi * 1.0001, False), (lo * 0.5, False)):
        s = torch.full((T,), sig)
        assert g.guided(s) == inside == g.guided(sig)
        got, want = g.prepare_inputs(x, s, c, m, uc), (v.prepare_inputs(x, s, c, m, uc) if inside else (x, s, c, m))
        assert all(torch.equal(a, b) for a, b in zip(got[:2] + got[3:], want[:2] + want[3:]))
        assert set(got[2]) == set(want[2]) and all(torch.equal(got[2][k], want[2][k]) for k in want[2])
        if inside:
            assert torch.equal(g(out2, s), v(out2, s))
        else:
            assert g(x, s) is x


# ------------------------------------------------------------------------------------------------------------------
# the torch loop and the fused loop on the tiny UNet
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network()


@pytest.fixture
def emulated(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    with patched_interval_ops(), torch.no_grad():
        yield


def runtime(net, dev):
    """The runtime the fused loop uses: its key holds the device of the latents (cuda:0, not cuda)."""
    d = torch.device(dev)
    if d.type == "cuda" and d.index is None:
        d = torch.device("cuda", torch.cuda.current_device())
    return net._rt_get(net.diffusion_model, 25, d)


def fresh(net, dev):
    runtime(net, dev).__dict__.pop("_loop_states", None)


def run_pair(tiny, smp, dev):
    """(fused, torch loop) samples of ``smp`` on the tiny inputs."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    run = lambda d: smp(d, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    return run(bden), run(lambda x, s, cc, m: den(net, x, s, cc, m))


def check_interval_ends(tiny, dev, kind, inner):
    """An interval holding every step is the wrapped guider's sample, an empty one IdentityGuider's, torch.equal in
    either loop."""
    every = run_pair(tiny, make(kind, interval_over(STEPS, 0, STEPS - 1, wrapped(inner)), device=dev), dev)
    plain = run_pair(tiny, make(kind, wrapped(inner), device=dev), dev)
    empty = run_pair(tiny, make(kind, interval_over(STEPS, 1, 0, wrapped(inner)), device=dev), dev)
    ident = run_pair(tiny, make(kind, IDENTITY, device=dev), dev)
    for got, want in zip(every + empty, plain + ident):
        assert torch.equal(got, want)
    assert not torch.equal(plain[0], ident[0])


def counting_forwards(monkeypatch, tiny, dev):
    """Records (rows, slot) of every UNet runtime forward and the batch of every network call of the torch loop."""
    cfg, sd, net, den, bden = tiny
    rt = runtime(net, dev)
    rows, real = [], rt.forward

    def forward(unet_in, c_noise, *a, **k):
        rows.append((c_noise.numel(), k.get("slot", "")))
        return real(unet_in, c_noise, *a, **k)
    monkeypatch.setattr(rt, "forward", forward)
    return rows


def check_boundary_rule(tiny, dev, kind, monkeypatch):
    """A hand-built table with sigma_lo and sigma_hi exactly on table values: the step at sigma_hi is guided, the one at
    sigma_lo is not, in both loops (the rows of each network call), and the fused loop is the torch loop.  The fused
    loop runs eagerly, so that every step's forward is seen."""
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    sig = [80.0, 9.5, 2.25, 0.5, 0.0]
    smp = make(kind, interval_cfg(sig[3], sig[1], tac.triangle_cfg()), device=dev)
    smp.discretization = TableDiscretization(sig)
    assert guided_steps(smp.guider, torch.tensor(sig), 4) == [False, True, True, False]
    fwd = counting_forwards(monkeypatch, tiny, dev)
    fused = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    assert [r for r, _ in fwd] == [25, 50, 50, 25] and [s for _, s in fwd] == ["cond", "", "", "cond"]
    calls = []
    generic = smp(lambda x, s, cc, m: (calls.append(x.shape[0]), den(net, x, s, cc, m))[1], noise.clone(), c, uc=uc,
                  cond_frame=z, cond_mask=mask)
    assert calls == [25, 50, 50, 25]
    assert rel_l2(fused, generic) < tac.FUSED_REL and torch.equal(fused[:1], z[:1])


# guided steps 1..2 of 4: unguided -> guided -> guided -> unguided, so a 2M sample crosses the boundary both ways
MIXED = (1, 2)


def check_mixed(tiny, dev, kind, inner, monkeypatch):
    """Guidance on steps 1..2 of 4: the fused loop against the torch loop within the 2M / ActionCFG bar, the UNet rows
    each loop runs equal to the schedule's counts, and the sample differs from both ends.  The fused loop runs eagerly,
    so that every step's forward is seen."""
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    fwd = counting_forwards(monkeypatch, tiny, dev)
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    smp = make(kind, interval_over(STEPS, *MIXED, wrapped(inner)), device=dev)
    sched = guided_steps(smp.guider, table(STEPS), STEPS)
    assert sched == [False, True, True, False]
    fused = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    fused_fwd = list(fwd)
    calls = []
    generic = smp(lambda x, s, cc, m: (calls.append(x.shape[0]), den(net, x, s, cc, m))[1], noise.clone(), c, uc=uc,
                  cond_frame=z, cond_mask=mask)
    n_g, n_u = sum(sched), STEPS - sum(sched)
    guided_rows = 75 if inner == "action" else 50
    assert calls.count(guided_rows) == n_g and calls.count(25) == n_u and len(calls) == STEPS
    assert fused_fwd.count((50, "")) == n_g and fused_fwd.count((25, "cond")) == n_u
    assert fused_fwd.count((25, "")) == (n_g if inner == "action" else 0) and len(fused_fwd) == STEPS + fused_fwd.count((25, ""))
    full = make(kind, wrapped(inner), device=dev)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    ident = make(kind, IDENTITY, device=dev)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    r = rel_l2(fused, generic)
    print(f"tiny {kind} IntervalCFG({inner}) on steps {MIXED} of {STEPS}: fused vs torch loop rel-L2 {r:.3e}; "
          f"against full guidance {rel_l2(fused, full):.3e}, against none {rel_l2(fused, ident):.3e}")
    assert r < tac.FUSED_REL and torch.equal(fused[:1], z[:1])
    assert not torch.equal(fused, full) and rel_l2(fused, ident) > 10 * r      # the row counts above tell the schedule
    return fused


def check_no_2t_buffers(dev, kind):
    """On a fresh runtime, an empty interval and IdentityGuider run no 2T-row forward: no 2T conditioning is set and
    no buffer of 2T rows is allocated; the unguided steps run under the runtime's own slot."""
    tiny = tdc.tiny_network(dev)
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    for g in (interval_over(STEPS, 1, 0, wrapped("action")), IDENTITY):
        make(kind, g, device=dev)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    rt = runtime(net, dev)
    T, hw = 25, 8 * 16
    assert set(rt.conds) == {(T, "cond")}, list(rt.conds)
    assert ("gn.stats", 2 * T) not in rt._bufs
    assert not [k for k in rt._bufs if len(k) >= 2 and k[1] in (2 * T, 2 * T * hw)], \
        sorted(str(k) for k in rt._bufs if k[1] in (2 * T, 2 * T * hw))
    return rt


def samplers_for_interleaving(dev):
    tri = tac.triangle_cfg()
    return [make("euler", tri, device=dev), make("euler", interval_over(STEPS, *MIXED, tri), device=dev),
            make("euler", IDENTITY, device=dev), make("euler", tac.action_cfg(5.0, tri), device=dev),
            make("dpm", interval_over(STEPS, *MIXED, tac.action_cfg(5.0, tri)), device=dev),
            make("dpm", interval_over(STEPS, 0, 0, tri), device=dev), make("dpm", IDENTITY, device=dev),
            make("dpm", tri, device=dev)]


def check_interleaved(tiny, dev):
    """Vanilla / Interval / Identity / ActionCFG, Euler and 2M, back to back and interleaved on one loop state and one
    runtime: each equals its standalone run on a fresh loop state."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    samplers = samplers_for_interleaving(dev)
    run = lambda smp: smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    alone = []
    for smp in samplers:
        fresh(net, dev)
        alone.append(run(smp))
    fresh(net, dev)
    seq = [run(smp) for smp in samplers + samplers[::-1]]
    for i, (got, want) in enumerate(zip(seq, alone + alone[::-1])):
        assert torch.equal(got, want), i
    assert not torch.equal(alone[0], alone[1]) and not torch.equal(alone[1], alone[2])
    return next(iter(runtime(net, dev)._loop_states.values()))


@pytest.mark.parametrize("kind", ["euler", "dpm"])
@pytest.mark.parametrize("inner", ["vanilla", "action"])
def test_interval_ends(tiny, emulated, kind, inner):
    check_interval_ends(tiny, "cpu", kind, inner)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_boundary_rule(tiny, emulated, kind, monkeypatch):
    check_boundary_rule(tiny, "cpu", kind, monkeypatch)


@pytest.mark.parametrize("inner", ["vanilla", "triangle", "action"])
@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_mixed_interval_fused_against_torch_loop(tiny, emulated, kind, inner, monkeypatch):
    check_mixed(tiny, "cpu", kind, inner, monkeypatch)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_empty_interval_allocates_no_2t_buffers(emulated, kind):
    check_no_2t_buffers("cpu", kind)


def test_interleaved_and_back_to_back_calls(tiny, emulated):
    check_interleaved(tiny, "cpu")


def test_routing(tiny, emulated, monkeypatch):
    """IntervalCFG and IdentityGuider reach the fused loop, through the reference's closure too; the frame-sharded loop
    refuses both."""
    cfg, sd, net, den, bden = tiny
    calls = tac.counting_fused(monkeypatch)
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)
    model = type("M", (), {"model": net, "denoiser": den})()

    def denoiser(x, sigma, cond, cond_mask):           # sample_utils.py:314-315, verbatim shape
        return model.denoiser(model.model, x, sigma, cond, cond_mask)
    for g in (interval_over(2, 0, 0, tac.triangle_cfg()), IDENTITY):
        smp = make("euler", g, steps=2)
        assert torch.equal(smp(denoiser, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask),
                           smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask))
    assert calls == ["IntervalCFG"] * 2 + ["IdentityGuider"] * 2
    monkeypatch.setattr(net, "frame_sharded", True, raising=False)
    for g in (interval_over(2, 0, 0, tac.triangle_cfg()), IDENTITY):
        with pytest.raises(NotImplementedError, match="frame-sharded"):
            make("euler", g, steps=2)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)


# ------------------------------------------------------------------------------------------------------------------
# engine paths above the sampler, on the tiny native engine (shared with tests/test_interval_cfg_gpu.py)
# ------------------------------------------------------------------------------------------------------------------
def interval_sampler(eng, kind="euler", inner=None, steps=None):
    """A sampler of ``kind`` with the engine's discretisation, guided on step 1 only of its schedule."""
    n = eng.sampler.num_steps if steps is None else steps
    g = interval_over(n, 1, 1, inner or tac.action_cfg(5.0, tac.triangle_cfg(sf.T)))
    return tac.with_guider(eng.sampler, kind, g, steps)


def check_session_equals_batch_rollout(eng, dev, monkeypatch, kind):
    """A session whose engine samples with IntervalCFG is byte for byte engine.rollout(..., u8=True) with the same
    sampler over 2 rounds, on the fused loop; and it repeats bit for bit."""
    from vista_b200.rollout import conditioner_recondition
    monkeypatch.setattr(eng, "sampler", interval_sampler(eng, kind))
    vd, z, noises = inputs(2, "interval_session")
    z, noises = z.to(dev), [n.to(dev) for n in noises]
    calls = tac.counting_fused(monkeypatch)

    def run_session():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        return torch.cat([sess.step(None, noise=nz) for nz in noises] + [sess.close()]), sess.samples_z

    frames, samples_z = run_session()
    assert calls == ["IntervalCFG"] * 2
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, 2, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                               u8=True)
    assert calls == ["IntervalCFG"] * 4
    assert torch.equal(frames, want) and torch.equal(samples_z, want_z)
    frames2, samples_z2 = run_session()
    assert torch.equal(frames, frames2) and torch.equal(samples_z, samples_z2)


def check_score_leaves_the_session_untouched(eng, dev, monkeypatch):
    """The engine samples with VanillaCFG; a session that scores with an IntervalCFG sampler before every step samples
    the same rounds as one that never scores.  Round 0's score is sample_ensemble with that sampler."""
    monkeypatch.setattr(eng, "sampler", tac.with_guider(eng.sampler, "euler", tac.vanilla_cfg()))
    vd, z, ns = inputs(2, "interval_score")
    z, ns = z.to(dev), [n.to(dev) for n in ns]
    itv = interval_sampler(eng, "dpm", tac.vanilla_cfg())
    calls = tac.counting_fused(monkeypatch)

    def run(scoring):
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        frames, scores = [], []
        for nz in ns:
            if scoring:
                scores.append(sess.score([tac.B, None], ensemble_size=2, num_steps=eng.sampler.num_steps, noises=ns,
                                         sampler=itv))
            frames.append(sess.step(tac.A, noise=nz))
        return torch.cat(frames + [sess.close()]), sess.samples_z, scores

    f0, z0, _ = run(False)
    f1, z1, scores = run(True)
    assert torch.equal(f0, f1) and torch.equal(z0, z1)
    assert calls.count("IntervalCFG") == 2 * 2 * 2                     # 2 rounds x 2 candidates x 2 members
    rewards, members = scores[0]
    monkeypatch.setattr(eng, "sampler", itv)
    reward, want = eng.sample_ensemble(*eng.condition({**vd, **tac.B}, sf.T, mgc.UC_KEYS), z, 2, noises=ns)
    assert calls[-2:] == ["IntervalCFG"] * 2
    assert torch.equal(members[0], torch.stack(want)) and torch.equal(rewards[0], reward)


@pytest.fixture(scope="module")
def eng():
    """The tiny native engine; its sampler is Euler with the Triangle guider, 3 steps."""
    e = native_engine(steps=3)
    e.en_and_decode_n_samples_a_time = 14
    return e


def test_yaml_guider_config(eng):
    """The YAML form of the sampler's guider_config builds the guider."""
    from vista_b200.diffusion import IntervalCFG, TrianglePredictionGuider, instantiate_from_config
    g = instantiate_from_config({"target": "vista_b200.diffusion.IntervalCFG",
                                 "params": {"sigma_lo": 0.28, "sigma_hi": 5.42, "guider_config": tac.triangle_cfg(sf.T)}})
    assert isinstance(g, IntervalCFG) and isinstance(g.guider, TrianglePredictionGuider)


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_session_equals_batch_rollout(eng, emulated, monkeypatch, kind):
    check_session_equals_batch_rollout(eng, torch.device("cpu"), monkeypatch, kind)


def test_score_leaves_the_session_untouched(eng, emulated, monkeypatch):
    check_score_leaves_the_session_untouched(eng, torch.device("cpu"), monkeypatch)


# ------------------------------------------------------------------------------------------------------------------
# conformance of the unguided update (the kernel in tests/test_interval_cfg_gpu.py, its CPU twin here)
# ------------------------------------------------------------------------------------------------------------------
def update_cond_reference(x, d, step, num_steps, coefs=None, d_prev=None):
    """fp64 unguided step from fp32 inputs -> (x', D, bound on x', bound on D).  D = x c_skip + c_out c, c the T
    conditional rows of net.  M = |x| + c_skip |x| + |c_out| |c| bounds |x|, |D| and |x - D| / 2.  D's roundings: c_skip
    3 U24, c_out 6, the two products and the sum 2: 11 U24 M; the Euler step adds 11 (test_conformance_small_cpu.
    update_reference), 22 U24 M <= UPDATE_EPS M.  The 2M step as in test_dpmpp2m_cpu.update_2m_reference, with this M."""
    from test_conformance_small_cpu import UPDATE_EPS
    T, h, w = d["T"], d["h"], d["w"]
    hw = h * w
    s, s1 = float(d["sigmas"][step]), float(d["sigmas"][step + 1])
    c_skip, c_out = 1.0 / (s * s + 1.0), -s * (s * s + 1.0) ** -0.5
    c = d["net"][T * hw:2 * T * hw, :4].double().reshape(T, h, w, 4).permute(0, 3, 1, 2)
    x64 = x.double()
    den = x64 * c_skip + c_out * c
    mag = x64.abs() + c_skip * x64.abs() + abs(c_out) * c.abs()
    if coefs is None:
        xn = x64 + (x64 - den) / s * (s1 - s)
        bound = UPDATE_EPS * mag
    else:
        ka, kb, kc, ke = (float(v) for v in coefs[step].double())
        dp = torch.zeros_like(x64) if ke == 0.0 else d_prev.double()
        xn = ka * x64 - kb * (kc * den - ke * dp)
        bound = UPDATE_EPS * (abs(ka) * x64.abs() + abs(kb) * ((abs(kc) + abs(ke)) * mag + abs(ke) * dp.abs()))
    if step + 1 == num_steps and d["mask"] is not None:
        m = d["mask"].double().reshape(T, 1, 1, 1)
        xn = xn * (1 - m) + d["cond_frame"].double() * m
        bound = bound * (1 - m)
    return xn, den, bound, UPDATE_EPS * mag


def check_update_cond(case, step, multistep, update, device):
    """One unguided update at `step` of the 50-step schedule through `update` (the op or its twin), Euler or 2M, on
    net_c = the conditional rows of the case's net (ld_net 8, columns 4.. NaN).  On 2M's first-order rows D_prev is NaN:
    it must not be read."""
    from test_conformance_small_cpu import NUM_STEPS, assert_elements, make_sampler_inputs, randn, sampler_case_id, sync
    d = make_sampler_inputs(case, device, seed=80 + step)
    T, h, w = d["T"], d["h"], d["w"]
    name = f"cond-only {'2M' if multistep else 'Euler'} {sampler_case_id(case)} step {step}"
    coefs = d_prev = None
    if multistep:
        coefs = tdc.coef_table(device)
        d_prev = (torch.full_like(d["x"], float("nan")) if float(coefs[step, 3]) == 0.0
                  else randn(d["x"].shape, 97 + step, device))
    x = d["x"].clone()
    xn_ref, den_ref, bound, den_bound = update_cond_reference(x, d, step, NUM_STEPS, coefs, d_prev)
    idx = torch.tensor([step], dtype=torch.int32, device=device)
    net_c = d["net"][T * h * w:]
    update(x, net_c, d["cond_frame"], d["mask"], coefs, d_prev, d["sigmas"], idx, NUM_STEPS, T, h, w)
    sync(device)
    assert int(idx[0]) == step + 1, f"{name}: step_idx {int(idx[0])}"
    assert bool(torch.isfinite(x).all()), f"{name}: non-finite x"
    assert_elements(x, xn_ref, bound + 2.0 ** -24 * xn_ref.abs(), f"{name}: x")
    if multistep:
        assert_elements(d_prev, den_ref, den_bound + 2.0 ** -24 * den_ref.abs(), f"{name}: D_prev")
    if step + 1 == NUM_STEPS and d["mask"] is not None:
        m = d["mask"].bool()
        assert torch.equal(x[m], d["cond_frame"][m]), f"{name}: conditioning frames not re-imposed exactly"


@pytest.mark.parametrize("multistep", [False, True], ids=["euler", "2m"])
@pytest.mark.parametrize("step", [0, 24, 49])
@pytest.mark.parametrize("case", [(25, 8, 16, "rollout", False, True, "const"), (25, 8, 16, "none", True, False, "triangle"),
                                  (3, 5, 7, "init", False, False, "const"), (1, 1, 1, "none", False, False, "triangle")],
                         ids=lambda c: "T{}x{}x{}-{}".format(*c[:4]))
def test_update_cond_twin(case, step, multistep):
    import interval_fake_ops
    check_update_cond(case, step, multistep, interval_fake_ops.sampler_update_cond, torch.device("cpu"))
