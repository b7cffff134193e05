"""Action guidance (vista_b200.diffusion.ActionCFG) without a GPU: the action-free conditioning against the conditioner's
forced-zero action keys, the guider's algebra, the order of convergence on a closed-form denoiser with three branch means
through the torch loop and the fused loop (on the CPU twins of the kernels, tests/action_fake_ops.py), the fused loop
against the torch loop on the tiny UNet, the routing, the engine paths above the sampler, and the fp64 reference of the
action-guided update (the kernel is held to it in tests/test_action_cfg_gpu.py, its twin here)."""
import math
import types

import pytest
import torch

import seam_fakes as sf
import test_dpmpp2m_cpu as tdc
from action_fake_ops import patched_action_ops
from helpers import rel_l2
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs

DISC = tdc.DISC
ACTION_KEYS = ("command", "trajectory", "speed", "angle", "goal")
CONTEXT_DIM = 1024
A = tdc.A
B = tdc.B


def vanilla_cfg(scale=2.5):
    return {"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": scale}}


def triangle_cfg(T=25):
    return {"target": "vista_b200.diffusion.TrianglePredictionGuider", "params": {"max_scale": 2.5, "num_frames": T}}


def action_cfg(action_scale, image=None, context_dim=CONTEXT_DIM):
    return {"target": "vista_b200.diffusion.ActionCFG",
            "params": {"action_scale": action_scale, "guider_config": image or vanilla_cfg(), "context_dim": context_dim}}


def make_sampler(kind, steps, action_scale, image=None, device="cpu", context_dim=CONTEXT_DIM):
    """An Euler or 2M sampler ("euler" / "dpm") guided by ActionCFG(action_scale, image)."""
    return tdc.make_sampler(kind, steps, device, guider=action_cfg(action_scale, image, context_dim))


def with_guider(sampler, kind, guider_config, steps=None):
    """A sampler of ``kind`` with ``sampler``'s discretisation and num_steps, guided by ``guider_config``."""
    s = tdc.make_sampler(kind, sampler.num_steps if steps is None else steps, sampler.device, guider=guider_config)
    s.discretization = sampler.discretization
    return s


# ------------------------------------------------------------------------------------------------------------------
# the guider
# ------------------------------------------------------------------------------------------------------------------
def test_action_free_zeroes_the_action_columns_only():
    from vista_b200.diffusion import ActionCFG
    g = ActionCFG(3.0, vanilla_cfg())
    c = {"crossattn": torch.randn(4, 1, CONTEXT_DIM + 2432), "vector": torch.randn(4, 768),
         "concat": torch.randn(4, 4, 2, 3)}
    ci = g.action_free(c)
    assert torch.equal(ci["crossattn"][..., :CONTEXT_DIM], c["crossattn"][..., :CONTEXT_DIM])
    assert not bool(ci["crossattn"][..., CONTEXT_DIM:].any())
    assert ci["vector"] is c["vector"] and ci["concat"] is c["concat"]
    assert bool(c["crossattn"][..., CONTEXT_DIM:].all())           # the caller's c is not modified


def check_action_free_equals_forced_zero_actions(eng, dev):
    """ActionCFG.action_free(c) is what the conditioner makes with the action keys forced to zero, in round 0 and in a
    re-conditioned round (the session's own round inputs)."""
    from vista_b200.diffusion import ActionCFG
    from vista_b200.rollout import conditioner_recondition
    g = ActionCFG(3.0, vanilla_cfg())
    vd, z, noises = inputs(1, "action_free")
    vd = {**vd, **A}
    c, _ = eng.condition(vd, sf.T, mgc.UC_KEYS)
    _, want = eng.condition(vd, sf.T, list(ACTION_KEYS))
    got = g.action_free(c)
    assert set(got) == set(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert not torch.equal(c["crossattn"], got["crossattn"])            # the action slots were not zero to begin with
    sess = eng.rollout_session(vd, z.to(dev), force_uc_zero_embeddings=mgc.UC_KEYS)
    sess.step(A, noise=noises[0].to(dev))
    c1, _, _, _ = sess._round_inputs(B)
    _, want1 = conditioner_recondition(eng, {**vd, **B}, list(ACTION_KEYS), sess.n_cond)(1, sess._sample,
                                                                                          lambda: sess._carry)
    got1 = g.action_free(c1)
    assert all(torch.equal(got1[k], want1[k]) for k in want1)
    assert not torch.equal(got1["crossattn"], got["crossattn"])         # round 1 re-embedded the frame


def test_guider_algebra():
    """On random denoiser outputs: ActionCFG(s, VanillaCFG(s)) is VanillaCFG(s) up to fp32 rounding, action_scale 0 is
    image-only guidance towards D_img, and a Triangle image guider applies s_img per frame."""
    from vista_b200.diffusion import ActionCFG, TrianglePredictionGuider, VanillaCFG
    T = 25
    g = torch.Generator().manual_seed(3)
    du, di, dc = (torch.randn(T, 4, 6, 8, generator=g) for _ in range(3))
    sigma = torch.full((3 * T,), 4.0)
    x3 = torch.cat((du, di, dc))
    s = 2.5
    got = ActionCFG(s, vanilla_cfg(s))(x3, sigma)
    want = VanillaCFG(s)(torch.cat((du, dc)), sigma[:2 * T])
    mag = du.abs() + 2 * s * (di.abs() + dc.abs() + du.abs())
    assert bool(((got - want).abs() <= 8 * 2.0 ** -24 * mag).all())
    zero = ActionCFG(0.0, vanilla_cfg(s))(x3, sigma)
    assert torch.equal(zero, du + s * (di - du) + 0.0 * (dc - di))
    assert torch.allclose(zero, du + s * (di - du), atol=0, rtol=0)
    tri = ActionCFG(4.0, triangle_cfg(T))(x3, sigma)
    si = TrianglePredictionGuider(num_frames=T, max_scale=2.5).scale_vector(T).reshape(T, 1, 1, 1)
    assert torch.equal(tri, (du + si * (di - du)) + 4.0 * (dc - di))
    assert not torch.equal(si[0], si[T // 2])


def test_prepare_inputs_stacks_uc_action_free_c_and_c():
    from vista_b200.diffusion import ActionCFG
    g = ActionCFG(2.0, vanilla_cfg(), context_dim=3)
    T = 2
    c = {"crossattn": torch.randn(T, 1, 5), "vector": torch.randn(T, 7), "concat": torch.randn(T, 4, 2, 2)}
    uc = {k: torch.randn_like(v) for k, v in c.items()}
    x, s, m = torch.randn(T, 4, 2, 2), torch.full((T,), 3.0), torch.tensor([1.0, 0.0])
    x3, s3, cc, m3 = g.prepare_inputs(x, s, c, m, uc)
    assert torch.equal(x3, torch.cat([x] * 3)) and torch.equal(s3, torch.cat([s] * 3)) and torch.equal(m3, torch.cat([m] * 3))
    ci = c["crossattn"].clone()
    ci[..., 3:] = 0
    assert torch.equal(cc["crossattn"], torch.cat((uc["crossattn"], ci, c["crossattn"])))
    for k in ("vector", "concat"):
        assert torch.equal(cc[k], torch.cat((uc[k], c[k], c[k])))


# ------------------------------------------------------------------------------------------------------------------
# order of convergence on a closed-form denoiser with three branch means
# ------------------------------------------------------------------------------------------------------------------
S_IMG, S_ACT = 2.5, 4.0


class ActionAnalytic(tdc.Analytic):
    """tests/test_dpmpp2m_cpu.Analytic with a third mean, mu_img, for the action-free branch.  The guided D is the same
    Gaussian form with mu_g = mu_u + s_img (mu_img - mu_u) + s_act (mu_c - mu_img) (the weights sum to 1), so the ODE's
    end point is closed-form as there.  A branch's mean is its ``vector`` plus the action columns of its crossattn
    (context_dim 1): c carries mu_img and mu_c - mu_img, its action-free copy mu_img, uc mu_u and zeros."""

    def __init__(self, T, h, w, device, seed=0):
        super().__init__(T, h, w, device, seed, S_IMG)
        g = torch.Generator().manual_seed(seed + 100)
        self.mu_img = (torch.randn(T, 4, h, w, generator=g) * 0.3 + 0.3).to(device)

    def conds(self):
        T, n = self.T, 4 * self.h * self.w
        flat = lambda t: t.reshape(T, 1, n)
        z = torch.zeros(T, 1, 1, device=self.mu_u.device)
        c = {"vector": self.mu_img, "crossattn": torch.cat((z, flat(self.mu_c - self.mu_img)), 2)}
        uc = {"vector": self.mu_u, "crossattn": torch.cat((z, torch.zeros_like(flat(self.mu_u))), 2)}
        return c, uc

    def generic_denoiser(self, x, sigma, c, cond_mask):
        mu = c["vector"] + c["crossattn"][:, 0, 1:].reshape(x.shape)
        return self.denoised(x, sigma.reshape(-1, 1, 1, 1), mu)

    def error(self, out, x0, sigma0):
        assert torch.equal(out[0], self.cond_frame[0])
        mu_g = (self.mu_u + S_IMG * (self.mu_img - self.mu_u) + S_ACT * (self.mu_c - self.mu_img)).double()
        exact = mu_g + (x0.double() - mu_g) * tdc.S / math.sqrt(tdc.S * tdc.S + sigma0 * sigma0)
        return float((out[1:].double() - exact[1:]).norm() / exact[1:].norm())


def generic_errors(kind, an):
    c, uc = an.conds()
    errs = []
    for n in tdc.ORDER_STEPS:
        smp = make_sampler(kind, n, S_ACT, vanilla_cfg(S_IMG), an.noise.device.type, context_dim=1)
        x0, s0 = tdc.start_state(an, smp, n)
        out = smp(an.generic_denoiser, an.noise.clone(), c, uc=uc, cond_frame=an.cond_frame, cond_mask=an.mask)
        errs.append(an.error(out, x0, s0))
    return errs


class ActionAnalyticRuntime(tdc.AnalyticRuntime):
    """tdc.AnalyticRuntime with the image branch: a forward of T rows returns the network output of the mu_img branch."""

    def __init__(self, an: ActionAnalytic):
        super().__init__(an)
        self.out_img = torch.zeros(an.T * an.h * an.w, 8, dtype=torch.float32, device=self.dev)

    def forward(self, unet_in, c_noise, mask2, h, w):
        if c_noise.numel() == 2 * self.an.T:
            return super().forward(unet_in, c_noise, mask2, h, w)
        st = self._loop_states[(self.an.T, h, w)]
        sig = st.sigmas.index_select(0, st.step.long()).double()
        x = st.x.double()
        c_skip, c_out = 1.0 / (sig * sig + 1.0), -sig / (sig * sig + 1.0).sqrt()
        d = self.an.denoised(x, sig, self.an.mu_img.double())
        self.out_img[:, :4].copy_(((d - c_skip * x) / c_out).permute(0, 2, 3, 1).reshape(-1, 4))
        return self.out_img


def fused_errors(kind, an):
    from vista_b200.fused import fused_sample
    rt = ActionAnalyticRuntime(an)
    net = types.SimpleNamespace(diffusion_model=None, frame_sharded=False, _rt_get=lambda m, T, dev: rt)
    den = types.SimpleNamespace(network=net, denoiser=types.SimpleNamespace(num_frames=an.T))
    z = lambda *shape: torch.zeros(*shape, device=an.noise.device)
    cond = {"vector": z(an.T, 1), "crossattn": z(an.T, 1, 2), "concat": z(an.T, 4, an.h, an.w)}
    errs = []
    for n in tdc.ORDER_STEPS:
        smp = make_sampler(kind, n, S_ACT, vanilla_cfg(S_IMG), an.noise.device.type, context_dim=1)
        x0, s0 = tdc.start_state(an, smp, n)
        out = fused_sample(smp, den, an.noise.clone(), cond, cond, an.cond_frame, an.mask, None)
        errs.append(an.error(out, x0, s0))
    return errs


def test_order_of_convergence_generic_loop():
    an = ActionAnalytic(3, 4, 6, "cpu")
    tdc.check_order(generic_errors("euler", an), generic_errors("dpm", an), "action guidance, torch loop")


def test_order_of_convergence_fused_loop(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    an = ActionAnalytic(3, 4, 6, "cpu")
    with patched_action_ops():
        tdc.check_order(fused_errors("euler", an), fused_errors("dpm", an), "action guidance, fused loop (CPU twins)")


# ------------------------------------------------------------------------------------------------------------------
# the fused loop on the tiny UNet (synthetic weights: the action adapters are non-zero)
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network()


@pytest.fixture
def emulated(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    with patched_action_ops(), torch.no_grad():
        yield


FUSED_REL = 1e-2        # the 2M bar (5e-3 from the oracle for either loop) doubled: the two loops' roundings, s_act = 5


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_fused_against_torch_loop_on_tiny_unet(tiny, emulated, kind):
    """The fused loop (prepare, the 2T forward, the T-row image forward, the action update) against the torch loop
    (ActionCFG.prepare_inputs / __call__ around one 3T-row network call); and s_act moves the sample where s_act == s_img
    is the image guider alone."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)
    smp = make_sampler(kind, 3, 5.0, triangle_cfg())
    fused = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    generic = smp(lambda x, s, cc, m: den(net, x, s, cc, m), noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    r = rel_l2(fused, generic)
    image_only = with_guider(smp, kind, triangle_cfg())(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    print(f"tiny {kind} + ActionCFG(5.0), 3 steps: fused vs torch loop rel-L2 {r:.3e}; "
          f"against the image guider alone {rel_l2(fused, image_only):.3e}")
    assert r < FUSED_REL and torch.equal(fused[:1], z[:1])
    assert rel_l2(fused, image_only) > 10 * r


def test_interleaved_and_back_to_back_calls(tiny, emulated):
    """Vanilla then ActionCFG, two ActionCFG samples with different action_scale, Euler and 2M, on one loop state: each
    equals its standalone run on a fresh state."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)

    def fresh():
        net._rt_get(net.diffusion_model, 25, torch.device("cpu")).__dict__.pop("_loop_states", None)

    samplers = [tdc.make_sampler("euler", 3, guider=triangle_cfg()), make_sampler("euler", 3, 5.0, triangle_cfg()),
                make_sampler("euler", 3, 1.0, triangle_cfg()), make_sampler("dpm", 3, 5.0, triangle_cfg()),
                tdc.make_sampler("dpm", 3, guider=triangle_cfg())]
    run = lambda smp: smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    alone = []
    for smp in samplers:
        fresh()
        alone.append(run(smp))
    fresh()
    seq = [run(smp) for smp in samplers + samplers[::-1]]
    for got, want in zip(seq, alone + alone[::-1]):
        assert torch.equal(got, want)
    assert not torch.equal(alone[1], alone[2]) and not torch.equal(alone[0], alone[1])


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
def test_reference_closure_reaches_the_fused_loop(tiny, emulated, monkeypatch):
    from vista_b200 import fused as fused_mod
    cfg, sd, net, den, bden = tiny
    calls = []
    real = fused_mod.fused_sample
    monkeypatch.setattr(fused_mod, "fused_sample",
                        lambda *a, **k: (calls.append(type(a[0].guider).__name__), real(*a, **k))[1])
    model = types.SimpleNamespace(model=net, denoiser=den)

    def denoiser(x, sigma, cond, cond_mask):           # sample_utils.py:314-315, verbatim shape
        return model.denoiser(model.model, x, sigma, cond, cond_mask)
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)
    for kind in ("euler", "dpm"):
        smp = make_sampler(kind, 2, 4.0, triangle_cfg())
        out = smp(denoiser, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
        assert torch.equal(out, smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask))
    assert calls == ["ActionCFG"] * 4


def test_frame_sharded_engine_raises(tiny, emulated, monkeypatch):
    cfg, sd, net, den, bden = tiny
    monkeypatch.setattr(net, "frame_sharded", True, raising=False)
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        make_sampler("euler", 2, 4.0)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)


# ------------------------------------------------------------------------------------------------------------------
# engine paths above the sampler, on the tiny native engine (shared with tests/test_action_cfg_gpu.py)
# ------------------------------------------------------------------------------------------------------------------
def action_sampler(eng, kind="euler", action_scale=5.0, steps=None):
    """A sampler of ``kind`` with the engine's discretisation and num_steps and ActionCFG over the engine's guider."""
    return with_guider(eng.sampler, kind, action_cfg(action_scale, triangle_cfg(sf.T)), steps)


def counting_fused(monkeypatch):
    """Records the guider class of every fused_sample call."""
    from vista_b200 import fused as fused_mod
    calls = []
    real = fused_mod.fused_sample
    monkeypatch.setattr(fused_mod, "fused_sample",
                        lambda *a, **k: (calls.append(type(a[0].guider).__name__), real(*a, **k))[1])
    return calls


def check_engine_sample(eng, dev, monkeypatch):
    """engine.sample with an ActionCFG engine.sampler runs the fused loop and differs from the image guider alone."""
    vd, z, noises = inputs(1, "action_sample")
    c, uc = eng.condition({**vd, **A}, sf.T, mgc.UC_KEYS)
    calls = counting_fused(monkeypatch)
    image_only = eng.sample(c, uc=uc, N=sf.T, shape=z.shape[1:], noise=noises[0].to(dev), cond_frame=z.to(dev))
    monkeypatch.setattr(eng, "sampler", action_sampler(eng))
    out = eng.sample(c, uc=uc, N=sf.T, shape=z.shape[1:], noise=noises[0].to(dev), cond_frame=z.to(dev))
    again = eng.sample(c, uc=uc, N=sf.T, shape=z.shape[1:], noise=noises[0].to(dev), cond_frame=z.to(dev))
    assert calls == ["TrianglePredictionGuider", "ActionCFG", "ActionCFG"]
    assert torch.equal(out, again) and not torch.equal(out, image_only)


def check_session_equals_batch_rollout(eng, dev, monkeypatch, kind):
    """A session whose engine samples with ActionCFG is byte for byte engine.rollout(..., u8=True) with the same
    sampler, on the fused loop; and it repeats bit for bit."""
    from vista_b200.rollout import conditioner_recondition
    monkeypatch.setattr(eng, "sampler", action_sampler(eng, kind))
    vd, z, noises = inputs(2, "action_session")
    z, noises = z.to(dev), [n.to(dev) for n in noises]
    calls = counting_fused(monkeypatch)

    def run_session():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        return torch.cat([sess.step(None, noise=nz) for nz in noises] + [sess.close()]), sess.samples_z

    frames, samples_z = run_session()
    assert calls == ["ActionCFG"] * 2
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, 2, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                               u8=True)
    assert calls == ["ActionCFG"] * 4
    assert torch.equal(frames, want) and torch.equal(samples_z, want_z)
    frames2, samples_z2 = run_session()
    assert torch.equal(frames, frames2) and torch.equal(samples_z, samples_z2)


def check_score_leaves_the_session_untouched(eng, dev, monkeypatch):
    """The engine samples with the image guider alone; a session that scores with an ActionCFG sampler before every
    step samples the same rounds as one that never scores.  Round 0's score is sample_ensemble with that sampler."""
    vd, z, ns = inputs(2, "action_score")
    z, ns = z.to(dev), [n.to(dev) for n in ns]
    act = action_sampler(eng)
    calls = counting_fused(monkeypatch)

    def run(scoring):
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        frames, scores = [], []
        for nz in ns:
            if scoring:
                scores.append(sess.score([B, None], ensemble_size=2, num_steps=eng.sampler.num_steps, noises=ns,
                                         sampler=act))
            frames.append(sess.step(A, noise=nz))
        return torch.cat(frames + [sess.close()]), sess.samples_z, scores

    f0, z0, _ = run(False)
    f1, z1, scores = run(True)
    assert torch.equal(f0, f1) and torch.equal(z0, z1)
    assert calls.count("ActionCFG") == 2 * 2 * 2                       # 2 rounds x 2 candidates x 2 members
    rewards, members = scores[0]
    monkeypatch.setattr(eng, "sampler", act)
    reward, want = eng.sample_ensemble(*eng.condition({**vd, **B}, sf.T, mgc.UC_KEYS), z, 2, noises=ns)
    assert calls[-2:] == ["ActionCFG"] * 2                             # sample_ensemble on the fused loop
    assert torch.equal(members[0], torch.stack(want)) and torch.equal(rewards[0], reward)


@pytest.fixture(scope="module")
def eng():
    """The tiny native engine; its sampler is Euler with the Triangle guider, 3 steps."""
    e = native_engine(steps=3)
    e.en_and_decode_n_samples_a_time = 14
    return e


def test_action_free_equals_forced_zero_actions(eng, emulated):
    check_action_free_equals_forced_zero_actions(eng, torch.device("cpu"))


def test_engine_sample(eng, emulated, monkeypatch):
    check_engine_sample(eng, torch.device("cpu"), monkeypatch)


def test_session_equals_batch_rollout(eng, emulated, monkeypatch):
    check_session_equals_batch_rollout(eng, torch.device("cpu"), monkeypatch, "dpm")


def test_score_leaves_the_session_untouched(eng, emulated, monkeypatch):
    check_score_leaves_the_session_untouched(eng, torch.device("cpu"), monkeypatch)


# ------------------------------------------------------------------------------------------------------------------
# conformance of the action-guided update (the kernel in tests/test_action_cfg_gpu.py, its CPU twin here)
# ------------------------------------------------------------------------------------------------------------------
LD_IMG = 12             # the image rows' leading dimension, unlike net_out's 8: the kernel must take it from its argument


def action_inputs(case, device, seed, s_act):
    """make_sampler_inputs of the Euler conformance table plus net_img [T h w, LD_IMG] (columns 4.. NaN) and the per-frame
    s_act: "zero", "same" (= s_img, per frame) or "above" (s_img + 1.5)."""
    from test_conformance_small_cpu import make_sampler_inputs, randn
    d = make_sampler_inputs(case, device, seed=seed)
    T, hw = d["T"], d["h"] * d["w"]
    ni = randn((T * hw, LD_IMG), seed + 5, device)
    ni[:, 4:] = float("nan")
    d["net_img"] = ni
    d["action_scales"] = {"zero": torch.zeros_like(d["scales"]), "same": d["scales"].clone(),
                          "above": d["scales"] + 1.5}[s_act]
    return d


def update_action_reference(x, d, step, num_steps, coefs=None, d_prev=None):
    """fp64 action-guided step from fp32 inputs -> (x', D, bound on x', bound on D).
    D = x c_skip + c_out (u + s (i - u) + a (c - i)).  M = |x| + (1 + 2|s| + 2|a|)(c_skip |x| + |c_out| (|u| + |i| + |c|))
    bounds |x|, |D| ((1 - s) du + (s - a) di + a dc) and every intermediate.  D's roundings: c_skip 3 U24, c_out 6, du, di,
    dc 2 each, i - u, the s product, the sum, c - i, the a product and the sum 1 each: 17 U24 M; the Euler step adds 11
    (test_conformance_small_cpu.update_reference), 28 U24 M <= UPDATE_EPS M.  The 2M step as in
    test_dpmpp2m_cpu.update_2m_reference, with this M."""
    from test_conformance_small_cpu import UPDATE_EPS
    T, h, w = d["T"], d["h"], d["w"]
    hw = h * w
    s, s1 = float(d["sigmas"][step]), float(d["sigmas"][step + 1])
    c_skip, c_out = 1.0 / (s * s + 1.0), -s * (s * s + 1.0) ** -0.5
    nch = lambda t: t[:, :4].double().reshape(T, h, w, 4).permute(0, 3, 1, 2)
    u, c, i = nch(d["net"][:T * hw]), nch(d["net"][T * hw:2 * T * hw]), nch(d["net_img"])
    sc = d["scales"].double().reshape(T, 1, 1, 1)
    sa = d["action_scales"].double().reshape(T, 1, 1, 1)
    x64 = x.double()
    den = x64 * c_skip + c_out * (u + sc * (i - u) + sa * (c - i))
    mag = x64.abs() + (1 + 2 * sc.abs() + 2 * sa.abs()) * (c_skip * x64.abs() + abs(c_out) * (u.abs() + i.abs() + c.abs()))
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


def check_update_action(case, step, s_act, multistep, update, device):
    """One action-guided update at `step` of the 50-step schedule through `update` (the op or its twin), Euler or 2M.
    On 2M's first-order rows D_prev is NaN: it must not be read."""
    from test_conformance_small_cpu import NUM_STEPS, assert_elements, randn, sampler_case_id, sync
    d = action_inputs(case, device, 60 + step, s_act)
    T, h, w = d["T"], d["h"], d["w"]
    name = f"action {'2M' if multistep else 'Euler'} s_act {s_act} {sampler_case_id(case)} step {step}"
    coefs = d_prev = None
    if multistep:
        coefs = tdc.coef_table(device)
        d_prev = (torch.full_like(d["x"], float("nan")) if float(coefs[step, 3]) == 0.0
                  else randn(d["x"].shape, 95 + step, device))
    x = d["x"].clone()
    xn_ref, den_ref, bound, den_bound = update_action_reference(x, d, step, NUM_STEPS, coefs, d_prev)
    idx = torch.tensor([step], dtype=torch.int32, device=device)
    update(x, d["net"], d["net_img"], d["cond_frame"], d["mask"], d["scales"], d["action_scales"], coefs, d_prev,
           d["sigmas"], idx, NUM_STEPS, T, h, w)
    sync(device)
    assert int(idx[0]) == step + 1, f"{name}: step_idx {int(idx[0])}"
    assert bool(torch.isfinite(x).all()), f"{name}: non-finite x"
    assert_elements(x, xn_ref, bound + 2.0 ** -24 * xn_ref.abs(), f"{name}: x")
    if multistep:
        assert_elements(d_prev, den_ref, den_bound + 2.0 ** -24 * den_ref.abs(), f"{name}: D_prev")
    if step + 1 == NUM_STEPS and d["mask"] is not None:
        m = d["mask"].bool()
        assert torch.equal(x[m], d["cond_frame"][m]), f"{name}: conditioning frames not re-imposed exactly"


def check_linear_in_s_act(update, device, multistep):
    """At fixed inputs, the update's difference between two D_c is linear in s_act, the property a planner relies on
    when it raises s_act to separate candidates: with net_c2 = net_c + delta, the difference of the two results at
    s_act = k a is k times the one at a (k = 2, 4), to within the fp32 bounds of update_action_reference on the four
    results (the fp64 differences are linear exactly); at s_act = 0 the two results are bit-identical."""
    from test_conformance_small_cpu import randn, sync
    case = (25, 8, 16, "none", True, True, "triangle")
    base = action_inputs(case, device, 7, "zero")
    T, h, w = base["T"], base["h"], base["w"]
    hw = T * h * w
    net2 = base["net"].clone()
    net2[hw:2 * hw, :4] += randn((hw, 4), 8, device, 0.5)
    coefs = tdc.coef_table(device) if multistep else None
    d_prev = randn(base["x"].shape, 9, device) if multistep else None
    step = 24

    def run(net, s_act):
        d = dict(base, net=net, action_scales=torch.full_like(base["scales"], s_act))
        x = base["x"].clone()
        dp = d_prev.clone() if multistep else None
        _, _, bound, _ = update_action_reference(x, d, step, 50, coefs, d_prev)
        idx = torch.tensor([step], dtype=torch.int32, device=device)
        update(x, net, base["net_img"], None, None, base["scales"], d["action_scales"], coefs, dp, base["sigmas"], idx, 50,
               T, h, w)
        sync(device)
        return x.double(), bound + 2.0 ** -24 * x.double().abs()

    runs = {a: (run(net2, a), run(base["net"], a)) for a in (0.0, 0.5, 1.0, 2.0)}
    (x2, _), (x1, _) = runs[0.0]
    assert torch.equal(x1, x2)
    diff = {a: r2[0] - r1[0] for a, (r2, r1) in runs.items()}
    tol = {a: r2[1] + r1[1] for a, (r2, r1) in runs.items()}
    for k, a in ((2, 1.0), (4, 2.0)):
        err = (diff[a] - k * diff[0.5]).abs()
        assert bool((err <= tol[a] + k * tol[0.5]).all()), (k, a, float(err.max()))
        assert float(diff[a].abs().max()) > 100 * float((tol[a] + k * tol[0.5]).max())     # the property is not vacuous
    return diff


S_ACT_KINDS = ("zero", "same", "above")


@pytest.mark.parametrize("multistep", [False, True], ids=["euler", "2m"])
@pytest.mark.parametrize("s_act", S_ACT_KINDS)
@pytest.mark.parametrize("step", [0, 24, 49])
@pytest.mark.parametrize("case", [(25, 8, 16, "rollout", False, True, "const"), (25, 8, 16, "none", True, False, "triangle"),
                                  (3, 5, 7, "init", False, False, "const"), (1, 1, 1, "none", False, False, "triangle")],
                         ids=lambda c: "T{}x{}x{}-{}".format(*c[:4]))
def test_update_action_twin(case, step, s_act, multistep):
    import action_fake_ops
    check_update_action(case, step, s_act, multistep, action_fake_ops.sampler_update_action, torch.device("cpu"))


@pytest.mark.parametrize("multistep", [False, True], ids=["euler", "2m"])
def test_update_linear_in_s_act_twin(multistep):
    import action_fake_ops
    check_linear_in_s_act(action_fake_ops.sampler_update_action, torch.device("cpu"), multistep)
