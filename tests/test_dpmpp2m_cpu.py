"""The DPM-Solver++(2M) sampler without a GPU: its coefficient table, its order of convergence on a closed-form denoiser
through the torch loop and through the fused loop (on the CPU twins of the kernels, tests/dpm_fake_ops.py), the fused
loop against the torch loop and the oracle restatement (tests/dpm_oracle.py) on the tiny UNet, and the engine paths
above the sampler on the tiny native engine.  tests/test_dpmpp2m_gpu.py runs the kernel and the device loops."""
import math
import types

import pytest
import torch

import seam_fakes as sf
from dpm_fake_ops import patched_dpm_ops
from helpers import rel_l2, to_t, unet_weights
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs
from vista_b200 import synth

DISC = {"target": "vista_b200.diffusion.EDMDiscretization", "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}}
VANILLA = {"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 2.5}}
ORDER_STEPS = (10, 20, 25, 40, 50, 80, 160)


def make_sampler(kind, steps, device="cpu", guider=VANILLA):
    from vista_b200.diffusion import DPMPP2MSampler, EulerEDMSampler
    if kind == "euler":
        return EulerEDMSampler(num_steps=steps, device=device, s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0,
                               discretization_config=DISC, guider_config=guider)
    return DPMPP2MSampler(discretization_config=DISC, num_steps=steps, guider_config=guider, verbose=False, device=device)


def as_dpm(sampler, steps=None):
    """A DPMPP2MSampler with ``sampler``'s discretisation and guider."""
    from vista_b200.diffusion import DPMPP2MSampler
    s = DPMPP2MSampler(discretization_config=DISC, num_steps=sampler.num_steps if steps is None else steps,
                       guider_config=VANILLA, device=sampler.device)
    s.discretization, s.guider = sampler.discretization, sampler.guider
    return s


# ------------------------------------------------------------------------------------------------------------------
# coefficient table
# ------------------------------------------------------------------------------------------------------------------
def test_coefficient_table_against_the_formula():
    from vista_b200.diffusion import EDMDiscretization, dpmpp2m_coefficients
    for n in (1, 2, 10, 50):
        sig = EDMDiscretization(0.002, 700.0, 7.0)(n).to(torch.float32)
        k = dpmpp2m_coefficients(sig)
        assert k.shape == (n, 4) and k.dtype == torch.float64
        s = sig.double().tolist()
        hs = [math.log(s[i] / s[i + 1]) if s[i + 1] > 0 else math.inf for i in range(n)]
        for i in range(n):
            a, b, c, e = k[i].tolist()
            if s[i + 1] == 0.0:
                assert (a, b, c, e) == (0.0, -1.0, 1.0, 0.0), i         # x = D
                continue
            assert a == s[i + 1] / s[i] and b == math.expm1(-hs[i])
            if i == 0:
                assert (c, e) == (1.0, 0.0)
            else:
                r = hs[i - 1] / hs[i]
                assert math.isclose(c, 1 + 1 / (2 * r), rel_tol=1e-15) and math.isclose(e, 1 / (2 * r), rel_tol=1e-15)
        assert k[0, 3] == 0.0 and k[n - 1, 3] == 0.0                     # rows 0 and n - 1 are first order


def test_one_step_equals_euler():
    """One step goes from sigma_max straight to 0: both samplers return the guided D, up to the fp32 rounding of Euler's
    x + (x - D) / s (0 - s), which cancels the state x(sigma_max) of magnitude ~ 700."""
    an = Analytic(3, 4, 6, "cpu")
    outs = []
    for kind in ("euler", "dpm"):
        smp = make_sampler(kind, 1)
        x0, _ = start_state(an, smp, 1)
        outs.append(smp(an.generic_denoiser, an.noise.clone(), {"vector": an.mu_c}, uc={"vector": an.mu_u},
                        cond_frame=an.cond_frame, cond_mask=an.mask))
    assert float((outs[0] - outs[1]).abs().max()) <= 4 * 2.0 ** -24 * float(x0.abs().max())
    assert torch.equal(outs[0][0], outs[1][0])


# ------------------------------------------------------------------------------------------------------------------
# order of convergence on a closed-form denoiser
# ------------------------------------------------------------------------------------------------------------------
S = 0.5


class Analytic:
    """Data per element N(mu, S^2), with one mean per CFG half: D(x, sigma) = mu + S^2 / (S^2 + sigma^2) (x - mu).  The
    guided D is the same form with mu_g = mu_u + scale (mu_c - mu_u), so the sampling ODE has the exact solution
    x(0) = mu_g + (x(sigma_0) - mu_g) S / sqrt(S^2 + sigma_0^2).  Frame 0 is a conditioning frame."""

    def __init__(self, T, h, w, device, seed=0, scale=2.5):
        g = torch.Generator().manual_seed(seed)
        r = lambda: torch.randn(T, 4, h, w, generator=g)
        self.T, self.h, self.w, self.scale = T, h, w, scale
        self.mu_u, self.mu_c = (r() * 0.3 + 0.3).to(device), (r() * 0.3 + 0.3).to(device)
        self.noise, self.cond_frame = r().to(device), r().to(device)
        self.mask = torch.zeros(T, device=device)
        self.mask[0] = 1.0

    @staticmethod
    def denoised(x, sigma, mu):
        return mu + S * S / (S * S + sigma * sigma) * (x - mu)

    def generic_denoiser(self, x, sigma, c, cond_mask):
        return self.denoised(x, sigma.reshape(-1, 1, 1, 1), c["vector"])

    def error(self, out, x0, sigma0):
        """rel-L2 of the unconditioned frames against the exact ODE solution; the conditioning frame must come back."""
        assert torch.equal(out[0], self.cond_frame[0])
        mu_g = (self.mu_u + self.scale * (self.mu_c - self.mu_u)).double()
        exact = mu_g + (x0.double() - mu_g) * S / math.sqrt(S * S + sigma0 * sigma0)
        return float((out[1:].double() - exact[1:]).norm() / exact[1:].norm())


def start_state(an, sampler, n):
    sig0 = sampler.discretization(n, device="cpu")[0]
    x0 = an.noise.clone()
    x0 *= torch.sqrt(1.0 + sig0 ** 2).to(x0.device)
    return x0, float(sig0)


def generic_errors(kind, an):
    errs = []
    for n in ORDER_STEPS:
        smp = make_sampler(kind, n, an.noise.device.type)
        x0, s0 = start_state(an, smp, n)
        out = smp(an.generic_denoiser, an.noise.clone(), {"vector": an.mu_c}, uc={"vector": an.mu_u},
                  cond_frame=an.cond_frame, cond_mask=an.mask)
        errs.append(an.error(out, x0, s0))
    return errs


class AnalyticRuntime:
    """Stands in for the UNet runtime of the fused loop: returns the network output whose preconditioned value
    net c_out + x c_skip is the closed-form D of each CFG half, from the loop's fp32 state (not from the fp16 UNet
    input, whose rounding would hide the order).  Only device tensor ops, so a CUDA graph can capture it."""

    def __init__(self, an: Analytic):
        self.an, self.dev = an, an.noise.device
        self.out = torch.zeros(2 * an.T * an.h * an.w, 8, dtype=torch.float32, device=self.dev)

    def set_conditioning(self, context, y):
        pass

    def forward(self, unet_in, c_noise, mask2, h, w):
        st = self._loop_states[(self.an.T, h, w)]
        sig = st.sigmas.index_select(0, st.step.long()).double()
        x = st.x.double()
        c_skip, c_out = 1.0 / (sig * sig + 1.0), -sig / (sig * sig + 1.0).sqrt()
        rows = [((self.an.denoised(x, sig, mu.double()) - c_skip * x) / c_out).permute(0, 2, 3, 1).reshape(-1, 4)
                for mu in (self.an.mu_u, self.an.mu_c)]
        self.out[:, :4].copy_(torch.cat(rows))
        return self.out


def analytic_denoiser(an: Analytic):
    """A B200Denoiser look-alike whose network hands fused_sample an AnalyticRuntime."""
    rt = AnalyticRuntime(an)
    net = types.SimpleNamespace(diffusion_model=None, frame_sharded=False, _rt_get=lambda m, T, dev: rt)
    return types.SimpleNamespace(network=net, denoiser=types.SimpleNamespace(num_frames=an.T))


def fused_errors(kind, an):
    from vista_b200.fused import fused_sample
    den = analytic_denoiser(an)
    z = lambda *shape: torch.zeros(*shape, device=an.noise.device)
    cond = {"vector": z(an.T, 1), "crossattn": z(an.T, 1, 1), "concat": z(an.T, 4, an.h, an.w)}
    errs = []
    for n in ORDER_STEPS:
        smp = make_sampler(kind, n, an.noise.device.type)
        x0, s0 = start_state(an, smp, n)
        out = fused_sample(smp, den, an.noise.clone(), cond, cond, an.cond_frame, an.mask, None)
        errs.append(an.error(out, x0, s0))
    return errs


def check_order(errs_euler, errs_dpm, name):
    """Second order for 2M, first order for Euler: the error ratio from 40 to 160 steps, and 2M below Euler at every
    step count up to 80."""
    i40, i160 = ORDER_STEPS.index(40), ORDER_STEPS.index(160)
    print(f"{name}: steps {ORDER_STEPS}\n  euler {['%.2e' % e for e in errs_euler]}\n  2M    {['%.2e' % e for e in errs_dpm]}")
    assert errs_dpm[i40] / errs_dpm[i160] >= 12.0, errs_dpm
    assert 3.5 <= errs_euler[i40] / errs_euler[i160] <= 4.5, errs_euler
    for n, ee, ed in zip(ORDER_STEPS, errs_euler, errs_dpm):
        if n <= 80:
            assert ed < ee, (n, ed, ee)


def test_order_of_convergence_generic_loop():
    an = Analytic(3, 4, 6, "cpu")
    check_order(generic_errors("euler", an), generic_errors("dpm", an), "torch loop")


def test_order_of_convergence_fused_loop(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    an = Analytic(3, 4, 6, "cpu")
    with patched_dpm_ops():
        check_order(fused_errors("euler", an), fused_errors("dpm", an), "fused loop (CPU twins)")


# ------------------------------------------------------------------------------------------------------------------
# the fused loop on the tiny UNet
# ------------------------------------------------------------------------------------------------------------------
def tiny_network(device="cpu"):
    from vista_b200.diffusion import B200Denoiser, Denoiser
    from vista_b200.modules import B200Wrapper, VideoUNet
    cfg, sd = unet_weights("tiny")
    with torch.device(device):
        unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                         num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                         channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                         context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                         use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                         use_linear_in_transformer=True, action_control=True)
    unet.load_state_dict(to_t(sd), strict=True)
    net = B200Wrapper(unet)
    if device == "cpu":
        net._require_cuda = unet._require_cuda = lambda dev: None
    den = Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=25)
    return cfg, sd, net, den, B200Denoiser(den, net)


def tiny_inputs(cfg, device="cpu", n_cond=1, seed=7):
    c, uc = synth.synth_conditioning(seed, 25, 8, 16, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
    noise, z, mask = synth.synth_latents(seed, 25, 8, 16)
    mask[:n_cond] = 1.0
    return (to_t(c, device), to_t(uc, device), torch.from_numpy(noise).to(device), torch.from_numpy(z).to(device),
            torch.from_numpy(mask).to(device))


@pytest.fixture(scope="module")
def tiny():
    return tiny_network()


@pytest.fixture
def emulated(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    with patched_dpm_ops(), torch.no_grad():
        yield


def test_fused_against_torch_loop_and_oracle_on_tiny_unet(tiny, emulated):
    from dpm_oracle import dpmpp2m_sample
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tiny_inputs(cfg)
    smp = make_sampler("dpm", 4)
    fused = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    generic = smp(lambda x, s, cc, m: den(net, x, s, cc, m), noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    ref = dpmpp2m_sample(to_t(sd), cfg, noise, c, uc, z, mask, 4, 25)
    rf, rg = rel_l2(fused, ref), rel_l2(generic, ref)
    print(f"tiny 2M, 4 steps: fused {rf:.3e}, torch loop {rg:.3e} rel-L2 from the oracle")
    assert rf < 5e-3 and rg < 5e-3
    assert torch.equal(fused[:1], z[:1])
    euler = make_sampler("euler", 4)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    assert rel_l2(euler, fused) > 10 * rf            # the two samplers are told apart by the check above


def test_interleaved_and_back_to_back_calls(tiny, emulated):
    """Euler and 2M calls at the same num_steps on one loop state, interleaved, each equal their standalone run; a 2M
    sample after another one equals the same sample on a fresh loop state, so nothing of D_prev carries over."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tiny_inputs(cfg)
    c2, uc2, noise2, z2, mask2 = tiny_inputs(cfg, n_cond=3, seed=8)
    euler, dpm = make_sampler("euler", 3), make_sampler("dpm", 3)

    def fresh():
        net._rt_get(net.diffusion_model, 25, torch.device("cpu")).__dict__.pop("_loop_states", None)

    run = lambda smp, nz, cc, u, zz, m: smp(bden, nz.clone(), cc, uc=u, cond_frame=zz, cond_mask=m)
    fresh()
    alone_e = run(euler, noise, c, uc, z, mask)
    fresh()
    alone_d = run(dpm, noise, c, uc, z, mask)
    fresh()
    alone_d2 = run(dpm, noise2, c2, uc2, z2, mask2)
    fresh()
    seq = [run(euler, noise, c, uc, z, mask), run(dpm, noise, c, uc, z, mask), run(euler, noise, c, uc, z, mask),
           run(dpm, noise, c, uc, z, mask), run(dpm, noise2, c2, uc2, z2, mask2)]
    assert not torch.equal(alone_e, alone_d)
    for got, want in zip(seq, [alone_e, alone_d, alone_e, alone_d, alone_d2]):
        assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
def test_reference_closure_reaches_the_fused_loop(tiny, emulated, monkeypatch):
    from vista_b200 import fused as fused_mod
    cfg, sd, net, den, bden = tiny
    calls = []
    real = fused_mod.fused_sample
    monkeypatch.setattr(fused_mod, "fused_sample", lambda *a, **k: (calls.append(type(a[0]).__name__), real(*a, **k))[1])
    model = types.SimpleNamespace(model=net, denoiser=den)

    def denoiser(x, sigma, cond, cond_mask):           # sample_utils.py:314-315, verbatim shape
        return model.denoiser(model.model, x, sigma, cond, cond_mask)
    c, uc, noise, z, mask = tiny_inputs(cfg)
    smp = make_sampler("dpm", 2)
    out = smp(denoiser, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    assert calls == ["DPMPP2MSampler"]
    assert torch.equal(out, smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask))


def test_frame_sharded_engine_raises(tiny, emulated, monkeypatch):
    cfg, sd, net, den, bden = tiny
    monkeypatch.setattr(net, "frame_sharded", True, raising=False)
    c, uc, noise, z, mask = tiny_inputs(cfg)
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        make_sampler("dpm", 2)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)


# ------------------------------------------------------------------------------------------------------------------
# engine paths above the sampler, on the tiny native engine
# ------------------------------------------------------------------------------------------------------------------
A = {"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}
B = {"trajectory": torch.tensor([-0.35, 2.41, -1.02, 4.66, -1.93, 6.74, -3.05, 8.62])}


@pytest.fixture(scope="module")
def eng():
    """The tiny native engine; its sampler is Euler (the config's), 3 steps."""
    e = native_engine(steps=3)
    e.en_and_decode_n_samples_a_time = 14
    return e


def session(eng, vd, z):
    return eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)


def test_session_equals_batch_rollout(eng, emulated, monkeypatch):
    """A session whose engine samples with 2M is byte for byte engine.rollout(..., u8=True) with the same sampler."""
    from vista_b200.rollout import conditioner_recondition
    monkeypatch.setattr(eng, "sampler", as_dpm(eng.sampler))
    vd, z, noises = inputs(2, "dpm_session")
    sess = session(eng, vd, z)
    frames = torch.cat([sess.step(None, noise=nz) for nz in noises] + [sess.close()])
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, 2, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                               u8=True)
    assert torch.equal(frames, want) and torch.equal(sess.samples_z, want_z)


def test_score_with_2m_leaves_the_session_untouched(eng, emulated, monkeypatch):
    """The engine samples with Euler; a session that scores with 2M at the engine's num_steps before every step samples
    the same rounds as one that never scores.  Round 0's 2M score is sample_ensemble with the 2M sampler."""
    vd, z, ns = inputs(2, "dpm_score")
    euler, dpm = eng.sampler, as_dpm(eng.sampler)

    def run(scoring):
        sess = session(eng, vd, z)
        frames, scores = [], []
        for nz in ns:
            if scoring:
                scores.append(sess.score([B, None], ensemble_size=2, num_steps=euler.num_steps, noises=ns, sampler=dpm))
            frames.append(sess.step(A, noise=nz))
        return torch.cat(frames + [sess.close()]), sess.samples_z, scores

    f0, z0, _ = run(False)
    f1, z1, scores = run(True)
    assert torch.equal(f0, f1) and torch.equal(z0, z1)
    rewards, members = scores[0]
    monkeypatch.setattr(eng, "sampler", dpm)
    reward, want = eng.sample_ensemble(*eng.condition({**vd, **B}, sf.T, mgc.UC_KEYS), z, 2, noises=ns)
    assert torch.equal(members[0], torch.stack(want)) and torch.equal(rewards[0], reward)


# ------------------------------------------------------------------------------------------------------------------
# conformance of the 2M update (the kernel in tests/test_dpmpp2m_gpu.py, its CPU twin here)
# ------------------------------------------------------------------------------------------------------------------
def coef_table(device, n=None):
    """The fp32 table the fused loop uploads for the conformance schedule (50 steps, sigma 700 -> 0.002 -> 0)."""
    from test_conformance_small_cpu import NUM_STEPS, edm_sigmas
    from vista_b200.diffusion import dpmpp2m_coefficients
    n = NUM_STEPS if n is None else n
    return dpmpp2m_coefficients(edm_sigmas(n)).to(torch.float32).to(device)


def update_2m_reference(x, d, step, coefs, d_prev, num_steps):
    """fp64 2M step from fp32 inputs and the fp32 coefficient row the kernel reads -> (x', D, bound on x', bound on D).
    D and its bound (UPDATE_EPS * M, with test_conformance_small_cpu.update_reference's M, which also bounds |x| and |D|)
    are the Euler update's.  Then c D, e D_prev, their difference, a x, b (.) and the final difference are 6 more
    roundings, against (|a| |x| + |b| ((|c| + |e|) M + |e| |D_prev|)); D's own error reaches x' times |b| (|c| + |e|)."""
    from test_conformance_small_cpu import UPDATE_EPS
    T, h, w = d["T"], d["h"], d["w"]
    hw = h * w
    s = float(d["sigmas"][step])
    c_skip, c_out = 1.0 / (s * s + 1.0), -s * (s * s + 1.0) ** -0.5
    nch = lambda t: t[:, :4].double().reshape(T, h, w, 4).permute(0, 3, 1, 2)
    u, c = nch(d["net"][:T * hw]), nch(d["net"][T * hw:2 * T * hw])
    sc = d["scales"].double().reshape(T, 1, 1, 1)
    x64 = x.double()
    den = x64 * c_skip + c_out * (u + sc * (c - u))
    mag = x64.abs() + (1 + 2 * sc.abs()) * (c_skip * x64.abs() + abs(c_out) * (u.abs() + c.abs()))
    ka, kb, kc, ke = (float(v) for v in coefs[step].double())
    dp = torch.zeros_like(x64) if ke == 0.0 else d_prev.double()
    xn = ka * x64 - kb * (kc * den - ke * dp)
    bound = UPDATE_EPS * (abs(ka) * x64.abs() + abs(kb) * ((abs(kc) + abs(ke)) * mag + abs(ke) * dp.abs()))
    if step + 1 == num_steps and d["mask"] is not None:
        m = d["mask"].double().reshape(T, 1, 1, 1)
        xn = xn * (1 - m) + d["cond_frame"].double() * m
        bound = bound * (1 - m)
    return xn, den, bound, UPDATE_EPS * mag


def check_update_2m(case, step, update, device):
    """One 2M update at `step` of the 50-step schedule through `update` (the op or its twin).  D_prev is NaN on the
    first-order rows (step 0 and the step to sigma = 0), where it must not be read, and random elsewhere."""
    from test_conformance_small_cpu import NUM_STEPS, assert_elements, make_sampler_inputs, randn, sampler_case_id, sync
    d = make_sampler_inputs(case, device, seed=40 + step)
    T, h, w = d["T"], d["h"], d["w"]
    name = f"2M {sampler_case_id(case)} step {step}"
    coefs = coef_table(device)
    first_order = float(coefs[step, 3]) == 0.0
    d_prev = torch.full_like(d["x"], float("nan")) if first_order else randn(d["x"].shape, 90 + step, device)
    x = d["x"].clone()
    xn_ref, den_ref, bound, den_bound = update_2m_reference(x, d, step, coefs, d_prev, NUM_STEPS)
    idx = torch.tensor([step], dtype=torch.int32, device=device)
    update(x, d["net"], d["cond_frame"], d["mask"], d["scales"], coefs, d_prev, d["sigmas"], idx, NUM_STEPS, T, h, w)
    sync(device)
    assert int(idx[0]) == step + 1, f"{name}: step_idx {int(idx[0])}"
    assert bool(torch.isfinite(x).all()), f"{name}: non-finite x (D_prev read on a first-order row?)"
    assert_elements(x, xn_ref, bound + 2.0 ** -24 * xn_ref.abs(), f"{name}: x")
    assert_elements(d_prev, den_ref, den_bound + 2.0 ** -24 * den_ref.abs(), f"{name}: D_prev")
    if step + 1 == NUM_STEPS and d["mask"] is not None:
        m = d["mask"].bool()
        assert torch.equal(x[m], d["cond_frame"][m]), f"{name}: conditioning frames not re-imposed exactly"


def trajectory_2m_reference(d, coefs, num_steps):
    """num_steps fp64 prepare -> 2M update steps with the fixed network output (the masked frames re-imposed first)."""
    T = d["T"]
    x = d["x"].double()
    m = d["mask"].double().reshape(T, 1, 1, 1)
    cf = d["cond_frame"].double()
    dp = None
    for k in range(num_steps):
        x = x * (1 - m) + cf * m
        xn, den, _, _ = update_2m_reference(x, d, k, coefs, torch.zeros_like(x) if dp is None else dp, num_steps)
        x, dp = xn, den
    return x


def run_trajectory_2m(d, prepare, update, coefs, num_steps):
    T, h, w = d["T"], d["h"], d["w"]
    x = d["x"].clone()
    d_prev = torch.full_like(x, float("nan"))
    idx = torch.zeros(1, dtype=torch.int32, device=x.device)
    for _ in range(num_steps):
        prepare(x, d["cond_frame"], d["mask"], d["concat_u"], d["concat_c"], d["sigmas"], idx, d["unet_in"], d["c_noise"],
                T, h, w)
        update(x, d["net"], d["cond_frame"], d["mask"], d["scales"], coefs, d_prev, d["sigmas"], idx, num_steps, T, h, w)
    return x, idx


TRAJ_REL = 1e-5         # 50 steps of a few fp32 roundings each, none amplified (|a|, |b| <= 1)


@pytest.mark.parametrize("step", [0, 1, 24, 49])
@pytest.mark.parametrize("case", [(25, 8, 16, "rollout", False, True, "const"), (25, 8, 16, "none", True, False, "triangle"),
                                  (3, 5, 7, "init", False, False, "const"), (1, 1, 1, "none", False, False, "triangle")],
                         ids=lambda c: "T{}x{}x{}-{}".format(*c[:4]))
def test_update_2m_twin(case, step):
    import dpm_fake_ops
    check_update_2m(case, step, dpm_fake_ops.sampler_update_2m, torch.device("cpu"))


def test_trajectory_2m_twin():
    import dpm_fake_ops
    import fake_ops
    from test_conformance_small_cpu import NUM_STEPS, trajectory_inputs
    d = trajectory_inputs(25, 8, 16, torch.device("cpu"))
    coefs = coef_table("cpu")
    x, idx = run_trajectory_2m(d, fake_ops.sampler_prepare, dpm_fake_ops.sampler_update_2m, coefs, NUM_STEPS)
    ref = trajectory_2m_reference(d, coefs, NUM_STEPS)
    assert int(idx[0]) == NUM_STEPS and rel_l2(x, ref) <= TRAJ_REL, rel_l2(x, ref)
