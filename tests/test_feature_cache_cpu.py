"""Feature caching (``cache_interval`` / ``cache_branch`` of the samplers, ``UNetRuntime.forward(..., cached=True)``)
without a GPU: the schedule rule on hand-built kind sequences, the argument errors and the loops that refuse to cache,
the oracle's cached forward against the real VideoUNet run with a hook that hands back the recorded feature
(tests/golden/unet_cached_*.npz), and the fused loop on the CPU twins of the kernels (tests/interval_fake_ops.py): a
cached forward launches a subsequence of the full forward's launches and touches only the outermost blocks, it is
bit-equal to the full forward on the same inputs, and cached samples follow the oracle loop (tests/cache_oracle.py)
with the same schedule for Euler and 2M over VanillaCFG, Triangle, ActionCFG and IntervalCFG.  The check functions
take a device; tests/test_feature_cache_gpu.py runs them on the H100."""
import pytest
import torch

import seam_fakes as sf
import test_action_cfg_cpu as tac
import test_dpmpp2m_cpu as tdc
import test_interval_cfg_cpu as tic
import cache_oracle as co
from cache_oracle import oracle_sample
from helpers import golden, rel_l2, to_t, unet_weights
from interval_fake_ops import patched_interval_ops
from oracle import make_golden_cond as mgc
from oracle import vista_oracle as vo
from oracle.make_golden_cached import UNET_CACHED_CASES, unet_cached_inputs
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs

STEPS = 6
T = 25
FORWARD_REL = 5e-3        # a cached forward of fp16 kernels against the fp32 oracle's, as for the full forward
# the fused loop (fp16 network) against the fp32 oracle loop over 6 steps, for the samplers and guiders of CASES:
# measured at up to 2.4e-3 (2M under IntervalCFG(ActionCFG)) on the H100 and on the CPU twins, 1.4e-3 for Euler
SAMPLE_REL = 5e-3


def guider(name):
    tri = tac.triangle_cfg(T)
    return {"vanilla": tac.vanilla_cfg(), "triangle": tri, "action": tac.action_cfg(5.0, tri),
            # guided on steps 1..3 of 6: kinds u g g g u u, full steps 0 1 3 4 at interval 2
            "interval": tic.interval_over(STEPS, 1, 3, tac.action_cfg(5.0, tri))}[name]


def make(kind, guider_config, interval=2, branch=1, steps=STEPS, device="cpu"):
    """An Euler or 2M sampler ("euler" / "dpm") with feature caching set through its keywords."""
    from vista_b200.diffusion import DPMPP2MSampler, EulerEDMSampler
    kw = dict(discretization_config=tdc.DISC, num_steps=steps, guider_config=guider_config, device=device,
              cache_interval=interval, cache_branch=branch)
    if kind == "euler":
        return EulerEDMSampler(s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, **kw)
    return DPMPP2MSampler(**kw)


# ------------------------------------------------------------------------------------------------------------------
# the schedule and the arguments
# ------------------------------------------------------------------------------------------------------------------
def test_cache_schedule():
    from vista_b200.diffusion import cache_schedule
    G, U = True, False
    assert cache_schedule([G] * 7, 3) == [True, False, False, True, False, False, True]
    assert cache_schedule([G] * 7, 1) == [True] * 7
    assert cache_schedule([G] * 5, 2) == [True, False, True, False, True]
    assert cache_schedule([G] * 4, 5) == [True, False, False, False]          # an interval beyond the schedule
    assert cache_schedule([G] * 4, 99) == [True, False, False, False]
    assert cache_schedule([U] * 3, 2) == [True, False, True]
    # a kind change is full and restarts the count
    assert cache_schedule([U, G, G, G, U, U], 2) == [True, True, False, True, True, False]
    assert cache_schedule([G, G, U, U, U, U, U], 3) == [True, False, True, False, False, True, False]
    assert cache_schedule([G, U, G, U], 4) == [True] * 4
    assert cache_schedule([], 3) == []
    for bad in (0, -1, 1.5, True, "2", None):
        with pytest.raises(ValueError, match="cache_interval"):
            cache_schedule([G, G], bad)


def test_sampler_arguments():
    from vista_b200.diffusion import instantiate_from_config
    for kind in ("euler", "dpm"):
        plain = tdc.make_sampler(kind, 4)
        assert (plain.cache_interval, plain.cache_branch) == (1, 0)
        s = make(kind, tac.vanilla_cfg(), interval=3, branch=2)
        assert (s.cache_interval, s.cache_branch) == (3, 2)
        for interval, branch, name in ((0, 0, "cache_interval"), (-2, 0, "cache_interval"), (2.0, 0, "cache_interval"),
                                       (True, 0, "cache_interval"), (2, -1, "cache_branch"), (2, 1.0, "cache_branch"),
                                       (2, False, "cache_branch"), (None, 0, "cache_interval")):
            with pytest.raises(ValueError, match=name):
                make(kind, tac.vanilla_cfg(), interval=interval, branch=branch)
    target = {"euler": "vista_b200.diffusion.EulerEDMSampler", "dpm": "vista_b200.diffusion.DPMPP2MSampler"}
    for kind, t in target.items():
        s = instantiate_from_config({"target": t, "params": {"discretization_config": tdc.DISC, "num_steps": 5,
                                                            "guider_config": tac.vanilla_cfg(), "cache_interval": 2,
                                                            "cache_branch": 1}})
        assert (s.cache_interval, s.cache_branch) == (2, 1)


@pytest.fixture(scope="module")
def tiny():
    return tdc.tiny_network()


@pytest.fixture
def emulated(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    with patched_interval_ops(), torch.no_grad():
        yield


def test_loops_that_do_not_cache_refuse(tiny, emulated, monkeypatch):
    """cache_interval > 1 raises NotImplementedError on the torch loop, with s_churn > 0 and on a frame-sharded engine,
    before the latent is touched; cache_interval 1 runs there as before.  A branch beyond the UNet is a ValueError."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg)
    generic = lambda x, s, cc, m: den(net, x, s, cc, m)
    for kind in ("euler", "dpm"):
        x = noise.clone()
        with pytest.raises(NotImplementedError, match="torch loop"):
            make(kind, tac.vanilla_cfg(), steps=2)(generic, x, c, uc=uc, cond_frame=z, cond_mask=mask)
        assert torch.equal(x, noise)
        make(kind, tac.vanilla_cfg(), interval=1, steps=2)(generic, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
        x = noise.clone()
        with pytest.raises(ValueError, match="cache_branch"):
            make(kind, tac.vanilla_cfg(), branch=4, steps=2)(bden, x, c, uc=uc, cond_frame=z, cond_mask=mask)
        assert torch.equal(x, noise)
    churn = make("euler", tac.vanilla_cfg(), steps=2)
    churn.s_churn = 0.5
    with pytest.raises(NotImplementedError, match="s_churn"):
        churn(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    monkeypatch.setattr(net, "frame_sharded", True, raising=False)
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        make("euler", tac.vanilla_cfg(), steps=2)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)


# ------------------------------------------------------------------------------------------------------------------
# the oracle's cached forward against the real VideoUNet (fixtures by oracle/make_golden_cached.py)
# ------------------------------------------------------------------------------------------------------------------
def scaled(x, sigma):
    """(x c_in, c_noise) of the VScalingWithEDMcNoise denoiser at one sigma for every row."""
    s = torch.full((x.shape[0],), float(sigma), dtype=torch.float32, device=x.device)
    c_skip, c_out, c_in, c_noise = vo.vscaling_edm_cnoise(s[:, None, None, None])
    return x * c_in, c_noise.reshape(-1)


@pytest.mark.parametrize("name", list(UNET_CACHED_CASES))
def test_oracle_cached_forward_matches_reference(name):
    from vista_b200 import synth
    preset, h, w, frames, branches, keep_full = UNET_CACHED_CASES[name]
    g = golden(name)
    cfg, sd = unet_weights(preset)
    assert synth.state_dict_checksum(sd) == str(g["weight_checksum"])
    x0, s0, x1, s1, cc, mask2 = unet_cached_inputs(cfg, h, w, frames)
    assert synth.checksum([x0, x1, mask2] + [cc[k] for k in sorted(cc)]) == str(g["input_checksum"])
    assert list(g["branches"]) == list(branches)
    sdt, cct, m2 = to_t(sd), to_t(cc), torch.from_numpy(mask2)
    run = lambda x, s, cache=None: co.wrapper_forward(sdt, cfg, *scaled(torch.from_numpy(x), s), cct, m2, frames, cache)
    with torch.no_grad():
        for b in branches:
            cache = {"branch": b}
            full0 = run(x0, s0, cache)
            if keep_full:
                assert rel_l2(full0, torch.from_numpy(g["full0"])) < 2e-5
            out = run(x1, s1, cache)
            ref = torch.from_numpy(g[f"cached_b{b}"])
            r = rel_l2(out, ref)
            print(f"{name} branch {b}: oracle cached forward {r:.2e} rel-L2 from the reference")
            assert r < 2e-5, (b, r)
            if keep_full:
                assert rel_l2(ref, torch.from_numpy(g["full1"])) > 1e-2       # the cache changed the output


def test_cached_oracle_restates_the_oracle():
    """Without a cache, and on the full call that records one, tests/cache_oracle.py's forward is vo.wrapper_forward
    operation for operation: torch.equal on the tiny fixture's inputs."""
    cfg, sd = unet_weights("tiny")
    x0, s0, x1, s1, cc, mask2 = unet_cached_inputs(cfg, 8, 16, T)
    sdt, cct, m2 = to_t(sd), to_t(cc), torch.from_numpy(mask2)
    xs, t = scaled(torch.from_numpy(x0), s0)
    with torch.no_grad():
        want = vo.wrapper_forward(sdt, cfg, xs, t, cct, m2, T)
        assert torch.equal(co.wrapper_forward(sdt, cfg, xs, t, cct, m2, T), want)
        for b in (0, 1, 3):
            cache = {"branch": b}
            assert torch.equal(co.wrapper_forward(sdt, cfg, xs, t, cct, m2, T, cache), want) and "h" in cache


# ------------------------------------------------------------------------------------------------------------------
# the runtime's cached forward (shared with the GPU file)
# ------------------------------------------------------------------------------------------------------------------
def rt_forward(rt, x_in, t, mask, h, w, slot="", **cache):
    """UNetRuntime.forward on NCHW (x c_in | concat) rows through zero-padded token rows, as the fused loop feeds it
    -> an NCHW fp32 copy of the network output."""
    from vista_b200 import ops
    from vista_b200.unet import padded_input_rows
    B = x_in.shape[0]
    tok = padded_input_rows(B * h * w, x_in.device)
    ops.nchw_to_tokens(x_in.float().contiguous(), tok, B, x_in.shape[1], h, w)
    out = rt.forward(tok, t.contiguous(), mask.contiguous(), h, w, slot=slot, **cache)
    res = torch.empty(B, rt.cfg.out_channels, h, w, dtype=torch.float32, device=x_in.device)
    ops.tokens_to_nchw(out, res, B, rt.cfg.out_channels, h, w)
    return res


def forward_problem(cfg, h, w, dev):
    """The fixture's inputs on ``dev``: per x, the network input (x c_in | concat) and c_noise of its 2T rows, and the
    2T-row conditioning -> (inputs of x0, inputs of x1, context, y, mask)."""
    x0, s0, x1, s1, cc, mask2 = unet_cached_inputs(cfg, h, w, T)
    cct = to_t(cc, dev)
    cat = lambda x, s: (lambda xs, t: (torch.cat((xs, cct["concat"]), 1), t))(*scaled(torch.from_numpy(x).to(dev), s))
    return cat(x0, s0), cat(x1, s1), cct["crossattn"], cct["vector"], torch.from_numpy(mask2).to(dev)


ROW_SETS = (("2T", slice(0, 2 * T), ""), ("T", slice(T, 2 * T), ""), ("T cond slot", slice(T, 2 * T), "cond"))


def check_same_input_equality(rt, problem, h, w, branches):
    """For the 2T rows, the T rows and the T rows of the "cond" slot (each conditioned on its own rows): a full forward,
    then a cached forward of every branch on the same x, sigma and conditioning, torch.equal to it."""
    (xin, t), _, ctx, y, mask = problem
    for name, rows, slot in ROW_SETS:
        ctx_r = ctx[rows] if slot == "" else ctx[:T]            # the slot holds another conditioning of T rows
        rt.set_conditioning(ctx_r, y[rows] if slot == "" else y[:T], slot=slot)
        run = lambda **cache: rt_forward(rt, xin[rows], t[rows], mask[rows], h, w, slot=slot, **cache)
        for b in branches:
            full = run()
            cached = run(cached=True, cache_branch=b)
            assert torch.equal(full, cached), f"{name}: branch {b} cached forward differs from the full forward"


def check_cached_against(rt, problem, h, w, branches, reference, bound=FORWARD_REL, rows=slice(0, 2 * T)):
    """A full forward at x0 then a cached forward at x1 (same conditioning), against ``reference(b)`` -> rel-L2s."""
    (x0, t0), (x1, t1), ctx, y, mask = problem
    rt.set_conditioning(ctx[rows], y[rows])
    errs = {}
    for b in branches:
        rt_forward(rt, x0[rows], t0[rows], mask[rows], h, w)
        out = rt_forward(rt, x1[rows], t1[rows], mask[rows], h, w, cached=True, cache_branch=b)
        ref = reference(b)
        errs[b] = rel_l2(out.cpu(), ref.cpu())
        print(f"cached forward, branch {b}: {errs[b]:.2e} rel-L2 from the fp32 reference")
        assert errs[b] <= bound, (b, errs[b])
    return errs


class Recorder:
    """Per forward: the layer prefixes the runtime looked up and the outputs (pointer, shape) of its GEMM launches."""

    def __init__(self, rt, monkeypatch):
        from vista_b200 import ops
        self.prefixes, self.gemms = set(), []
        rec = self

        class Layers(dict):
            def __getitem__(self, k):
                rec.prefixes.add(k)
                return dict.__getitem__(self, k)
        monkeypatch.setattr(rt, "layers", Layers(rt.layers))
        real = ops.gemm
        monkeypatch.setattr(ops, "gemm", lambda a, w, out, **k: (self.gemms.append((out.data_ptr(), tuple(out.shape))),
                                                                  real(a, w, out, **k))[1])

    def take(self):
        got = self.prefixes, self.gemms
        self.prefixes, self.gemms = set(), []
        return got


def is_subsequence(sub, seq):
    it = iter(seq)
    return all(any(s == v for v in it) for s in sub)


def block_size(plan, b, h, w):
    """(h, w) of input block b's output, the spatial size of output block n-1-b."""
    from vista_b200.spec import ConvSpec
    for blk in plan.input_blocks[:b + 1]:
        if isinstance(blk.layers[0], ConvSpec) and blk.layers[0].kind == "down":
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return h, w


def check_cached_launches(rt, problem, h, w, monkeypatch):
    """A cached forward of branch b looks up the layers of input blocks 0..b and output blocks n-1-b.. only, its GEMM
    launches are a subsequence of the full forward's, and it leaves the h half of cat{n-1-b} and its GroupNorm
    partials as the full forward wrote them."""
    (x0, t0), (x1, t1), ctx, y, mask = problem
    plan = rt.plan
    n = len(plan.output_blocks)
    rt.set_conditioning(ctx, y)
    rec = Recorder(rt, monkeypatch)
    for b in range(len(plan.input_blocks)):
        rt_forward(rt, x0, t0, mask, h, w)
        full_prefixes, full_gemms = rec.take()
        assert full_prefixes == set(rt.layers.keys())
        j = n - 1 - b
        hb, wb = block_size(plan, b, h, w)
        cat = next(v for k, v in rt._bufs.items() if k[0] == f"cat{j}" and k[1] == x0.shape[0] * hb * wb)
        part = [v for k, v in rt._bufs.items() if k[0] == f"part.cat{j}" and k[1] == cat.shape[0]]
        ch = cat.shape[1] - plan.skip_channels[b]
        kept = cat[:, :ch].clone(), [p[:, :ch].clone() for p in part]
        rt_forward(rt, x1, t1, mask, h, w, cached=True, cache_branch=b)
        prefixes, gemms = rec.take()
        want = {l.prefix for blk in plan.input_blocks[:b + 1] + plan.output_blocks[j:] for l in blk.layers}
        assert prefixes == want, (b, sorted(prefixes ^ want))
        assert is_subsequence(gemms, full_gemms) and len(gemms) < len(full_gemms), b
        assert torch.equal(cat[:, :ch], kept[0]) and all(torch.equal(p[:, :ch], q) for p, q in zip(part, kept[1]))
    return rec


def runtime(cfg, sd, dev):
    from vista_b200.unet import UNetRuntime
    return UNetRuntime(cfg, to_t(sd, dev), dev, T)


@pytest.fixture(scope="module")
def tiny_rt():
    cfg, sd = unet_weights("tiny")
    return cfg, runtime(cfg, sd, "cpu")


def test_cached_forward_same_input_equality(tiny_rt, emulated):
    cfg, rt = tiny_rt
    check_same_input_equality(rt, forward_problem(cfg, 8, 16, "cpu"), 8, 16, (0, 1, 3))


def test_cached_forward_against_reference(tiny_rt, emulated):
    cfg, rt = tiny_rt
    g = golden("unet_cached_tiny")
    check_cached_against(rt, forward_problem(cfg, 8, 16, "cpu"), 8, 16, (0, 1, 3),
                         lambda b: torch.from_numpy(g[f"cached_b{b}"]))


def test_cached_forward_launches(tiny_rt, emulated, monkeypatch):
    cfg, rt = tiny_rt
    check_cached_launches(rt, forward_problem(cfg, 8, 16, "cpu"), 8, 16, monkeypatch)


def test_cached_forward_needs_a_full_forward(emulated):
    cfg, sd = unet_weights("tiny")
    rt = runtime(cfg, sd, "cpu")
    (x0, t0), _, ctx, y, mask = forward_problem(cfg, 8, 16, "cpu")
    rt.set_conditioning(ctx, y)
    with pytest.raises(RuntimeError, match="full forward"):
        rt_forward(rt, x0, t0, mask, 8, 16, cached=True, cache_branch=0)
    rt_forward(rt, x0, t0, mask, 8, 16)
    with pytest.raises(ValueError, match="cache_branch"):
        rt_forward(rt, x0, t0, mask, 8, 16, cached=True, cache_branch=4)


# ------------------------------------------------------------------------------------------------------------------
# cached samples on the fused loop
# ------------------------------------------------------------------------------------------------------------------
def counting_forwards(monkeypatch, net, dev):
    """Records (rows, slot, cached branch or None) of every UNet runtime forward."""
    rt = tic.runtime(net, dev)
    rows, real = [], rt.forward
    monkeypatch.setattr(rt, "forward", lambda unet_in, c_noise, *a, **k: (
        rows.append((c_noise.numel(), k.get("slot", ""), k.get("cache_branch") if k.get("cached") else None)),
        real(unet_in, c_noise, *a, **k))[1])
    return rows


def forwards_per_step(name):
    return {"vanilla": 1, "triangle": 1, "action": 2}.get(name)


def check_cached_sample(tiny, dev, kind, name, branch, monkeypatch, interval=2):
    """The fused loop with feature caching against the oracle loop on the same schedule; the cached forwards it runs
    are the schedule's; caching changes the sample."""
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    smp = make(kind, guider(name), interval, branch, device=dev)
    fwd = counting_forwards(monkeypatch, net, dev)
    fused = smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    ref, full = oracle_sample(smp, to_t(sd, dev), cfg, noise, c, uc, z, mask)
    per = forwards_per_step(name)
    cached = [f for f in fwd if f[2] is not None]
    assert all(f[2] == branch for f in cached)
    if per is not None:
        assert len(cached) == per * full.count(False) and len(fwd) == per * STEPS
    else:       # interval: guided steps run 2T + T rows, the others the T rows of the "cond" slot
        assert full == [True, True, False, True, True, False]
        assert [f for f in fwd if f[1] == "cond"] == [(T, "cond", None), (T, "cond", None), (T, "cond", branch)]
        assert len(cached) == 3
    uncached = make(kind, guider(name), 1, device=dev)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    r, moved = rel_l2(fused, ref), rel_l2(fused, uncached)
    print(f"tiny {kind} {name} interval {interval} branch {branch}: fused vs oracle loop {r:.3e}; vs uncached {moved:.3e}")
    assert r < SAMPLE_REL and torch.equal(fused[:1], z[:1])
    # the forward records above tell the schedule; where caching moves the sample well beyond the bar, the bar tells
    # a cached sample from an uncached one too
    assert not torch.equal(fused, uncached) and (name == "interval" or moved > 4 * r)
    return fused


CASES = [("vanilla", 0), ("vanilla", 1), ("vanilla", 3), ("triangle", 1), ("action", 1), ("interval", 1)]


@pytest.mark.parametrize("name,branch", CASES, ids=[f"{n}-b{b}" for n, b in CASES])
@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_cached_sample_against_oracle_loop(tiny, emulated, kind, name, branch, monkeypatch):
    check_cached_sample(tiny, "cpu", kind, name, branch, monkeypatch)


def check_interval_one_is_uncached(tiny, dev):
    """cache_interval = 1 is the sampler built without the keyword, torch.equal, for every guider."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    for kind in ("euler", "dpm"):
        for name in ("vanilla", "action", "interval"):
            a = make(kind, guider(name), 1, 3, steps=4, device=dev)(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
            b = tdc.make_sampler(kind, 4, dev, guider=guider(name))(bden, noise.clone(), c, uc=uc, cond_frame=z,
                                                                    cond_mask=mask)
            assert torch.equal(a, b), (kind, name)


def test_interval_one_is_uncached(tiny, emulated):
    check_interval_one_is_uncached(tiny, "cpu")


def samplers_for_interleaving(dev):
    tri = tac.triangle_cfg(T)
    return [make("euler", tri, 2, 1, steps=4, device=dev), make("euler", tri, 1, steps=4, device=dev),
            make("dpm", guider("interval"), 2, 0, device=dev), make("dpm", tac.action_cfg(5.0, tri), 3, 2, steps=4, device=dev),
            make("euler", tri, 2, 3, steps=4, device=dev)]


def check_interleaved(tiny, dev):
    """Cached and uncached samples of one shape back to back and interleaved on one loop state: each equals its
    standalone run on a fresh loop state."""
    cfg, sd, net, den, bden = tiny
    c, uc, noise, z, mask = tdc.tiny_inputs(cfg, dev)
    samplers = samplers_for_interleaving(dev)
    run = lambda smp: smp(bden, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
    alone = []
    for smp in samplers:
        tic.fresh(net, dev)
        alone.append(run(smp))
    tic.fresh(net, dev)
    seq = [run(smp) for smp in samplers + samplers[::-1]]
    for i, (got, want) in enumerate(zip(seq, alone + alone[::-1])):
        assert torch.equal(got, want), i
    assert not torch.equal(alone[0], alone[1]) and not torch.equal(alone[0], alone[4])
    return next(iter(tic.runtime(net, dev)._loop_states.values()))


def test_interleaved_and_back_to_back_calls(tiny, emulated):
    check_interleaved(tiny, "cpu")


# ------------------------------------------------------------------------------------------------------------------
# engine paths above the sampler, on the tiny native engine (shared with the GPU file)
# ------------------------------------------------------------------------------------------------------------------
def cached_sampler(eng, kind="euler", interval=2, branch=1, guider_config=None):
    s = tac.with_guider(eng.sampler, kind, guider_config or tac.triangle_cfg(sf.T))
    s.cache_interval, s.cache_branch = interval, branch
    return s


def check_session_equals_batch_rollout(eng, dev, monkeypatch, kind):
    """A session whose engine samples with caching is byte for byte engine.rollout(..., u8=True) with the same sampler
    over 2 rounds, and it repeats bit for bit."""
    from vista_b200.rollout import conditioner_recondition
    monkeypatch.setattr(eng, "sampler", cached_sampler(eng, kind))
    vd, z, noises = inputs(2, "cache_session")
    z, noises = z.to(dev), [n.to(dev) for n in noises]

    def run_session():
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        return torch.cat([sess.step(None, noise=nz) for nz in noises] + [sess.close()]), sess.samples_z

    frames, samples_z = run_session()
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, 2, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                               u8=True)
    assert torch.equal(frames, want) and torch.equal(samples_z, want_z)
    frames2, samples_z2 = run_session()
    assert torch.equal(frames, frames2) and torch.equal(samples_z, samples_z2)


def check_score_leaves_the_session_untouched(eng, dev, monkeypatch):
    """A session that scores with a cached sampler before every step samples the same rounds as one that never scores;
    round 0's score is sample_ensemble with that sampler."""
    monkeypatch.setattr(eng, "sampler", tac.with_guider(eng.sampler, "euler", tac.vanilla_cfg()))
    vd, z, ns = inputs(2, "cache_score")
    z, ns = z.to(dev), [n.to(dev) for n in ns]
    smp = cached_sampler(eng, "dpm", 2, 1, tac.vanilla_cfg())

    def run(scoring):
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        frames, scores = [], []
        for nz in ns:
            if scoring:
                scores.append(sess.score([tac.B, None], ensemble_size=2, num_steps=eng.sampler.num_steps, noises=ns,
                                         sampler=smp))
            frames.append(sess.step(tac.A, noise=nz))
        return torch.cat(frames + [sess.close()]), sess.samples_z, scores

    f0, z0, _ = run(False)
    f1, z1, scores = run(True)
    assert torch.equal(f0, f1) and torch.equal(z0, z1)
    rewards, members = scores[0]
    monkeypatch.setattr(eng, "sampler", smp)
    reward, want = eng.sample_ensemble(*eng.condition({**vd, **tac.B}, sf.T, mgc.UC_KEYS), z, 2, noises=ns)
    assert torch.equal(members[0], torch.stack(want)) and torch.equal(rewards[0], reward)


@pytest.fixture(scope="module")
def eng():
    e = native_engine(steps=3)
    e.en_and_decode_n_samples_a_time = 14
    return e


@pytest.mark.parametrize("kind", ["euler", "dpm"])
def test_session_equals_batch_rollout(eng, emulated, monkeypatch, kind):
    check_session_equals_batch_rollout(eng, torch.device("cpu"), monkeypatch, kind)


def test_score_leaves_the_session_untouched(eng, emulated, monkeypatch):
    check_score_leaves_the_session_untouched(eng, torch.device("cpu"), monkeypatch)
