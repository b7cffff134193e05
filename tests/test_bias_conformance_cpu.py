"""Gain conformance without a GPU: the estimator of tests/bias.py on synthetic data with known answers, then five
systematic defects planted in the operator twins (each under one ulp per element, each with a fixed sign) that pass the
element / rel-L2 rule of the launch harness and fail its gain check naming the op, the key and the term, and the two
layer-level defects of tests/trajectory.py on the tiny UNet."""
import math

import pytest
import torch
import torch.nn.functional as F

import bias
import fake_ops
import shadow
from test_conformance_cpu import FAMILY, U24, assert_conform, gemm_reference, ulp
from test_production_conformance_cpu import rnd
from vista_b200 import ops

U16 = bias.U16


# ==================================================================================================================
# The estimator
# ==================================================================================================================
def _data(seed, n_frames=16, per=4096):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(n_frames * per, generator=g, dtype=torch.float64)
    b = torch.randn(n_frames * per, generator=g, dtype=torch.float64) * 0.5
    frame = torch.arange(n_frames * per) // per
    return a, b, frame


def test_honest_rounding_passes():
    """Round-to-nearest of a continuous reference with no bias passes at half its bound or less: the pre-rounding
    value carries an unbiased accumulation error of 2^-16 relative (an fp32 sum over thousands of terms)."""
    a, b, frame = _data(1)
    ref = a + b
    noisy = ref * (1 + 2 ** -16 * torch.randn(ref.shape, generator=torch.Generator().manual_seed(11), dtype=ref.dtype))
    terms = bias.fit(noisy.half(), ref, {"a": a, "b": b}, {"a": 2 ** -14, "b": 2 ** -14}, frame)
    for t in terms:
        print(t)
        assert not t.skipped and t.ratio <= 0.5, t


@pytest.mark.parametrize("gain", [U16 / 2, U16 / 4])
def test_injected_gain_is_recovered(gain):
    """A gain of U16 / 2 or U16 / 4 on one term, below one ulp per element, is recovered within 10 % and fails."""
    a, b, frame = _data(2)
    ref = a + b
    out = (a * (1 + gain) + b).half()
    terms = {t.name: t for t in bias.fit(out, ref, {"a": a, "b": b}, {"a": 2 ** -14, "b": 2 ** -14}, frame)}
    print(terms)
    assert abs(terms["a"].beta - gain) <= 0.1 * gain, terms["a"]
    assert terms["a"].ratio > 1.0 and terms["b"].ratio <= 1.0
    assert bool(((out.double() - ref).abs() <= ulp(a.abs() + b.abs(), torch.float16)).all())   # under one ulp


def test_swallowed_branch():
    """out = RN16(res + a), res on the fp16 grid and |a| small next to its ulp: against out - ref the branch a regresses
    to beta = -1; against out - RN16(ref), the fit's error, it passes.  A branch swallowed whole is below 2^-11 of the
    output's norm, so the skip rule would drop it: here it is kept (energy_min = 0) to test the error's definition."""
    g = torch.Generator().manual_seed(3)
    n = 16 * 4096
    res = (torch.randn(n, generator=g) + 4).half().double()
    a = torch.randn(n, generator=g, dtype=torch.float64) * 2 ** -14
    ref = res + a
    out = ref.half()
    frame = torch.arange(n) // 4096
    dirs, bnd = {"res": res, "a": a}, {"res": 2 ** -14, "a": 2 ** -14}
    raw = {t.name: t for t in bias.fit(out, ref, dirs, bnd, frame, against_rounded=False, energy_min=0)}
    assert abs(raw["a"].beta + 1) < 0.05 and raw["a"].ratio > 1, raw["a"]
    good = {t.name: t for t in bias.fit(out, ref, dirs, bnd, frame, energy_min=0)}
    assert all(t.ratio <= 1 for t in good.values()), good


def test_nuisance_intercepts_and_bands():
    """Per-(frame, channel) constants absorbed by the intercepts; the fit accumulated band by band equals the one-shot
    fit; a direction of negligible norm is skipped and reported."""
    g = torch.Generator().manual_seed(4)
    F_, C, P = 8, 16, 512
    a = torch.randn(F_, C, P, generator=g, dtype=torch.float64)
    const = torch.randn(F_, C, 1, generator=g, dtype=torch.float64) * 2 ** -9      # a constant rounded once per frame
    tiny = torch.randn(F_, C, P, generator=g, dtype=torch.float64) * 1e-6
    ref = a + 3
    out = (ref + const).half()
    frame = torch.arange(F_)[:, None, None].expand(F_, C, P)
    group = (torch.arange(F_)[:, None, None] * C + torch.arange(C)[None, :, None]).expand(F_, C, P)
    bnd = {"a": 2 ** -14, "tiny": 2 ** -14}
    plain = {t.name: t for t in bias.fit(out, ref, {"a": a, "tiny": tiny}, bnd, frame)}
    nuis = {t.name: t for t in bias.fit(out, ref, {"a": a, "tiny": tiny}, bnd, frame, group=group, n_groups=F_ * C)}
    assert nuis["tiny"].skipped and "skipped" in repr(nuis["tiny"])
    assert nuis["a"].ratio <= 0.5, nuis["a"]
    f = bias.GainFit(["a", "tiny"], bnd, F_, F_ * C)
    e = out.double() - bias.rn(ref, torch.float16)
    for p0 in range(0, P, 100):                   # bands of pixels, every frame in each
        s = slice(p0, p0 + 100)
        f.add(e[:, :, s], [a[:, :, s], tiny[:, :, s]], frame[:, :, s], group[:, :, s], out=ref[:, :, s])
    banded = {t.name: t for t in f.result()}
    assert math.isclose(banded["a"].beta, nuis["a"].beta, rel_tol=1e-9, abs_tol=1e-15)
    assert math.isclose(banded["a"].sigma, nuis["a"].sigma, rel_tol=1e-6)
    print(plain["a"], nuis["a"])


# ==================================================================================================================
# Planted launch defects: each twin passes the element / rel-L2 rule and fails the gain check by op, key and term
# ==================================================================================================================
S_ACC, S_RES1 = 1.0 / 3.0, 2.0 / 3.0          # a blend and its complement: each loses U16 / 2 in fp16


def fp16_scale(s):
    return float(torch.tensor(s, dtype=torch.float64).half())


def run_gain_planted(monkeypatch, op, defective, term, *args, **kwargs):
    """The defect fails exactly one key of ``op``, on the gain check alone (its element and rel-L2 rule passed first),
    naming the op, its key and ``term``; returns the harness."""
    monkeypatch.setattr(ops, op, defective)
    with shadow.Shadow(random_rows=4096) as sh:
        getattr(ops, op)(*args, **kwargs)
    assert len(sh.failures) == 1, sh.failures
    (key, msg), = sh.failures.items()
    print("\n" + msg)
    assert key[0] == op and msg.startswith(f"{op} key {key[1:]}"), msg
    assert "systematic gain on" in msg and f"{term}: beta" in msg, msg
    return sh


def rz16(v):
    """fp32 -> fp16 rounded toward zero: round to nearest, then one step back toward zero where that went away from it
    (one less in the bit pattern, for either sign)."""
    h = v.half()
    away = h.double().abs() > v.double().abs()
    return torch.where(away, (h.view(torch.int16) - 1).view(torch.float16), h)


def rz16_after_extra_bit(v):
    """fp32 -> fp16 in two steps: round to nearest with one mantissa bit more than fp16, then toward zero.  A fraction
    f of an fp16 ulp goes up only from f >= 3/4: the error is -ulp / 4 on average, its RMS 1.3 x round-to-nearest's."""
    v64 = v.double()
    u = ulp(v64, torch.float16)
    a = v64.abs() / u
    k = torch.floor(a)
    return (torch.sign(v64) * torch.where(a - k >= 0.75, k + 1, k) * u).half()


def _gemm_operands():
    M, K, N = 2048, 576, 192
    a, w = rnd(M, K, seed=21), rnd(N, K, seed=22, scale=K ** -0.5)
    bias_v, res = rnd(N, seed=23, dtype=torch.float32), rnd(M, N, seed=24, scale=0.5)
    return a, w, bias_v, res


def test_planted_gemm_scales_rounded_to_fp16(monkeypatch):
    """1. The epilogue converts s_acc and s_res1 to fp16 before use: 1/3 and 2/3 each lose U16 / 2 of their value.
    (A scale that loses more, such as 1 - sigmoid(-0.3) at 0.8 U16, already fails the element rule where its term
    dominates the output.)"""
    for s in (S_ACC, S_RES1):
        assert abs(fp16_scale(s) - s) / s >= U16 / 2 * (1 - 1e-9)

    def bad(a, w, out, **kw):
        return fake_ops.gemm(a, w, out, **dict(kw, s_acc=fp16_scale(kw["s_acc"]), s_res1=fp16_scale(kw["s_res1"])))
    a, w, b, res = _gemm_operands()
    sh = run_gain_planted(monkeypatch, "gemm", bad, "acc", a, w, torch.empty(a.shape[0], w.shape[0], dtype=torch.float16),
                          bias=b, res1=res, s_res1=S_RES1, s_acc=S_ACC)
    assert "res1: beta" in next(iter(sh.failures.values()))


def _rz_twin(store):
    def bad(a, w, out, **kw):
        tmp = torch.empty(out.shape, dtype=torch.float32)
        fake_ops.gemm(a, w, tmp, **kw)
        out.copy_(store(tmp))
        return out
    return bad


def test_planted_gemm_store_rounds_toward_zero(monkeypatch):
    """2. The epilogue's store rounds toward zero.  A plain round-toward-zero store errs by [0, 1) ulp: its rel-L2 is
    sqrt(12 / 3) = 2 x the round-to-nearest floor, the rule's own factor, so the rule catches it by a hair or misses it
    by one.  Here the store truncates after rounding to one extra bit: -ulp / 4 per element on average, 1.3 x the floor,
    which the rule passes and the gain check fails on every term (a gain of about -2^-12.5)."""
    a, w, b, res = _gemm_operands()
    out = torch.empty(a.shape[0], w.shape[0], dtype=torch.float16)
    sh = run_gain_planted(monkeypatch, "gemm", _rz_twin(rz16_after_extra_bit), "acc", a, w, out, bias=b, res1=res,
                          s_res1=0.5)
    assert sh.worst_gain("gemm").beta < 0


def test_plain_round_toward_zero_sits_on_the_rel_l2_factor(monkeypatch):
    """The plain round-toward-zero store of the same GEMM: rel-L2 within 5 % of 2 x the floor (the rule's factor), and
    the gain check fails it at several times its bound whether or not the rule does."""
    a, w, b, res = _gemm_operands()
    out = torch.empty(a.shape[0], w.shape[0], dtype=torch.float16)
    _rz_twin(rz16)(a, w, out, bias=b, res1=res, s_res1=0.5)
    terms = {}
    ref, _ = gemm_reference(a, w, taps=[(0, 0)], geom=None, bias=b, res1=res, s_res1=0.5, terms=terms)
    rel = float((out.double() - ref).norm() / ref.norm())
    floor = float((bias.rn(ref, torch.float16) - ref).norm() / ref.norm())
    assert abs(rel / floor - 2.0) < 0.1, rel / floor
    res_t = bias.fit(out, ref, terms, {n: 2 ** -14 for n in terms}, bias.clusters(torch.arange(a.shape[0]))[:, None])
    assert min(t.ratio for t in res_t) >= 3.0, res_t


def test_planted_spatial_attention_scaled(monkeypatch):
    """3. The spatial attention's output scaled by 1 - 2^-11 (a softmax normaliser one rounding too large)."""
    frames, seq, heads = 4, 300, 2

    def bad(q, k, v, out, frames, seq, heads, impl=None):
        tmp = torch.empty(out.shape, dtype=torch.float32)
        fake_ops.attention_spatial(q, k, v, tmp, frames, seq, heads)
        out.copy_((tmp * (1 - U16)).to(out.dtype))
        return out
    C = heads * 64
    qkv = rnd(frames * seq, 3 * C, seed=25, scale=2.0)
    run_gain_planted(monkeypatch, "attention_spatial", bad, "ref", qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:],
                     torch.empty(frames * seq, C, dtype=torch.float16), frames, seq, heads)


GN_RSTD_GAIN = 2.0 ** -12


def test_planted_groupnorm_apply_rstd_high(monkeypatch):
    """4. The GroupNorm apply multiplies rstd by 1 + 2^-12.  (At 1 + 2^-11 the rel-L2 rule already fails it, at about
    2.4 x the floor: 2^-12 is the largest power-of-two gain below that rule.)  The statistics come from fused GEMM
    partials of the same tensor, as on the decoder's path.  beta is zero: with cancelling beta terms the element rule's eps of a 2048-element
    group is below the gain where an element nears zero (at production group sizes it is not)."""
    frames, tpf, C = 4, 1024, 64
    x = (rnd(frames * tpf, C, seed=26, dtype=torch.float32) * 1.5 + 0.3).half()
    gamma, beta = rnd(C, seed=27, dtype=torch.float32) * 0.2 + 1, torch.zeros(C)
    partials = torch.zeros(frames * tpf // 128 * 4, C, 2)
    fake_ops._stats_partials(x, partials)
    stats = torch.zeros(frames, 32, 2)
    monkeypatch.setattr(ops, "groupnorm_from_partials", fake_ops.groupnorm_from_partials)

    def bad(x, y, frames, tokens_per_frame, gamma, beta, silu, stats, frames_per_stat=1, groups=32):
        s = stats.clone()
        s[..., 1] *= 1 + GN_RSTD_GAIN
        return fake_ops.groupnorm_apply(x, y, frames, tokens_per_frame, gamma, beta, silu, s, frames_per_stat, groups)
    monkeypatch.setattr(ops, "groupnorm_apply", bad)
    with shadow.Shadow(random_rows=4096) as sh:
        ops.groupnorm_from_partials(partials, frames, tpf, C, 1e-6, stats)
        ops.groupnorm_apply(x, torch.empty_like(x), frames, tpf, gamma, beta, False, stats)
    assert list(sh.failures) and all(k[0] == "groupnorm_apply" for k in sh.failures), sh.failures
    msg, = sh.failures.values()
    print("\n" + msg)
    assert "systematic gain on" in msg and "norm: beta" in msg, msg


def test_planted_time_mix_blend_high(monkeypatch):
    """5. The time mix's chunk-overlap blend weight one ulp above 0.5.  Its outputs are fp32, held per element to
    12 U24 of their magnitude: one fp16 ulp of 0.5 (2^-10 relative) fails that rule outright, so the weight here is
    one fp32 ulp high (2^-23 relative), under it; the gain check's B for fp32 outputs is U24 / 8."""
    T, Hh, Ww = 5, 16, 32

    def bad(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0=0, skip_frames=0, keep_f32_from=-1):
        prev = out.clone()
        fake_ops.time_mix_small_u8(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0, skip_frames, keep_f32_from)
        for t in range(skip_frames, T):
            if blend is not None and int(blend[t]):
                f = out_frame0 + t
                mix = 2 * out[f] - prev[f]                      # exact: the twin's fp32 blend undone
                out[f] = (0.5 + U24) * (prev[f] + mix)
        return out_u8
    x = rnd(T * Hh * Ww, 8, seed=29, dtype=torch.float32, scale=0.8)
    w, b = rnd(3, 3, 3, seed=30, dtype=torch.float32, scale=0.5), rnd(3, seed=31, dtype=torch.float32, scale=0.1)
    out = rnd(T + 1, 3, Hh, Ww, seed=32, dtype=torch.float32, scale=0.7)
    out8 = torch.zeros(T + 1, Hh, Ww, 3, dtype=torch.uint8)
    blend = torch.tensor([1, 1, 1, 0, 0], dtype=torch.int32)
    run_gain_planted(monkeypatch, "time_mix_small_u8", bad, "prev", x, w, b, out, out8, blend, T, Hh * Ww, 3,
                     out_frame0=1)


# ==================================================================================================================
# Planted layer defects (tests/trajectory.py): the layer harness's gain check on the tiny UNet over the twins
# ==================================================================================================================
@pytest.fixture
def eager(monkeypatch):
    from vista_b200 import fused
    monkeypatch.setattr(fused, "USE_GRAPH", False)


def test_tiny_unet_layers_clean_gain(eager):
    """The clean tiny-UNet forward: every layer passes the partition rule and the gain check."""
    from test_block_conformance_cpu import run_unet
    bs, _ = run_unet()
    print("\n" + bs.report())
    bs.assert_ok()
    assert {"unet.resblock", "unet.svt"} <= set(bs.worst_gain_by_kind())


@pytest.mark.parametrize("defect,direction", [("residual", "res"), ("alpha", "d_alpha")])
def test_planted_layer_defect_fails_the_gain_check(eager, defect, direction):
    """Every residual GEMM's s_res1 x (1 + 2^-11), and every time mixer's alpha one fp16 ulp high: each passes the
    partition rule of every layer and fails the gain check at 2x its bound or more, naming a layer and the direction."""
    import trajectory as tj
    from test_block_conformance_cpu import run_unet
    with tj.planted(defect, fake_ops):
        bs, _ = run_unet()
    print("\n" + bs.report())
    for msg in bs.failures.values():
        print("   ", msg)
    assert bs.failures and all(k[0] == "gain" for k in bs.failures), list(bs.failures)
    hits = [bs.census[k[1]] for k in bs.failures if any(t.name.startswith(direction) and t.ratio > 1.0
                                                        for t in [bs.census[k[1]].gain_term])]
    assert hits, f"no layer fails on a {direction} direction: {list(bs.failures.values())}"
    worst = max(e.gain for e in hits)
    assert worst >= 2.0, f"{defect}: fails at only {worst:.2f} x the bound"
