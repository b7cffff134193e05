"""GroupNorm statistics on offset and near-flat groups: the inputs, the bound, and its self-checks.

A group whose mean is large next to its spread, or that is nearly constant, loses its variance when the statistics are
taken in one pass as E x^2 - mean^2 from fp32 sums: about (mean / std)^2 sqrt(n) 2^-24 of it.  The bound here is
GroupNorm's own (groupnorm_reference, shadow.check_mean_rstd), with no term that grows with |mean| / std:

    |y - ref| <= ulp16(ref) + c sqrt(n) U24 |x - mean| rstd |gamma| + 4 ulp32(mean) rstd |gamma|   (+ c sqrt(n) U24 |beta|)
    |d mean|  <= ulp32(mean) + c sqrt(n_add) U24 std
    |d rstd| / rstd <= c sqrt(n_add) U24 + 4 U24

against fp64 two-pass statistics of the tensor that is normalised.  This module shows the bound is reachable (torch's
fp32 group_norm meets it on every case), that a host emulation of one-pass fp32 sums (the scheme gn_stats_kernel and
the GEMM's STATS epilogue used) violates it on the offset and near-flat cases, and that emulations of the shifted sums
and of the deviation partials meet it.  The operator twins meet it too.  tests/test_norm_statistics_gpu.py runs the
same cases through every statistics path of the kernels."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fake_ops
from test_conformance_cpu import FAMILY, U24, check_stats, groupnorm_reference, quarters, ulp

C_ACC = FAMILY["norm"].c_acc
EPS = 1e-6                       # the VAE's GroupNorm eps: the smallest of the path, the least forgiving of a variance error

# (name, mean, std): std 0 is an exactly constant group; 2^-10 at mean 1 is about one fp16 ulp
SPECS = [("zero", 0.0, 1.0), ("m8", 8.0, 1.0), ("m64", 64.0, 1.0), ("m512", 512.0, 1.0), ("m-300", -300.0, 0.25),
         ("flat7", 1.0, 2.0 ** -7), ("flat10", 1.0, 2.0 ** -10), ("const", 3.0, 0.0)]
SPEC = {s[0]: s for s in SPECS}
# one table per case: every group of every statistic takes the spec; "mixed" cycles through all of them (a group or
# statistic index mix-up then pairs the wrong group's statistics with the data); "onech" puts the offset on one
# channel of each group only
CASES = [s[0] for s in SPECS] + ["mixed", "onech-m512", "onech-flat10"]
OFFSET_CASES = {"m64", "m512", "m-300", "flat7", "flat10", "mixed"}
# 32-term fp32 sums of squares of fp16 values near 64 happen to be exact: the GEMM partials' old scheme fails the rest
RAW_PARTIALS_FAIL = OFFSET_CASES - {"m64"}
SHARED_OFFSET = [c for c in CASES if not c.startswith("onech-")]    # shifting every channel of a group leaves GN as is


def grid_step(mean, std):
    """A grid on which every value of the group, and the group shifted by -mean, is an exact fp16 number."""
    top = abs(mean) + 6 * std
    u16 = 2.0 ** (math.floor(math.log2(top)) - 10) if top > 0 else 2.0 ** -24
    return max(std / 8, u16) if std > 0 else u16


def group_table(case, n_stat, groups):
    """[(mean, std, one_channel)] per (statistic, group)."""
    if case == "mixed":
        return [[SPECS[(s * 3 + g) % len(SPECS)][1:] + (False,) for g in range(groups)] for s in range(n_stat)]
    one = case.startswith("onech-")
    _, m, sd = SPEC[case[6:] if one else case]
    return [[(m, sd, one)] * groups for _ in range(n_stat)]


def make_input(case, frames, tpf, C, fps, groups=32, seed=0, centred=False):
    """fp16 [frames tpf, C] with the case's (mean, std) per (statistic, group), every value on grid_step's grid, and
    the per-(statistic, group) offsets [n_stat, groups] fp64.  ``centred``: the same tensor minus its offsets (exact)."""
    g = torch.Generator().manual_seed(seed)
    n_stat, per, cpg = frames // fps, fps * tpf, C // groups
    x = torch.empty(n_stat, per, groups, cpg, dtype=torch.float64)
    off = torch.zeros(n_stat, groups, cpg, dtype=torch.float64)
    for s, row in enumerate(group_table(case, n_stat, groups)):
        for j, (m, sd, one) in enumerate(row):
            st = grid_step(m, sd)
            k = torch.round(torch.randn(per, cpg, generator=g, dtype=torch.float64) * (sd / st)).clamp(-6 * sd / st,
                                                                                                    6 * sd / st)
            x[s, :, j] = k * st
            if one:
                off[s, j, 0] = m
            else:
                off[s, j] = m
    if not centred:
        x = x + off[:, None]
    out = x.reshape(frames * tpf, C)
    assert torch.equal(out.half().double(), out), "grid values not exact in fp16"
    return out.half(), off


def affine(C, seed=5):
    g = torch.Generator().manual_seed(seed)
    gamma = (torch.randn(C, generator=g) * 0.1 + 1).float()
    beta = (torch.randn(C, generator=g) * 0.1).float()
    return gamma, beta


def moments(x, frames, tpf, C, fps, groups=32):
    """fp64 two-pass (mean, var) [n_stat, groups]."""
    v = x[:, :C].double().reshape(frames // fps, fps * tpf, groups, C // groups)
    mean = v.mean(dim=(1, 3))
    var = ((v - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    return mean, var


def output_ratio(y, x, frames, tpf, gamma, beta, eps, silu, fps, groups=32):
    """Worst |y - ref| / bound over the elements (> 1 fails)."""
    C = gamma.numel()
    ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, eps, silu, fps, groups)
    tol = ulp(ref, torch.float16) + C_ACC * math.sqrt(fps * tpf * C // groups) * U24 * mag + extra
    return float(((y.double() - ref).abs() / tol).max())


def stats_ratio(mean_got, rstd_got, mean, var, eps, acc):
    """Worst error / bound of (mean, rstd) against fp64 (shadow.check_mean_rstd's bound)."""
    tol_m = ulp(mean, torch.float32) + acc * var.sqrt()
    rstd = torch.rsqrt(var + eps)
    tol_r = rstd * (acc + 4 * U24)
    return max(float(((mean_got.double() - mean).abs() / tol_m).max()),
               float(((rstd_got.double() - rstd).abs() / tol_r).max()))


def apply_fp32(x, frames, tpf, gamma, beta, silu, fps, mean, rstd, groups=32):
    """gn_apply_kernel's arithmetic on the host: fp32 scale = rstd gamma, shift = beta - mean scale, fma, fp16 store."""
    C = gamma.numel()
    m = mean.float().repeat_interleave(C // groups, dim=1)[:, None]
    sc = rstd.float().repeat_interleave(C // groups, dim=1)[:, None] * gamma
    sf = beta - m * sc
    xs = x[:, :C].float().reshape(frames // fps, fps * tpf, C)
    r = (xs.double() * sc.double() + sf.double()).float()            # one rounding, as fmaf
    r = F.silu(r) if silu else r
    return r.reshape(-1, C).half()


# ----------------------------------------------------------------------------------------------------------------
# Host emulations of the accumulation schemes: per "thread", n_add fp16 values of one channel into fp32 sums, the
# threads then combined in fp64 (gn_stats_kernel); per 32-row quarter, fp32 column partials (the GEMM's STATS epilogue)
# ----------------------------------------------------------------------------------------------------------------
def _threads(x, frames, tpf, C, fps, n_add, groups):
    v = x[:, :C].float().numpy().reshape(frames // fps, fps * tpf, groups, C // groups)
    per = v.shape[1]
    pad = (-per) % n_add
    valid = np.ones((v.shape[0], per + pad, groups, C // groups), dtype=bool)
    valid[:, per:] = False
    v = np.concatenate([v, np.zeros((v.shape[0], pad) + v.shape[2:], np.float32)], axis=1)
    return v.reshape(v.shape[0], -1, n_add, groups, C // groups), valid.reshape(v.shape[0], -1, n_add, groups, C // groups)


def emulate_one_pass(x, frames, tpf, C, fps, n_add, eps, groups=32):
    """The old gn_stats_kernel: fp32 sum x and sum x^2 per thread, fp64 combine, var = E x^2 - mean^2."""
    v, _ = _threads(x, frames, tpf, C, fps, n_add, groups)
    s = np.zeros(v.shape[:2] + v.shape[3:], np.float32)
    q = np.zeros_like(s)
    for i in range(n_add):
        s = s + v[:, :, i]
        q = q + v[:, :, i] * v[:, :, i]
    return _finalise(s.astype(np.float64).sum(axis=(1, 3)), q.astype(np.float64).sum(axis=(1, 3)),
                     fps * tpf * (C // groups), eps)


def emulate_shifted(x, frames, tpf, C, fps, n_add, eps, groups=32):
    """The new gn_stats_kernel: pivot K = the thread's first value, fp32 sums of d = x - K and d^2, rebuilt in fp64."""
    v, ok = _threads(x, frames, tpf, C, fps, n_add, groups)
    K = v[:, :, 0]
    s = np.zeros_like(K)
    q = np.zeros_like(K)
    for i in range(n_add):
        d = np.where(ok[:, :, i], v[:, :, i] - K, np.float32(0))
        s = s + d
        q = q + d * d
    c = ok.sum(axis=2).astype(np.float64)
    K, s, q = K.astype(np.float64), s.astype(np.float64), q.astype(np.float64)
    return _finalise((c * K + s).sum(axis=(1, 3)), (c * K * K + 2 * K * s + q).sum(axis=(1, 3)),
                     fps * tpf * (C // groups), eps)


def _finalise(a, b, count, eps):
    mean = a / count
    var = np.maximum(b / count - mean * mean, 0.0)
    return torch.from_numpy(mean).float(), torch.from_numpy(1.0 / np.sqrt(var + eps)).float()


def raw_square_partials(stored):
    """The old STATS epilogue's partials: fp32 column sums and sums of squares per 32-row quarter."""
    v = stored.float()
    pad = (-v.shape[0]) % 128
    v = F.pad(v, (0, 0, 0, pad)).reshape(-1, 32, v.shape[1])
    return torch.stack([v.sum(1), (v * v).sum(1)], dim=-1)


def partials_stats(p, frames, tpf, C, fps, eps, raw, groups=32):
    """(mean, rstd) from GEMM partials: ``raw`` = (sum, sum of squares), else (sum, deviation sum) as the kernels now."""
    n_stat, rows = frames // fps, fps * tpf // 32
    pp = p.double() if raw else fake_ops.partials_raw_sums(p)
    s = pp[: n_stat * rows].reshape(n_stat, rows, groups, C // groups, 2).sum(dim=(1, 3))
    return _finalise(s[..., 0].numpy(), s[..., 1].numpy(), fps * tpf * (C // groups), eps)


# ----------------------------------------------------------------------------------------------------------------
SHAPE = (2, 256, 320, 1)          # frames, tokens per frame, C, frames per statistic
N_ADD = 218                       # per-thread additions of the production decoder's statistics (order of)


def test_inputs_are_exact_and_have_the_spec():
    for case in CASES:
        x, off = make_input(case, 4, 256, 64, 2, seed=3)
        z, _ = make_input(case, 4, 256, 64, 2, seed=3, centred=True)
        d = (x.double() - z.double()).reshape(2, 512, 32, 2)
        assert torch.equal(d, off[:, None].expand_as(d)), case
    x, _ = make_input("flat10", 1, 4096, 64, 1)
    k = (x.double() - 1) * 1024                      # one-ulp steps around 1, about one step of spread
    assert torch.equal(k, torch.round(k)) and 0.8 < float(k.std()) < 1.2
    c, _ = make_input("const", 1, 64, 64, 1)
    assert bool((c == 3.0).all())


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_torch_fp32_group_norm_meets_the_bound(case, silu):
    """The bound is reachable: torch's fp32 group_norm meets it on every case (so it was not fitted to a kernel)."""
    frames, tpf, C, fps = SHAPE
    x, _ = make_input(case, frames, tpf, C, fps, seed=11)
    gamma, beta = affine(C)
    xt = x.float().reshape(frames // fps, fps * tpf, C).permute(0, 2, 1)
    y = F.group_norm(xt, 32, gamma, beta, EPS).permute(0, 2, 1).reshape(-1, C)
    y = (F.silu(y) if silu else y).half()
    assert output_ratio(y, x, frames, tpf, gamma, beta, EPS, silu, fps) <= 1.0


@pytest.mark.parametrize("case", CASES)
def test_one_pass_fp32_violates_and_shifted_sums_meet_the_bound(case):
    """Host emulation of the statistics kernel's accumulation (N_ADD fp16 values per fp32 accumulator, fp64 combine):
    one-pass E x^2 - mean^2 fails the offset and near-flat cases; the shifted sums meet every case, statistics and
    output alike."""
    frames, tpf, C, fps = 2, 2048, 64, 2
    x, _ = make_input(case, frames, tpf, C, fps, seed=13)
    gamma, beta = affine(C)
    mean, var = moments(x, frames, tpf, C, fps)
    acc = C_ACC * math.sqrt(N_ADD + 1) * U24
    ratios = {}
    for name, emu in (("one-pass", emulate_one_pass), ("shifted", emulate_shifted)):
        m, r = emu(x, frames, tpf, C, fps, N_ADD, EPS)
        y = apply_fp32(x, frames, tpf, gamma, beta, False, fps, m, r)
        ratios[name] = (stats_ratio(m, r, mean, var, EPS, acc), output_ratio(y, x, frames, tpf, gamma, beta, EPS, False,
                                                                            fps))
    assert max(ratios["shifted"]) <= 1.0, ratios
    if case in OFFSET_CASES:
        assert ratios["one-pass"][1] > 1.0, ratios
    elif case in ("zero", "m8"):
        assert ratios["one-pass"][1] <= 1.0, ratios


@pytest.mark.parametrize("case", CASES)
def test_gemm_partials_deviation_form_meets_raw_squares_violate(case):
    """The GEMM's column partials: sums of squares per 32-row quarter fail the offset and near-flat cases once
    finalised; (sum, squared deviations from the quarter mean), as the twin and the kernel now write them, meet the
    bound, and check_stats tells the two apart."""
    frames, tpf, C, fps = 2, 1024, 64, 2
    x, _ = make_input(case, frames, tpf, C, fps, seed=17)
    gamma, beta = affine(C)
    mean, var = moments(x, frames, tpf, C, fps)
    part = torch.zeros(frames * tpf // 32, C, 2)
    fake_ops._stats_partials(x, part)
    check_stats(part, x, f"{case} twin partials")
    old = raw_square_partials(x)
    acc = C_ACC * math.sqrt(32) * U24
    for raw, p in ((False, part), (True, old)):
        m, r = partials_stats(p, frames, tpf, C, fps, EPS, raw)
        y = apply_fp32(x, frames, tpf, gamma, beta, False, fps, m, r)
        ratio = max(stats_ratio(m, r, mean, var, EPS, acc), output_ratio(y, x, frames, tpf, gamma, beta, EPS, False, fps))
        if not raw:
            assert ratio <= 1.0, (case, ratio)
        elif case in RAW_PARTIALS_FAIL:
            assert ratio > 1.0, (case, ratio)
    if case in RAW_PARTIALS_FAIL:
        with pytest.raises(AssertionError):
            check_stats(torch.stack([old[..., 0], old[..., 1] - old[..., 0] ** 2 / 32], -1), x, "raw-square partials")


def test_quarters_counts_a_partial_last_tile():
    v, n = quarters(torch.ones(200, 8))
    assert v.shape == (8, 32, 8) and n.flatten().tolist() == [32, 32, 32, 32, 32, 32, 8, 0]
    part = torch.zeros(8, 8, 2)
    fake_ops._stats_partials(torch.ones(200, 8, dtype=torch.float16) * 7, part)
    assert part[6, 0, 0] == 56 and part[7, 0, 0] == 0 and bool((part[..., 1] == 0).all())


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_twins_meet_the_bound(case, silu):
    """The operator twins (fp32 torch) on the same cases: groupnorm, the STATS GEMM twin into groupnorm_from_partials
    and groupnorm_apply, and the shift invariance GN(x + c_g) = GN(x)."""
    frames, tpf, C, fps = 4, 256, 320, 2
    x, off = make_input(case, frames, tpf, C, fps, seed=19)
    z, _ = make_input(case, frames, tpf, C, fps, seed=19, centred=True)
    gamma, beta = affine(C)
    y = torch.empty_like(x)
    fake_ops.groupnorm(x, y, frames, tpf, gamma, beta, EPS, silu, frames_per_stat=fps)
    assert output_ratio(y, x, frames, tpf, gamma, beta, EPS, silu, fps) <= 1.0
    yz = torch.empty_like(z)
    fake_ops.groupnorm(z, yz, frames, tpf, gamma, beta, EPS, silu, frames_per_stat=fps)
    if case in SHARED_OFFSET:
        ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, EPS, silu, fps)
        tol = ulp(ref, torch.float16) + C_ACC * math.sqrt(fps * tpf * C // 32) * U24 * mag + extra
        assert bool(((y.double() - yz.double()).abs() <= 2 * tol).all()), case
    # STATS GEMM twin: identity weights
    out = torch.empty_like(x)
    part = torch.zeros(frames * tpf // 32, C, 2)
    fake_ops.gemm(x, torch.eye(C, dtype=torch.float16), out, stats=part)
    st = torch.empty(frames // fps, 32, 2)
    fake_ops.groupnorm_from_partials(part, frames, tpf, C, EPS, st, fps)
    mean, var = moments(out, frames, tpf, C, fps)
    assert stats_ratio(st[..., 0], st[..., 1], mean, var, EPS, C_ACC * math.sqrt(32) * U24) <= 1.0
    ya = torch.empty_like(out)
    fake_ops.groupnorm_apply(out, ya, frames, tpf, gamma, beta, silu, st, fps)
    assert output_ratio(ya, out, frames, tpf, gamma, beta, EPS, silu, fps) <= 1.0
