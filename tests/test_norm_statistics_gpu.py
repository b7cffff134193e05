"""GroupNorm and LayerNorm on offset and near-flat groups, through every statistics path of the kernels, against fp64
two-pass statistics of the tensor that is normalised and GroupNorm's own bound (test_norm_statistics_cpu.py: the
inputs, the bound and its self-checks).

Paths: ops.groupnorm (gn_stats_kernel + gn_apply_kernel) at J = 1 / 2 / 3 (C 64 and 320, 2560, 4608), one and 25
frames per statistic, single- and multi-chunk, with the statistics out and SiLU on and off; the tap-GEMM's STATS
epilogue (the offset from a per-column bias or from res1; linear, tap and upsampling modes; a partial last tile) into
groupnorm_from_partials and groupnorm_apply; the frame-sharded halves on simulated ranks (groupnorm_sums and
groupnorm_from_partials(raw_sums=) into groupnorm_finalize_apply); and both LayerNorm kernels on offset and
near-constant rows.  Shift invariance is checked as well: GN(x + c_g) = GN(x) within the bound for an exact per-group
shift, LN(x + c_row) = LN(x) per row.  Each test prints its worst error / bound per path."""
import math

import pytest
import torch

from shadow import PARTIALS_ACCUMULATION, gn_stats_accumulation, moments64, n_tiles, tile_tokens
from test_conformance_cpu import FAMILY, U24, check_stats, groupnorm_reference, ulp
from test_norm_statistics_cpu import CASES, EPS, SHARED_OFFSET, affine, make_input

pytestmark = pytest.mark.gpu
C_ACC = FAMILY["norm"].c_acc
TAPS_3X3 = [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as _ops
    lib.load()
    return _ops


def dev():
    return torch.device("cuda:0")


def sample_rows(total, n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = torch.cat([torch.arange(min(total, 512)), torch.arange(max(0, total - 512), total),
                   torch.randint(0, total, (n,), generator=g)])
    return torch.unique(r).to(dev())


class Ratios:
    """Worst error / bound per path of one test; fails at the end, naming every path over 1."""

    def __init__(self, name):
        self.name, self.r = name, {}

    def note(self, what, ratio):
        self.r[what] = max(self.r.get(what, 0.0), ratio)

    def stats(self, what, got, mean, var, eps, acc):
        tol_m = ulp(mean, torch.float32) + acc * var.sqrt()
        rstd = torch.rsqrt(var + eps)
        tol_r = rstd * (acc + 4 * U24)
        self.note(f"{what} mean", float(((got[..., 0].double() - mean).abs() / tol_m).max()))
        self.note(f"{what} rstd", float(((got[..., 1].double() - rstd).abs() / tol_r).max()))

    def output(self, what, y, x, frames, tpf, gamma, beta, eps, silu, fps, mean, var, rows, groups=32, other=None):
        C = gamma.numel()
        ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, eps, silu, fps, groups, rows=rows,
                                              moments=(mean, torch.rsqrt(var + eps)))
        tol = ulp(ref, torch.float16) + C_ACC * math.sqrt(fps * tpf * C // groups) * U24 * mag + extra
        self.note(what, float(((y[rows, :C].double() - ref).abs() / tol).max()))
        if other is not None:              # the same GroupNorm of a shifted input: equal within both bounds
            self.note(f"{what} shift", float(((y[rows, :C].double() - other[rows, :C].double()).abs() / (2 * tol)).max()))

    def check(self):
        print(f"{self.name}: " + ", ".join(f"{k} {v:.3g}" for k, v in self.r.items()))
        bad = {k: v for k, v in self.r.items() if not v <= 1.0}
        assert not bad, f"{self.name}: worst error / bound over 1: {bad}"


def inputs(case, frames, tpf, C, fps, seed):
    x, off = make_input(case, frames, tpf, C, fps, seed=seed)
    z, _ = make_input(case, frames, tpf, C, fps, seed=seed, centred=True)
    return x.to(dev()), z.to(dev()), off


# (frames, tokens per frame, C, frames per statistic): J = 1 single chunk (tokens per frame below kGnMinChunk), J = 1
# multi-chunk, 25 frames per statistic, J = 2 (C 2560), J = 3 (C 4608, the JT = 4 kernel)
GN_SHAPES = [(2, 13, 64, 1), (2, 4096, 320, 1), (25, 40, 320, 25), (2, 600, 2560, 2), (1, 256, 4608, 1)]


@pytest.mark.parametrize("shape", GN_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("case", CASES)
def test_groupnorm_offset_and_flat(ops, case, shape):
    frames, tpf, C, fps = shape
    x, z, _ = inputs(case, frames, tpf, C, fps, seed=21)
    gamma, beta = (t.to(dev()) for t in affine(C))
    mean, var, _, _ = moments64(x, frames, tpf, C, fps, 32)
    rows = sample_rows(frames * tpf)
    acc = gn_stats_accumulation(frames, tpf, C)
    R = Ratios(f"groupnorm {case} {shape}")
    for silu in (False, True):
        st = torch.empty(frames // fps, 32, 2, dtype=torch.float32, device=dev())
        y = torch.empty_like(x)
        ops.groupnorm(x, y, frames, tpf, gamma, beta, EPS, silu, stats=st, frames_per_stat=fps)
        yz = torch.empty_like(z)
        ops.groupnorm(z, yz, frames, tpf, gamma, beta, EPS, silu, frames_per_stat=fps)
        torch.cuda.synchronize()
        R.stats("gn_stats", st, mean, var, EPS, acc)
        R.output(f"groupnorm silu={silu}", y, x, frames, tpf, gamma, beta, EPS, silu, fps, mean, var, rows,
                 other=yz if case in SHARED_OFFSET else None)
    R.check()


@pytest.mark.parametrize("case", ["m512", "flat10", "const"])
def test_groupnorm_offset_and_flat_decoder_scale(ops, case):
    """The full-resolution decoder's statistics shape class: C 128, 8 frames of 576 x 1024 per statistic, ~125
    additions per thread accumulator.  The input is drawn on the GPU, on the case's grid."""
    from test_norm_statistics_cpu import SPEC, grid_step
    frames, tpf, C, fps = 8, 576 * 1024, 128, 8
    _, m, sd = SPEC[case]
    st_ = grid_step(m, sd)
    gen = torch.Generator(device=dev()).manual_seed(23)
    k = torch.randn(frames * tpf, C, generator=gen, device=dev()) * (sd / st_)
    x = (m + torch.round(k).clamp(-6 * sd / st_, 6 * sd / st_) * st_).half()
    del k
    gamma, beta = (t.to(dev()) for t in affine(C))
    mean, var, _, _ = moments64(x, frames, tpf, C, fps, 32)
    R = Ratios(f"groupnorm {case} decoder scale")
    st = torch.empty(1, 32, 2, dtype=torch.float32, device=dev())
    y = torch.empty_like(x)
    ops.groupnorm(x, y, frames, tpf, gamma, beta, EPS, True, stats=st, frames_per_stat=fps)
    torch.cuda.synchronize()
    R.stats("gn_stats", st, mean, var, EPS, gn_stats_accumulation(frames, tpf, C))
    R.output("groupnorm", y, x, frames, tpf, gamma, beta, EPS, True, fps, mean, var, sample_rows(frames * tpf))
    R.check()


# ----------------------------------------------------------------------------------------------------------------
# Tap-GEMM STATS epilogue -> groupnorm_from_partials -> groupnorm_apply
# ----------------------------------------------------------------------------------------------------------------
def column_offsets(case, C, groups=32):
    """fp32 [C] per-column offsets of one statistic of the case (the bias that makes the GEMM output offset)."""
    _, off = make_input(case, 1, 8, C, 1)
    return off.reshape(-1).float()


def spread(case):
    from test_norm_statistics_cpu import SPEC
    return SPEC[case[6:] if case.startswith("onech-") else case][2] if case != "mixed" else 1.0


# (mode, frames, geometry or tokens per frame, Cin, C): linear (a_mode 0), 3 x 3 taps over 32 x 16 frames (a_mode 1),
# the upsampling 3 x 3 over 16 x 8 -> 32 x 16 frames (a_mode 2)
GEMM_MODES = {"linear": (2, 1024, 64, 320), "taps": (2, (32, 16), 64, 128), "upsample": (2, (16, 8), 64, 128)}


@pytest.mark.parametrize("source", ["bias", "res1"])
@pytest.mark.parametrize("mode", list(GEMM_MODES))
@pytest.mark.parametrize("case", CASES)
def test_gemm_stats_offset_and_flat(ops, case, mode, source):
    if mode == "upsample" and source == "res1":
        pytest.skip("the upsampling GEMM takes a bias only")
    frames, g, Cin, C = GEMM_MODES[mode]
    geom = None if mode == "linear" else (g[0], g[1], frames)
    tpf = g if mode == "linear" else g[0] * g[1] * (4 if mode == "upsample" else 1)
    taps = [(0, 0)] if mode == "linear" else TAPS_3X3
    tokens_in = frames * (g if mode == "linear" else g[0] * g[1])
    gen = torch.Generator().manual_seed(31)
    a = torch.randn(tokens_in, Cin, generator=gen).half().to(dev())
    K = len(taps) * Cin
    if source == "bias":             # out = a w^T + bias: the spread from the product, the offset from the bias
        w = (torch.randn(C, K, generator=gen) * (spread(case) / math.sqrt(K))).half().to(dev())
        bias, res1 = column_offsets(case, C).to(dev()), None
    else:                            # out = x + (a w^T, tiny): the case's tensor through the residual
        w = (torch.randn(C, K, generator=gen) * (2.0 ** -16 / math.sqrt(K))).half().to(dev())
        bias = None
        res1 = make_input(case, frames, tpf, C, frames, seed=33)[0].to(dev())
    out = torch.empty(frames * tpf, C, dtype=torch.float16, device=dev())
    part = torch.full((frames * tpf // 32, C, 2), float("nan"), dtype=torch.float32, device=dev())
    ops.gemm(a, w, out, taps=taps, geom=geom, bias=bias, res1=res1, stats=part, upsample=mode == "upsample")
    torch.cuda.synchronize()
    R = Ratios(f"gemm stats {case} {mode} {source}")
    # partials against the stored values, tile by tile in the kernel's row order
    a_mode = {"linear": 0, "taps": 1, "upsample": 2}[mode]
    box = None if geom is None else (ops.upsample_stats_box(*geom[:2]) if a_mode == 2 else ops.stats_box(*geom))
    for m in range(n_tiles(a_mode, geom, box, tokens_in)):
        tr = tile_tokens(a_mode, geom, box, m, tokens_in).to(dev())
        check_stats(part[4 * m:4 * m + 4], out[tr], f"{R.name} tile {m}")
    gamma, beta = (t.to(dev()) for t in affine(C))
    mean, var, _, _ = moments64(out, frames, tpf, C, frames, 32)
    rows = sample_rows(frames * tpf)
    for silu in (False, True):
        st = torch.empty(1, 32, 2, dtype=torch.float32, device=dev())
        ops.groupnorm_from_partials(part, frames, tpf, C, EPS, st, frames)
        y = torch.empty_like(out)
        ops.groupnorm_apply(out, y, frames, tpf, gamma, beta, silu, st, frames)
        torch.cuda.synchronize()
        R.stats("from_partials", st, mean, var, EPS, PARTIALS_ACCUMULATION)
        R.output(f"apply silu={silu}", y, out, frames, tpf, gamma, beta, EPS, silu, frames, mean, var, rows)
    R.check()


@pytest.mark.parametrize("case", ["m512", "flat10", "mixed"])
def test_gemm_stats_partial_last_tile(ops, case):
    """A linear STATS GEMM whose last 128-token tile holds 72 tokens: its quarters count 32, 32, 8 and 0 rows."""
    tokens, Cin, C = 5 * 128 + 72, 64, 320
    gen = torch.Generator().manual_seed(41)
    a = torch.randn(tokens, Cin, generator=gen).half().to(dev())
    w = (torch.randn(C, Cin, generator=gen) * (spread(case) / 8)).half().to(dev())
    out = torch.empty(tokens, C, dtype=torch.float16, device=dev())
    part = torch.full((6 * 4, C, 2), float("nan"), dtype=torch.float32, device=dev())
    ops.gemm(a, w, out, bias=column_offsets(case, C).to(dev()), stats=part)
    torch.cuda.synchronize()
    check_stats(part, out, f"partial tile {case}")


def test_gemm_stats_refuses_bf16_output(ops):
    """Fused statistics are fp16-output only: a bf16 STATS GEMM is refused, not computed some other way."""
    a = torch.randn(128, 64).to(torch.bfloat16).to(dev())
    w = torch.randn(64, 64).to(torch.bfloat16).to(dev())
    out = torch.empty(128, 64, dtype=torch.bfloat16, device=dev())
    part = torch.zeros(4, 64, 2, device=dev())
    with pytest.raises(Exception):
        ops.gemm(a, w, out, stats=part)
        torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------
# Frame-sharded halves on simulated ranks
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", CASES)
def test_sharded_offset_and_flat(ops, case, world):
    """groupnorm_sums per rank -> fp64 sum over ranks -> groupnorm_finalize_apply, and the same from the ranks' STATS
    GEMM partials through groupnorm_from_partials(raw_sums=)."""
    from vista_b200.parallel import frame_shards
    nb, T, hw, C, G = 1, 9, 128, 320, 32
    x, _ = make_input(case, nb * T, hw, C, T, seed=51)
    x = x.to(dev())
    gamma, beta = (t.to(dev()) for t in affine(C))
    shards = frame_shards(T, world)
    count = float(C // G) * hw * T
    R = Ratios(f"sharded {case} W={world}")
    # 1. statistics pass per rank
    total = torch.zeros(nb * G, 2, dtype=torch.float64, device=dev())
    for s0, e in shards:
        sums = torch.empty(nb * G, 2, dtype=torch.float64, device=dev())
        ops.groupnorm_sums(x[s0 * hw:e * hw], e - s0, hw, C, sums, e - s0, groups=G)
        total += sums
    mean, var, _, _ = moments64(x, T, hw, C, T, G)
    for s0, e in shards:
        xr = x[s0 * hw:e * hw]
        y = torch.empty_like(xr)
        st = torch.empty(nb, G, 2, dtype=torch.float32, device=dev())
        ops.groupnorm_finalize_apply(xr, y, e - s0, hw, gamma, beta, EPS, True, total, count, st, e - s0, groups=G)
        torch.cuda.synchronize()
        R.stats("sums+finalize", st, mean, var, EPS, gn_stats_accumulation(e - s0, hw, C))
        yf = torch.zeros_like(x)
        yf[s0 * hw:e * hw] = y
        R.output("finalize_apply", yf, x, T, hw, gamma, beta, EPS, True, T, mean, var,
                 torch.arange(s0 * hw, e * hw, device=dev()))
    # 2. the ranks' GEMM partials (out = x + tiny product through res1)
    gen = torch.Generator().manual_seed(53)
    total = torch.zeros(nb * G, 2, dtype=torch.float64, device=dev())
    outs = []
    for s0, e in shards:
        a = torch.randn((e - s0) * hw, 64, generator=gen).half().to(dev())
        w = (torch.randn(C, 64, generator=gen) * 2.0 ** -19).half().to(dev())
        o = torch.empty((e - s0) * hw, C, dtype=torch.float16, device=dev())
        part = torch.zeros((e - s0) * hw // 32, C, 2, dtype=torch.float32, device=dev())
        ops.gemm(a, w, o, res1=x[s0 * hw:e * hw], stats=part)
        sums = torch.empty(nb * G, 2, dtype=torch.float64, device=dev())
        ops.groupnorm_from_partials(part, e - s0, hw, C, EPS, None, e - s0, G, raw_sums=sums)
        total += sums
        outs.append(o)
    o_full = torch.cat(outs)
    mean, var, _, _ = moments64(o_full, T, hw, C, T, G)
    for (s0, e), o in zip(shards, outs):
        y = torch.empty_like(o)
        st = torch.empty(nb, G, 2, dtype=torch.float32, device=dev())
        ops.groupnorm_finalize_apply(o, y, e - s0, hw, gamma, beta, EPS, False, total, count, st, e - s0, groups=G)
        torch.cuda.synchronize()
        R.stats("partials raw+finalize", st, mean, var, EPS, PARTIALS_ACCUMULATION)
        yf = torch.zeros_like(o_full)
        yf[s0 * hw:e * hw] = y
        R.output("partials finalize_apply", yf, o_full, T, hw, gamma, beta, EPS, False, T, mean, var,
                 torch.arange(s0 * hw, e * hw, device=dev()))
    R.check()


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm (two-pass in registers): offset and near-constant rows
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [320, 640, 1280, 512, 2560])     # layernorm40 at 320 / 640 / 1280, the generic kernel else
@pytest.mark.parametrize("case", CASES)
def test_layernorm_offset_and_flat(ops, case, C):
    """Rows with the case's (mean, std) (a "row" is one group of C channels and one token), against fp64 with the
    operation's bound (|x - mean| rstd |gamma| + |beta|, 4 ulp32(mean) rstd |gamma|), and LN(x + c_row) = LN(x)."""
    tokens = 600                     # one token per "statistic": "mixed" cycles the specs over the rows
    x, _ = make_input(case, tokens, 1, C, 1, groups=1, seed=61)
    z, _ = make_input(case, tokens, 1, C, 1, groups=1, seed=61, centred=True)
    x, z = x.to(dev()), z.to(dev())
    gamma, beta = (t.to(dev()) for t in affine(C))
    R = Ratios(f"layernorm {case} C={C}")
    y, yz = torch.empty_like(x), torch.empty_like(z)
    ops.layernorm(x, y, gamma, beta, 1e-5)
    ops.layernorm(z, yz, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    v = x.double()
    mean = v.mean(1, keepdim=True)
    rstd = torch.rsqrt(((v - mean) ** 2).mean(1, keepdim=True) + 1e-5)
    g, b = gamma.double(), beta.double()
    ref = (v - mean) * rstd * g + b
    tol = (ulp(ref, torch.float16) + C_ACC * math.sqrt(C) * U24 * ((v - mean).abs() * rstd * g.abs() + b.abs())
           + 4 * ulp(mean, torch.float32) * rstd * g.abs())
    R.note("layernorm", float(((y.double() - ref).abs() / tol).max()))
    if case in SHARED_OFFSET:
        R.note("layernorm shift", float(((y.double() - yz.double()).abs() / (2 * tol)).max()))
    R.check()
