"""Conformance of the CUDA kernels against fp64 references on the GPU, everywhere the library launches them: every tap-GEMM
instantiation, the frame-sharded kernels on simulated ranks, attention at the production shapes, the norms and the
small ops without op tests.  The case tables, the references and the tolerance rule live in test_conformance_cpu.py
(which runs the same tables on the CPU twins); where a twin exists, the tests here also run it on the same inputs and
hold it to the same reference."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

import fake_ops
from test_conformance_cpu import (ATTN_EPS, CPU, FAMILY, GN_CASES, IM2COL_CASES, LN_CASES, SOFTMAX_CASES,
                                  SPATIAL_CASES, TEMPORAL_T, U24, VARIANT_ARGS, assert_conform, case_id,
                                  check_gemm_case, expected_instantiations, gemm_cases, gemm_reference,
                                  groupnorm_reference, im2col_asym_reference, layernorm_reference, make_gemm_case,
                                  nstages, padded, rnd,
                                  sharded_kv, softmax_reference, spatial_inputs, spatial_ref, temporal_ref, ulp)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as _ops
    lib.load()
    return _ops


def dev():
    return torch.device("cuda:0")


def cpu(t):
    return None if t is None else t.detach().cpu()


# ==================================================================================================================
# Tap-GEMM
# ==================================================================================================================
@pytest.mark.parametrize("case", gemm_cases(), ids=case_id)
def test_gemm_sweep(ops, case):
    """Every (tile width, epilogue variant) instantiation on one case of the edge table (tokens < 128 or not a multiple
    of 128, N below / not a multiple of tile_n, K = 64, partial 7 x 5 x 3 boxes, strided A / out / residuals, fp32 and
    bf16 outputs, in-place residual, halo rows with fused statistics, more tiles than SMs with a ring phase carry).
    Catches a wrong column / row mask, a dropped or doubled epilogue term (bias not scaled by s_acc, a residual read at
    the wrong stride, a row vector indexed by the wrong token), a stage / phase slip between tiles: each is an O(1)
    error on whole rows or columns against a bound of one fp16 ulp.  The twin runs on the same inputs (same seeds) on
    the CPU and meets the same bound."""
    check_gemm_case(case, ops.gemm, dev())
    check_gemm_case(case, fake_ops.gemm, CPU)


def _variant_of(args: str):
    vals = [a.strip() for a in args.split(",")]
    norm = [1 if v == "true" else 0 if v == "false" else int(v) for v in vals]
    tn, rest = norm[0], tuple(norm[1:]) + (0,) * (7 - len(norm))
    for v, va in VARIANT_ARGS.items():
        if va == rest:
            return tn, v
    raise AssertionError(f"unknown tapgemm_kernel instantiation <{args}>")


def test_gemm_sweep_launches_every_instantiation(ops):
    """Runs the sweep under torch.profiler and reads back the demangled tapgemm_kernel<...> names: the set launched must
    be every (width, variant) pair the launcher can select (100).  A launcher that maps a feature set to the wrong
    variant index, or a table entry that never reaches its kernel, shows up as a missing or extra pair."""
    from torch.profiler import ProfilerActivity, profile
    cases = gemm_cases(small=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in cases:
            check_gemm_case(c, ops.gemm, dev())
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    kernels = [n for n in names if "tapgemm_kernel" in n]
    assert kernels, "the profiler returned no tapgemm_kernel events"
    launched = set()
    for n in kernels:
        m = re.search(r"tapgemm_kernel<([^>]*)>", n)
        if m is None:          # a mangled name: tapgemm_kernelILi128ELi0ELb0ELi1ELb0ELb0ELb0E...
            m2 = re.search(r"tapgemm_kernelI((?:L[ib]\d+E)+)", n)
            assert m2, n
            launched.add(_variant_of(",".join(re.findall(r"L[ib](\d+)E", m2.group(1)))))
        else:
            launched.add(_variant_of(m.group(1)))
    want = expected_instantiations()
    assert launched == want, f"missing {sorted(want - launched)}, unexpected {sorted(launched - want)}"


def test_gemm_sweep_phase_carry_tiles(ops):
    """The sweep really runs the persistent tile loop with a ring phase carry on at least three widths: cases with more
    tiles than this GPU has SMs and a K-chunk count that is not a multiple of the ring depth.  The tile and chunk counts
    are derived from the arguments each case passes, so an edit of the table cannot drop the edge unnoticed."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    widths = set()
    for c in gemm_cases():
        d = make_gemm_case(c, CPU)
        kw = d["kw"]
        if kw["geom"] is None:
            m_tiles = -(-d["M"] // 128)
        else:
            W, H, NB = kw["geom"]
            bw, bh, bb = ops.pick_box(W, H, NB) if kw.get("stats") is None else ops.stats_box(W, H, NB)
            m_tiles = -(-W // bw) * -(-H // bh) * -(-NB // bb)
        tiles = m_tiles * -(-d["N"] // c["tn"])
        kc = d["K"] // 64
        if tiles > sms and kc % nstages(c["tn"]):
            widths.add(c["tn"])
    assert len(widths) >= 3, widths


def test_gemm_production_conv_sampled(ops):
    """The UNet level-0 3x3 convolution at production size (2 x 25 frames of 72 x 128, 320 -> 320, K 2880) against fp64
    over a sampled token set holding every boundary class: all four image borders, the first and the last token, and
    the whole last m-tile.  A mistake in the 4-D box arithmetic at one border or in the last tile corrupts exactly those
    rows, which a strided subsample or a block mean of the full output would dilute."""
    W, H, NB, C = 128, 72, 50, 320
    g = torch.Generator(device=dev()).manual_seed(5)
    a = torch.randn(NB * H * W, C, generator=g, device=dev()).half()
    w = (torch.randn(C, 9 * C, generator=g, device=dev()) * (9 * C) ** -0.5).half()
    bias = torch.randn(C, generator=g, device=dev())
    emb = torch.randn(NB, C, generator=g, device=dev())
    res = torch.randn(NB * H * W, C, generator=g, device=dev()).half()
    out = torch.empty(NB * H * W, C, dtype=torch.float16, device=dev())
    kw = dict(taps=ops.TAPS_3X3, geom=(W, H, NB), bias=bias, rowvec=emb, rv_div=H * W, rv_mod=NB, res1=res)
    ops.gemm(a, w, out, **kw)
    torch.cuda.synchronize()
    bw, bh, bb = ops.pick_box(W, H, NB)
    tw, th, tb = -(-W // bw), -(-H // bh), -(-NB // bb)
    idx = lambda b, h, w_: ((b * H + h) * W + w_).reshape(-1)
    ar = torch.arange
    sets = [torch.randperm(NB * H * W, generator=torch.Generator().manual_seed(6))[:2048].to(dev())]
    for b in (0, NB // 2, NB - 1):
        sets += [idx(torch.tensor(b), torch.tensor(0), ar(W)), idx(torch.tensor(b), torch.tensor(H - 1), ar(W)),
                 idx(torch.tensor(b), ar(H), torch.tensor(0)), idx(torch.tensor(b), ar(H), torch.tensor(W - 1))]
    lb, lh, lw = ar((tb - 1) * bb, NB), ar((th - 1) * bh, H), ar((tw - 1) * bw, W)
    sets.append(((lb[:, None, None] * H + lh[None, :, None]) * W + lw[None, None, :]).reshape(-1))
    sets.append(torch.tensor([0, NB * H * W - 1]))
    rows = torch.unique(torch.cat([s.to(dev()) for s in sets]))
    ref, mag = gemm_reference(a, w, rows=rows, **kw)
    assert_conform(out[rows], ref, mag, FAMILY["gemm"].c_acc * math.sqrt(9 * C) * U24, "gemm", "level-0 conv")


def test_gemm_rejects_operands_the_kernel_would_misread(ops):
    """The kernel reads residuals as 16-bit values even for an fp32 output, and bias / row vector as fp32: other dtypes
    would be reinterpreted silently.  ops.gemm refuses them, and GEGLU with an s_acc it would ignore."""
    a = rnd((128, 64), 1, dev())
    w = rnd((64, 64), 2, dev())
    out32 = torch.empty(128, 64, dtype=torch.float32, device=dev())
    with pytest.raises(AssertionError):
        ops.gemm(a, w, out32, res1=torch.zeros(128, 64, device=dev()))
    with pytest.raises(AssertionError):
        ops.gemm(a, w, out32, bias=torch.zeros(64, dtype=torch.float16, device=dev()))
    with pytest.raises(AssertionError):
        ops.gemm(a, w, out32, rowvec=torch.zeros(1, 64, dtype=torch.float16, device=dev()))
    with pytest.raises(AssertionError):
        ops.gemm(a, w, torch.empty(128, 32, dtype=torch.float16, device=dev()), act=2, tile_n=64, s_acc=0.5)


# ==================================================================================================================
# Frame-sharded kernels on one GPU (simulated ranks)
# ==================================================================================================================
def _shards(T, world):
    from vista_b200.parallel import frame_shards
    return frame_shards(T, world)


@pytest.mark.parametrize("nb,T,S,heads,world", [(2, 25, 40, 2, 2), (1, 25, 24, 5, 3), (2, 7, 16, 1, 4), (1, 4, 32, 2, 4),
                                                (2, 25, 20, 1, 1),
                                                # many items per warp with Tq < T: the reused Q tile
                                                (2, 25, 2304, 5, 3)])
def test_attention_temporal_sharded(ops, nb, T, S, heads, world):
    """attention_temporal_sharded on every simulated rank of an uneven split (Tq = 1 with 4 frames on 4 ranks, Tq = T on
    one rank), K|V gathered into T_pad-padded slabs with NaN padding and addressed through the frame table built like
    ShardedUNetRuntime._frame_table.  A wrong table row, a padded slot read, or a query row confused with a key row gives
    a NaN or an attention over the wrong frames (O(1)); the largest case runs ~3 items per warp with Tq < T, where
    stale Q-tile rows from the previous item would surface if they reached a stored row."""
    C = heads * 64
    qkv = rnd((nb * T * S, 3 * C), 71, dev())
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    ref, mag = temporal_ref(q, k, v, nb, T, S, heads)
    shards = _shards(T, world)
    kv, tab = sharded_kv(k, v, nb, T, S, C, shards, dev())
    q4 = q.reshape(nb, T, S, C)
    small = nb * T * S <= 4096
    for s0, e in shards:
        Tq = e - s0
        qr = q4[:, s0:e].reshape(nb * Tq * S, C)
        out = torch.full((nb * Tq * S, C), float("nan"), dtype=torch.float16, device=dev())
        ops.attention_temporal_sharded(qr, kv[:, :C], kv[:, C:], out, nb, Tq, T, S, heads, tab)
        torch.cuda.synchronize()
        rows = lambda t: t.reshape(nb, T, S, C)[:, s0:e].reshape(-1, C)
        assert_conform(out, rows(ref), rows(mag), ATTN_EPS, "attn", f"sharded W={world} [{s0},{e})")
        if small:
            tw = torch.empty(nb * Tq * S, C, dtype=torch.float16)
            fake_ops.attention_temporal_sharded(cpu(qr), cpu(kv[:, :C]), cpu(kv[:, C:]), tw, nb, Tq, T, S, heads, cpu(tab))
            assert_conform(tw, cpu(rows(ref)), cpu(rows(mag)), ATTN_EPS, "attn", "sharded twin")


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_sums_finalize_sharded(ops, world, silu):
    """Frame-sharded temporal GroupNorm: every rank's groupnorm_sums over its frames, added in fp64 in rank order, then
    groupnorm_finalize_apply per rank == fp64 group_norm over the whole clip.  A sum over the wrong frames / groups, a
    count that is not the clip's, or a finalize indexed per rank instead of per clip moves mean or rstd by O(1)."""
    nb, T, hw, C, G = 2, 25, 48, 320, 32
    x = (rnd((nb * T * hw, C), 81, dev(), dtype=torch.float32) * 2 + 0.7).half()
    gamma = rnd((C,), 82, dev(), dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 83, dev(), dtype=torch.float32) * 0.1
    ref, mag, extra = groupnorm_reference(x, nb * T, hw, gamma, beta, 1e-5, silu, T)
    x4 = x.reshape(nb, T, hw, C)
    shards = _shards(T, world)
    total = torch.zeros(nb * G, 2, dtype=torch.float64, device=dev())
    parts = []
    for s0, e in shards:
        xr = x4[:, s0:e].reshape(-1, C)
        sums = torch.empty(nb * G, 2, dtype=torch.float64, device=dev())
        ops.groupnorm_sums(xr, nb * (e - s0), hw, C, sums, e - s0, groups=G)
        total += sums
        parts.append(xr)
    count = float(C // G) * hw * T
    eps_n = FAMILY["norm"].c_acc * math.sqrt(T * hw * C // G) * U24
    for (s0, e), xr in zip(shards, parts):
        y = torch.empty_like(xr)
        st = torch.empty(nb, G, 2, dtype=torch.float32, device=dev())
        ops.groupnorm_finalize_apply(xr, y, nb * (e - s0), hw, gamma, beta, 1e-5, silu, total, count, st, e - s0, groups=G)
        torch.cuda.synchronize()
        rows = lambda t: t.reshape(nb, T, hw, C)[:, s0:e].reshape(-1, C)
        assert_conform(y, rows(ref), rows(mag), eps_n, "norm", f"sharded GN W={world} [{s0},{e})", extra=rows(extra))
        tw = torch.empty(xr.shape, dtype=torch.float16)
        fake_ops.groupnorm_finalize_apply(cpu(xr), tw, nb * (e - s0), hw, cpu(gamma), cpu(beta), 1e-5, silu, cpu(total),
                                          count, None, e - s0, groups=G)
        assert_conform(tw, cpu(rows(ref)), cpu(rows(mag)), eps_n, "norm", "sharded GN twin", extra=cpu(rows(extra)))


@pytest.mark.parametrize("world", [2, 3])
def test_groupnorm_from_partials_raw_sums_sharded(ops, world):
    """The same with the statistics taken in the epilogue of the producing GEMM: per rank a STATS GEMM writes its
    output and column partials, groupnorm_from_partials(raw_sums=...) turns them into fp64 sums, the ranks' sums are
    added in rank order and finalised.  Must equal fp64 group_norm over the whole clip of the stored GEMM outputs (the
    partials describe the stored values)."""
    nb, T, hw, Cin, C, G = 2, 9, 128, 64, 320, 32
    x = rnd((nb * T * hw, Cin), 91, dev())
    w = rnd((C, Cin), 92, dev(), scale=Cin ** -0.5)
    bias = rnd((C,), 93, dev(), dtype=torch.float32)
    gamma = rnd((C,), 94, dev(), dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 95, dev(), dtype=torch.float32) * 0.1
    x4 = x.reshape(nb, T, hw, Cin)
    shards = _shards(T, world)
    total = torch.zeros(nb * G, 2, dtype=torch.float64, device=dev())
    outs = []
    for s0, e in shards:
        B = nb * (e - s0)
        xr = x4[:, s0:e].reshape(-1, Cin)
        o = torch.empty(B * hw, C, dtype=torch.float16, device=dev())
        part = torch.zeros(B * hw // 128 * 4, C, 2, dtype=torch.float32, device=dev())
        ops.gemm(xr, w, o, bias=bias, stats=part)
        sums = torch.empty(nb * G, 2, dtype=torch.float64, device=dev())
        ops.groupnorm_from_partials(part, B, hw, C, 1e-5, None, e - s0, G, raw_sums=sums)
        total += sums
        outs.append(o)
    o_full = torch.cat([o.reshape(nb, -1, hw, C) for o in outs], dim=1).reshape(-1, C)
    ref, mag, extra = groupnorm_reference(o_full, nb * T, hw, gamma, beta, 1e-5, True, T)
    count = float(C // G) * hw * T
    eps_n = FAMILY["norm"].c_acc * math.sqrt(T * hw * C // G) * U24
    for (s0, e), o in zip(shards, outs):
        y = torch.empty_like(o)
        st = torch.empty(nb, G, 2, dtype=torch.float32, device=dev())
        ops.groupnorm_finalize_apply(o, y, nb * (e - s0), hw, gamma, beta, 1e-5, True, total, count, st, e - s0, groups=G)
        torch.cuda.synchronize()
        rows = lambda t: t.reshape(nb, T, hw, C)[:, s0:e].reshape(-1, C)
        assert_conform(y, rows(ref), rows(mag), eps_n, "norm", f"from_partials W={world} [{s0},{e})", extra=rows(extra))


@pytest.mark.parametrize("world", [2, 3, 4])
def test_halo_correction_in_place(ops, world):
    """The frame-sharded (3,1,1) convolution without halo slots: each rank convolves its frames (zero padded at the
    shard ends), then the in-place correction GEMMs (res1 is out, read with __ldg by the kernel that overwrites it) add
    the neighbours' boundary frames through taps 0 and 2.  First and last frames must equal the full-clip convolution:
    a correction that reads its residual after its own store, or adds the wrong tap, is off by a whole tap (O(1))."""
    nb, T, hw, C = 2, 11, 96, 128
    x = rnd((nb * T * hw, C), 101, dev())
    w = rnd((C, 3 * C), 102, dev(), scale=(3 * C) ** -0.5)
    bias = rnd((C,), 103, dev(), dtype=torch.float32)
    s_acc = 0.4
    ref, mag = gemm_reference(x, w, taps=ops.TAPS_T3, geom=(hw, T, nb), bias=bias, s_acc=s_acc)
    w0, w2 = w[:, :C].contiguous(), w[:, 2 * C:].contiguous()
    x4 = x.reshape(nb, T, hw, C)
    shards = _shards(T, world)
    for r, (s0, e) in enumerate(shards):
        Tl = e - s0
        out = torch.empty(nb * Tl * hw, C, dtype=torch.float16, device=dev())
        xl = x4[:, s0:e].reshape(-1, C)
        ops.gemm(xl, w, out, taps=ops.TAPS_T3, geom=(hw, Tl, nb), bias=bias, s_acc=s_acc)
        # the boundary frames are stored twice: the main launch rounds the partial sum (without the neighbour's tap) to
        # fp16 before the correction adds that tap, so those rows also carry one fp16 ulp of the partial value
        part, _ = gemm_reference(xl, w, taps=ops.TAPS_T3, geom=(hw, Tl, nb), bias=bias, s_acc=s_acc)
        extra = torch.zeros_like(part).reshape(nb, Tl, hw, C)
        p4 = ulp(part, torch.float16).reshape(nb, Tl, hw, C)
        if r > 0:
            extra[:, 0] = p4[:, 0]
        if r < world - 1:
            extra[:, Tl - 1] = p4[:, Tl - 1]
        ov = out.reshape(nb, Tl, hw, C)
        for b in range(nb):
            if r > 0:
                o = ov[b, 0]
                ops.gemm(x4[b, s0 - 1], w0, o, s_acc=s_acc, res1=o)
            if r < world - 1:
                o = ov[b, Tl - 1]
                ops.gemm(x4[b, e], w2, o, s_acc=s_acc, res1=o)
        torch.cuda.synchronize()
        rows = lambda t: t.reshape(nb, T, hw, C)[:, s0:e].reshape(-1, C)
        # L2: the boundary frames' extra rounding (above) on top of the usual factor
        assert_conform(out, rows(ref), rows(mag), FAMILY["gemm"].c_acc * math.sqrt(3 * C) * U24, "gemm",
                       f"halo W={world} rank {r}", factor=2 * FAMILY["gemm"].factor, extra=extra.reshape(-1, C))


# ==================================================================================================================
# Attention
# ==================================================================================================================
@pytest.mark.parametrize("frames,seq,heads", SPATIAL_CASES)
def test_attention_spatial_edges(ops, frames, seq, heads):
    """seq 1 / 64 / 127 / 128 / 129 / 257 (a last key block of one key, query tiles of one row), separate q / k / v with
    different row strides, output into a column slice whose neighbours hold a sentinel.  A key mask off by one admits a
    zero-padded key (weight exp(0 - max), O(1/seq)); a wrong stride mixes rows; a store without the column bound
    overwrites the sentinel."""
    C = heads * 64
    q, k, v = spatial_inputs(frames, seq, heads, dev(), seed=111)
    obuf = torch.full((frames * seq, C + 128), 3.0, dtype=torch.float16, device=dev())
    out = obuf[:, 64:64 + C]
    ops.attention_spatial(q, k, v, out, frames, seq, heads)
    torch.cuda.synchronize()
    ref, mag = spatial_ref(q, k, v, frames, seq, heads)
    assert_conform(out, ref, mag, ATTN_EPS, "attn", f"spatial {frames}x{seq}x{heads}")
    assert bool((obuf[:, :64] == 3.0).all()) and bool((obuf[:, 64 + C:] == 3.0).all()), "sentinel columns overwritten"
    tw = torch.empty(frames * seq, C, dtype=torch.float16)
    fake_ops.attention_spatial(cpu(q), cpu(k), cpu(v), tw, frames, seq, heads)
    assert_conform(tw, cpu(ref), cpu(mag), ATTN_EPS, "attn", "spatial twin")


def test_attention_spatial_identical_keys(ops):
    """Identical keys: every weight is equal, the output is the mean of V exactly up to rounding.  A running-max rescale
    applied twice or a missing final normalisation breaks the mean (O(1))."""
    frames, seq, heads = 2, 300, 2
    C = heads * 64
    q, _, v = spatial_inputs(frames, seq, heads, dev(), seed=121)
    k = rnd((1, C), 122, dev(), scale=3.0).expand(frames * seq, C).contiguous()
    out = torch.empty(frames * seq, C, dtype=torch.float16, device=dev())
    ops.attention_spatial(q, k, v, out, frames, seq, heads)
    torch.cuda.synchronize()
    vm = v.double().reshape(frames, seq, C).mean(1, keepdim=True).expand(frames, seq, C).reshape(-1, C)
    mag = v.double().abs().reshape(frames, seq, C).mean(1, keepdim=True).expand(frames, seq, C).reshape(-1, C)
    assert_conform(out, vm, mag, ATTN_EPS, "attn", "identical keys")


def test_attention_spatial_level0_sampled(ops):
    """The level-0 sequence, 9216 = 72 x 128 tokens, 2 frames, 5 heads, against fp64 over 700 sampled query rows per
    (frame, head): rows of both consumer warpgroups (0-63, 64-127 of a block) and the whole last block.  An error
    confined to tail tiles, or to one warpgroup, is held to the element bound here instead of being diluted in a
    full-step golden."""
    frames, seq, heads = 2, 9216, 5
    C = heads * 64
    qkv = rnd((frames * seq, 3 * C), 131, dev())
    out = torch.empty(frames * seq, C, dtype=torch.float16, device=dev())
    ops.attention_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, frames, seq, heads)
    torch.cuda.synchronize()
    rows = torch.unique(torch.cat([torch.arange(0, 128), torch.arange(seq - 128, seq), torch.arange(4096, 4224),
                                   torch.randperm(seq, generator=torch.Generator().manual_seed(7))[:400]])).to(dev())
    assert rows.numel() >= 512
    ref, mag = spatial_ref(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], frames, seq, heads, rows=rows)
    got = out.reshape(frames, seq, C)[:, rows].reshape(-1, C)
    assert_conform(got, ref, mag, ATTN_EPS, "attn", "spatial 9216")


@pytest.mark.parametrize("nb,T,S,heads", [(2, t, 12, 2) for t in TEMPORAL_T] + [(2, 25, 2304, 5), (1, 25, 9216, 5)])
def test_attention_temporal_conformance(ops, nb, T, S, heads):
    """T from 1 to 32 (key masks at 8 / 16 / 24 / 32 boundaries) and the production shapes (2, 25, 2304, 5) and
    (1, 25, 9216, 5), where the grid (16 blocks x 4 warps per SM) is smaller than the item count and every warp walks
    several items.  A mask off by one admits a zero key (weight e^0); an item stride error leaves rows unwritten (the
    output starts as NaN)."""
    C = heads * 64
    qkv = rnd((nb * T * S, 3 * C), 141 + T, dev())
    out = torch.full((nb * T * S, C), float("nan"), dtype=torch.float16, device=dev())
    ops.attention_temporal(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, nb, T, S, heads)
    torch.cuda.synchronize()
    ref, mag = temporal_ref(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], nb, T, S, heads)
    assert_conform(out, ref, mag, ATTN_EPS, "attn", f"temporal {nb}x{T}x{S}x{heads}")
    if S <= 12:
        tw = torch.empty(nb * T * S, C, dtype=torch.float16)
        q, k, v = (cpu(t) for t in (qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]))
        fake_ops.attention_temporal(q, k, v, tw, nb, T, S, heads)
        assert_conform(tw, cpu(ref), cpu(mag), ATTN_EPS, "attn", "temporal twin")


# ==================================================================================================================
# Norms, softmax, im2col
# ==================================================================================================================
@pytest.mark.parametrize("tokens,C", LN_CASES)
@pytest.mark.parametrize("addvec", [False, True])
def test_layernorm_conformance(ops, tokens, C, addvec):
    """Both LayerNorm kernels: layernorm40 at C = 320 / 640 / 1280 (4 / 2 / 1 rows per warp) with token counts that leave
    a warp's rows partly dead (1, 3, 5 tokens) or run the grid-stride loop (20001, 9217), and the generic kernel at
    NV 1 / 2 / 3 / 5 / 10; strided x and y, with and without the row-indexed add vector.  A dead row that stores, a
    shuffle that mixes two rows of a warp, or a grid stride that skips rows is an O(1) error."""
    x = padded(tokens, C, 16, 151, dev(), scale=1.5, offset=8)
    x.sub_(0.3)                                            # in place: x stays a strided view (row stride C + 16)
    assert x.stride(0) == C + 16
    gamma = rnd((C,), 152, dev(), dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 153, dev(), dtype=torch.float32) * 0.1
    add = rnd((5, C + 4), 154, dev(), dtype=torch.float32)[:, :C] if addvec else None
    ybuf = torch.full((tokens, C + 24), 5.0, dtype=torch.float16, device=dev())
    y = ybuf[:, 16:16 + C]
    ops.layernorm(x, y, gamma, beta, 1e-5, addvec=add, av_div=3, av_mod=5)
    torch.cuda.synchronize()
    ref, mag = layernorm_reference(x, gamma, beta, 1e-5, add, 3, 5)
    eps = FAMILY["norm"].c_acc * math.sqrt(C) * U24
    assert_conform(y, ref, mag, eps, "norm", f"layernorm {tokens}x{C}")
    assert bool((ybuf[:, :16] == 5.0).all()) and bool((ybuf[:, 16 + C:] == 5.0).all())
    if tokens <= 1024:
        tw = torch.empty(tokens, C, dtype=torch.float16)
        fake_ops.layernorm(cpu(x), tw, cpu(gamma), cpu(beta), 1e-5, addvec=cpu(add), av_div=3, av_mod=5)
        assert_conform(tw, cpu(ref), cpu(mag), eps, "norm", "layernorm twin")


@pytest.mark.parametrize("frames,tpf,C,fps", GN_CASES)
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_conformance(ops, frames, tpf, C, fps, silu):
    """GroupNorm with J = 1 and 2 (C 2560), tokens per frame below kGnMinChunk and not a multiple of 8 (9, 13), strided
    x and y, an input with |mean| / std ~ 30 (the E[x^2] - mean^2 cancellation), and two shapes back to back on one
    workspace, so the self-resetting ticket counters of the first launch must be back at zero for the second.  A counter
    left dirty finalises too early (statistics of a partial sum, O(1)); a lost chunk shifts the mean by its share."""
    from vista_b200.ops import GNWorkspace
    ws = GNWorkspace(dev())
    gamma = rnd((C,), 162, dev(), dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 163, dev(), dtype=torch.float32) * 0.1
    n = fps * tpf * C // 32
    eps = FAMILY["norm"].c_acc * math.sqrt(n) * U24
    # a warm-up shape on the same workspace first: its counters must reset themselves
    xw = rnd((3 * 100, C), 164, dev())
    ops.groupnorm(xw, torch.empty_like(xw), 3, 100, gamma, beta, 1e-5, silu, frames_per_stat=1, ws=ws)
    for offset in (0.7, 30.0):
        x = (padded(frames * tpf, C, 8, 161, dev(), dtype=torch.float32) + offset).half()
        xs = torch.zeros(frames * tpf, C + 16, dtype=torch.float16, device=dev())
        xs[:, 8:8 + C] = x
        xv = xs[:, 8:8 + C]
        assert xv.stride(0) == C + 16
        ybuf = torch.full((frames * tpf, C + 8), 5.0, dtype=torch.float16, device=dev())
        y = ybuf[:, :C]
        ops.groupnorm(xv, y, frames, tpf, gamma, beta, 1e-5, silu, frames_per_stat=fps, ws=ws)
        torch.cuda.synchronize()
        ref, mag, extra = groupnorm_reference(xv, frames, tpf, gamma, beta, 1e-5, silu, fps)
        assert_conform(y, ref, mag, eps, "norm", f"groupnorm {frames}x{tpf}x{C} fps {fps} mean {offset}", extra=extra)
        assert bool((ybuf[:, C:] == 5.0).all())
        tw = torch.empty(frames * tpf, C, dtype=torch.float16)
        fake_ops.groupnorm(cpu(xv), tw, frames, tpf, cpu(gamma), cpu(beta), 1e-5, silu, frames_per_stat=fps)
        assert_conform(tw, cpu(ref), cpu(mag), eps, "norm", "groupnorm twin", extra=cpu(extra))


@pytest.mark.parametrize("rows,cols", SOFTMAX_CASES)
def test_softmax_rows_conformance(ops, rows, cols):
    """The decoder mid-attention row softmax at 4, 1028 and 9216 columns (one block per row, 256 threads x 4 columns),
    with one row of large logits (|x| ~ 160): a max taken over part of the row overflows exp or leaves the row
    unnormalised (O(1)); strided input and output."""
    x = padded(rows, cols, 4, 171, dev(), dtype=torch.float32)
    x[0] *= 40.0
    assert x.stride(0) == cols + 4
    ybuf = torch.full((rows, cols + 8), 5.0, dtype=torch.float16, device=dev())
    y = ybuf[:, :cols]
    ops.softmax_rows(x, y)
    torch.cuda.synchronize()
    ref, mag = softmax_reference(x)
    eps = FAMILY["softmax"].c_acc * math.sqrt(cols) * U24
    assert_conform(y, ref, mag, eps, "softmax", f"softmax {rows}x{cols}")
    assert bool((ybuf[:, cols:] == 5.0).all())
    tw = torch.empty(rows, cols, dtype=torch.float16)
    fake_ops.softmax_rows(cpu(x), tw)
    assert_conform(tw, cpu(ref), cpu(mag), eps, "softmax", "softmax twin")


@pytest.mark.parametrize("NB,H,W,C", IM2COL_CASES)
def test_im2col_s2_asym_exact(ops, NB, H, W, C):
    """The encoder Downsample gather: exactly F.pad(x, (0,1,0,1)) followed by a stride-2 3x3 unfold, odd and even H and W
    (the right / bottom zero column appears only for odd sizes), from a strided x."""
    x = padded(NB * H * W, C, 16, 181, dev(), offset=8)
    assert x.stride(0) == C + 16
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    out = torch.full((NB * Ho * Wo, 9 * C), 5.0, dtype=torch.float16, device=dev())
    ops.im2col_s2_asym(x, out, NB, H, W, C)
    torch.cuda.synchronize()
    want = im2col_asym_reference(x, NB, H, W, C)
    assert torch.equal(out, want)
    tw = torch.empty(NB * Ho * Wo, 9 * C, dtype=torch.float16)
    fake_ops.im2col_s2_asym(cpu(x), tw, NB, H, W, C)
    assert torch.equal(tw, cpu(want))
