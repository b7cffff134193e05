"""Conformance of the operators against fp64 references: the case tables, the references, the tolerance rule, and the
CPU run of every table with the operator twin of tests/fake_ops.py standing in for the kernel.

tests/test_conformance_gpu.py runs the same tables on the kernels (and the twins beside them, on the same inputs).  Here
they check the reference code and the twins before any GPU time is spent: a twin that drifts from the operator it
models would let the CPU executor suite check host code against a wrong model.

Tolerance rule (one per operator family, see FAMILY):
  * every element: |out - ref| <= ulp_out(|ref|) + eps * mag, where ulp_out is one unit in the last place of the output
    type at |ref| (the rounding of the store, with room for a pre-rounding value that is itself slightly off), mag an
    fp64 magnitude of the operation's terms (|A|.|W| for a GEMM) and eps the family's accumulation factor;
  * the whole output: rel-L2(out) <= factor * rel-L2(ref rounded to the 16-bit output type), the rounding nobody can
    avoid.
Pure data movement must match exactly."""
import math

import pytest
import torch
import torch.nn.functional as F

import fake_ops

U24 = 2.0 ** -24


class Family:
    def __init__(self, c_acc: float, factor: float, why: str):
        self.c_acc, self.factor, self.why = c_acc, factor, why


FAMILY = {
    # fp32 accumulation (random walk, sqrt(K)); the store rounds a value already off by that error: <= 2x the bare rounding
    "gemm": Family(8.0, 2.0, "fp32 accumulation over K, then one rounding of the store"),
    # P is rounded to fp16 (half an ulp per weight, 2^-25 absolute below 2^-14) before P.V; O rounds once more
    "attn": Family(2.0, 4.0, "P rounded to fp16 before P.V, on top of the output rounding"),
    # fp32 statistics over n elements, fp32 normalisation, one rounding of the store
    "norm": Family(8.0, 2.0, "fp32 statistics over n elements, then one rounding of the store"),
    # __expf (ex2.approx, relative ~2^-22) and an fp32 sum over the row, one rounding of the store
    "softmax": Family(8.0, 2.0, "approximate exp and an fp32 row sum, then one rounding of the store"),
    # a fixed, short chain of fp32 operations per element (sampler step, time mix, embeddings): eps counts its roundings
    # (and the documented ulp errors of rsqrtf / logf / expf / cosf / sinf), derived next to each operation's reference
    "elementwise": Family(1.0, 2.0, "a few fp32 operations per element, each rounding counted in eps, then the store"),
}


def ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """One unit in the last place of `dtype` at |x| (fp64), subnormals included."""
    mant, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}[dtype]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin)))
    return torch.exp2(e - mant)


def rel_l2(a: torch.Tensor, ref: torch.Tensor) -> float:
    return float((a.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def assert_conform(out: torch.Tensor, ref: torch.Tensor, mag: torch.Tensor, eps: float, family: str, name: str,
                   factor: float = None, extra: torch.Tensor = None):
    """The tolerance rule: element bound ulp_out(|ref|) + eps * mag and rel-L2 <= factor * rel-L2(ref rounded to 16
    bits).  fp32 outputs are held to an fp32 ulp per element and to the fp16 rounding in L2.  ``extra``: a per-element
    term for a rounding the operation itself performs before the last one (stated where it is passed)."""
    fam = FAMILY[family]
    factor = fam.factor if factor is None else factor
    o = out.double()
    assert o.shape == ref.shape, (name, o.shape, ref.shape)
    assert bool(torch.isfinite(o).all()), f"{name}: non-finite output"
    err = (o - ref).abs()
    tol = ulp(ref, out.dtype) + eps * mag
    if extra is not None:
        tol = tol + extra
    bad = err > tol
    if bool(bad.any()):
        i = int(torch.argmax(err - tol))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; worst flat index {i}: "
                             f"out {float(o.flatten()[i]):.6g} ref {float(ref.flatten()[i]):.6g} "
                             f"err {float(err.flatten()[i]):.3g} tol {float(tol.flatten()[i]):.3g}")
    r16 = torch.bfloat16 if out.dtype == torch.bfloat16 else torch.float16
    floor = rel_l2(ref.to(r16), ref)
    rel = rel_l2(o, ref)
    assert rel <= factor * floor + 1e-12, f"{name}: rel-L2 {rel:.3g} > {factor} x rounding floor {floor:.3g}"
    return rel


def gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cpu").manual_seed(seed)


def rnd(shape, seed, device, scale=1.0, dtype=torch.float16):
    return (torch.randn(*shape, generator=gen(seed)) * scale).to(dtype).to(device)


def padded(rows: int, cols: int, extra: int, seed: int, device, scale=1.0, dtype=torch.float16, offset=0):
    """[rows, cols] view at column `offset` of a [rows, cols + extra] buffer (row stride cols + extra) filled with random
    values: a strided operand."""
    buf = rnd((rows, cols + extra), seed, device, scale, dtype)
    return buf[:, offset:offset + cols]


# ==================================================================================================================
# Tap-GEMM (b200v_gemm)
# ==================================================================================================================
WIDTHS = (32, 64, 96, 128, 160, 192, 224, 256)
# Epilogue variants of gemm_tc.cuh: (ACT, RV, NRES, GEN, STATS, BF16) template arguments of tapgemm_kernel
VARIANT_ARGS = {0: (0, 0, 0, 0, 0, 0), 1: (0, 0, 1, 0, 0, 0), 2: (0, 0, 2, 0, 0, 0), 3: (0, 1, 0, 0, 0, 0),
                4: (0, 1, 1, 0, 0, 0), 5: (1, 0, 0, 0, 0, 0), 6: (2, 0, 0, 0, 0, 0), 7: (0, 1, 2, 1, 0, 0),
                8: (3, 0, 0, 0, 0, 0), 9: (0, 0, 0, 0, 1, 0), 10: (0, 0, 1, 0, 1, 0), 11: (0, 1, 0, 0, 1, 0),
                12: (0, 1, 2, 1, 0, 1)}


def nstages(tn: int) -> int:
    """Ring depth the launcher picks for tile width tn (gemm_tc.cu)."""
    stage = 128 * 64 * 2 + ((tn * 128 + 1023) // 1024) * 1024
    return min(8, (227 * 1024 - 2048 - 2 * 2 * 64 * 32 * 4) // stage)


def expected_instantiations():
    """Every (tile width, variant) pair the launcher can select: GEGLU only at widths that are multiples of 64."""
    return {(tn, v) for tn in WIDTHS for v in range(13) if v != 6 or tn % 64 == 0}


def gemm_cases(small: bool = False):
    """One case per selectable (width, variant) pair; the geometry, N and the strides rotate over the edge classes:
      lin50    tokens < 128 with K = 64 (one K-chunk)
      lin300   tokens % 128 != 0
      conv753  3x3 convolution on a 7 x 5 x 3 image: partial boxes in W, H and NB
      many     KC = 9 (not a multiple of any ring depth) and more tiles than SMs (132 on an H100)
      tconv    (3,1,1) convolution over frames; with STATS: h_pad = 1 halo frames
    N: 'lt' N < tile_n, 'p8' N % tile_n == 8 (a last tile of 8 columns), 'eq' N == 2 tile_n.
    ``small`` shrinks the 'many' class for the CPU run."""
    geoms = ("lin50", "lin300", "conv753", "many", "tconv")
    nkinds = ("lt", "p8", "eq")
    cases = []
    i = 0
    for tn in WIDTHS:
        for v in range(13):
            if v == 6 and tn % 64:
                continue
            c = dict(tn=tn, variant=v, geom=geoms[i % 5], nkind=nkinds[(i // 5 + i) % 3], strided=bool(i % 2),
                     inplace=False, out_f32=False, bf16=(v == 12), act=0, rowvec=v in (3, 4, 11), nres=0, small=small,
                     seed=1000 + i)
            c["nres"] = {1: 1, 2: 2, 4: 1, 10: 1}.get(v, 0)
            if v == 5:
                c["act"] = 1
            elif v == 6:
                c["act"] = 2
                c["nkind"] = "eq" if i % 2 else "one"      # GEGLU: N a multiple of tile_n
            elif v == 8:
                c["act"] = 3
            elif v == 7:                                   # generic fp16: fp32 output, or SiLU with a residual
                if (tn // 32) % 2:
                    c.update(out_f32=True, act=1, rowvec=True, nres=2)
                else:
                    c.update(act=1, nres=1)
            elif v == 12:                                  # generic bf16: 16-bit and fp32 outputs
                c.update(out_f32=bool((tn // 32) % 2), rowvec=True, nres=1 + (tn // 32) % 2)
            if v in (9, 10, 11):                            # fused statistics: token tiles of 128 consecutive tokens
                c["geom"] = ("lin300", "stats_conv", "stats_halo")[i % 3]
            if v in (1, 4, 10) and tn in (64, 160, 224, 256):
                c["inplace"] = True                         # res1 is out: the sharded halo correction
            cases.append(c)
            i += 1
    # the persistent tile loop with a phase carry: force 'many' on three more widths for the plain variant
    for c in cases:
        if c["variant"] == 0 and c["tn"] in (96, 160, 224):
            c["geom"] = "many"
    return cases


def case_id(c):
    return f"tn{c['tn']}-v{c['variant']}-{c['geom']}-{c['nkind']}" + ("-inplace" if c["inplace"] else "") + \
        ("-strided" if c["strided"] else "")


def _n_of(c):
    tn = c["tn"]
    return {"lt": max(8, tn - 24), "p8": 2 * tn + 8, "eq": 2 * tn, "one": tn}[c["nkind"]]


def make_gemm_case(c, device):
    """Inputs and the ops.gemm keyword arguments of one sweep case."""
    tn, s = c["tn"], c["seed"]
    N = _n_of(c)
    if c["geom"] == "many":
        N = 4 * tn                                        # 4 n-tiles x 35 m-tiles = 140 tiles > 132 SMs
    g = c["geom"]
    taps, geom, h_pad = [(0, 0)], None, 0
    if g == "lin50":
        M, cin = 50, 64
    elif g == "lin300":
        M, cin = 300, 192
    elif g == "conv753":
        geom, cin, taps = (7, 5, 3), 64, [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]
    elif g == "many":
        M, cin = (300 if c["small"] else 35 * 128 - 88), 576
    elif g == "tconv":
        geom, cin, taps = (24, 5, 2), 128, [(-1, 0), (0, 0), (1, 0)]
    elif g == "stats_conv":
        geom, cin, taps = (16, 8, 3), 64, [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]
    elif g == "stats_halo":
        geom, cin, taps, h_pad = (128, 3, 2), 64, [(-1, 0), (0, 0), (1, 0)], 1
    if geom is not None:
        M = geom[0] * geom[1] * geom[2]
    K = cin * len(taps)
    act = c["act"]
    n_out = N // 2 if act == 2 else N
    op_dt = torch.bfloat16 if c["bf16"] else torch.float16
    out_dt = torch.float32 if c["out_f32"] else op_dt
    ex = 64 if c["strided"] else 0
    rows_a = M if not h_pad else geom[2] * (geom[1] + 2 * h_pad) * geom[0]
    a = padded(rows_a, cin, ex, s, device, dtype=op_dt, offset=ex // 2 if ex else 0)
    w = rnd((N, K), s + 1, device, scale=K ** -0.5, dtype=op_dt)
    kw = dict(taps=taps, geom=geom, h_pad=h_pad, tile_n=tn, act=act)
    kw["bias"] = rnd((N,), s + 2, device, dtype=torch.float32)
    if act != 2:
        kw["s_acc"] = 0.6
    if c["rowvec"]:
        mod = 5
        rv = torch.zeros(mod, N + 4, dtype=torch.float32, device=device)
        rv[:, :N] = rnd((mod, N), s + 3, device, dtype=torch.float32)
        kw.update(rowvec=rv[:, :N], rv_div=7, rv_mod=mod)
    out_ex = 16 if c["strided"] else 0
    obuf = torch.full((M, n_out + out_ex), 7.0, dtype=out_dt, device=device)
    out = obuf[:, out_ex // 2: out_ex // 2 + n_out]
    if c["nres"] >= 1:
        if c["inplace"]:
            out.copy_(rnd((M, n_out), s + 4, device, dtype=op_dt).to(out_dt))
            kw.update(res1=out, s_res1=0.5)
        else:
            kw.update(res1=padded(M, n_out, 24 if c["strided"] else 0, s + 4, device, dtype=op_dt), s_res1=0.5)
    if c["nres"] >= 2:
        kw.update(res2=padded(M, n_out, 40 if c["strided"] else 0, s + 5, device, dtype=op_dt, offset=8 if c["strided"] else 0),
                  s_res2=-0.75)
    if c["variant"] in (9, 10, 11):
        kw["stats"] = torch.zeros(-(-M // 128) * 4, n_out, 2, dtype=torch.float32, device=device)
    return dict(a=a, w=w, out=out, obuf=obuf, kw=kw, M=M, N=N, K=K, cin=cin, n_out=n_out)


def im2col64(a, cin, taps, geom, h_pad, rows=None, upsample=False):
    """fp64 implicit-GEMM operand [tokens (or `rows`), ntaps * cin]: out row (b, h, w) reads a[b, h + h_pad + dh, w + dw],
    zero outside the stored rows (the halo slots are real rows).  ``upsample``: the taps run over the nearest-2x
    upsampled view of ``a`` (geometry ``geom``): out row (b, y, x) of the 2H x 2W frame reads a[b, (y + dh) // 2,
    (x + dw) // 2], zero outside the upsampled frame."""
    if geom is None:
        x = a[:, :cin] if rows is None else a[rows, :cin]
        return x.double()
    W, H, NB = geom
    s = 2 if upsample else 1
    He = H + 2 * h_pad
    tok = torch.arange(W * H * NB * s * s, device=a.device) if rows is None else rows
    w, h, b = tok % (s * W), (tok // (s * W)) % (s * H), tok // (s * s * W * H)
    parts = []
    for dh, dw in taps:
        hs, ws = h + h_pad + dh, w + dw
        ok = (hs >= 0) & (hs < s * He) & (ws >= 0) & (ws < s * W)
        src = torch.where(ok, (b * He + hs.div(s, rounding_mode="floor")) * W + ws.div(s, rounding_mode="floor"),
                          torch.zeros_like(tok))
        parts.append(a[src, :cin].double() * ok[:, None])
    return torch.cat(parts, dim=1)


def gemm_reference(a, w, *, taps, geom, h_pad=0, bias=None, rowvec=None, rv_div=1, rv_mod=1, res1=None, s_res1=1.0,
                   res2=None, s_res2=1.0, s_acc=1.0, act=0, tile_n=None, stats=None, rows=None, upsample=False,
                   terms=None):
    """fp64 epilogue(tap-GEMM) and its magnitude (|A|.|W| propagated through the epilogue).  ``rows``: token subset;
    ``upsample``: the taps read the nearest-2x upsampled view of ``a`` (im2col64).  ``terms`` (a dict) receives the
    terms the output is the sum of, for the gain check of tests/bias.py: with act = 0 'acc' (s_acc acc), 'bias'
    (s_acc bias + rowvec), 'res1' and 'res2' (each times its scale); with an activation the activated part as 'ref'
    beside the residuals."""
    cin = w.shape[1] // len(taps)
    cols = im2col64(a, cin, taps, geom, h_pad, rows, upsample)
    w64 = w.double()
    acc = cols @ w64.t()
    mag = cols.abs() @ w64.abs().t()
    tok = rows if rows is not None else torch.arange(acc.shape[0], device=a.device)
    b = bias.double() if bias is not None else torch.zeros(w.shape[0], dtype=torch.float64, device=a.device)
    if act == 2:
        N = w.shape[0]
        t = (acc + b).reshape(acc.shape[0], N // tile_n, 2, tile_n // 2)
        tm = (mag + b.abs()).reshape(acc.shape[0], N // tile_n, 2, tile_n // 2)
        val, gate = t[:, :, 0], t[:, :, 1]
        gl = F.gelu(gate)
        ref = (val * gl).reshape(acc.shape[0], N // 2)
        mag = (tm[:, :, 0] * gl.abs() + val.abs() * 1.2 * tm[:, :, 1] + val.abs()).reshape(acc.shape[0], N // 2)
        if terms is not None:
            terms["ref"] = ref
        return ref, mag
    t = {"acc": s_acc * acc}
    if bias is not None:
        t["bias"] = s_acc * b
    o = t["acc"] + s_acc * b
    mag = abs(s_acc) * (mag + b.abs())
    if rowvec is not None:
        rvv = rowvec.double()[(tok // rv_div) % rv_mod]
        t["bias"] = t.get("bias", 0) + rvv
        o = o + rvv
        mag = mag + rvv.abs()
    if act == 1:
        o, mag = F.silu(o), 1.2 * mag
    elif act == 3:
        o, mag = F.gelu(o), 1.2 * mag
    if act != 0:
        t = {"ref": o}
    for name, res, sc in (("res1", res1, s_res1), ("res2", res2, s_res2)):
        if res is not None:
            r = sc * res[tok].double()
            t[name] = r
            o, mag = o + r, mag + r.abs()
    if terms is not None:
        terms.update(t)
    return o, mag


def check_gemm_case(c, op, device):
    """Runs `op` (ops.gemm or its twin) on one sweep case and holds it to the fp64 reference."""
    d = make_gemm_case(c, device)
    kw = dict(d["kw"])
    ref_kw = dict(kw)
    if c["inplace"]:
        ref_kw["res1"] = kw["res1"].clone()               # the residual is what `out` held before the launch
    obuf_before = d["obuf"].clone()
    op(d["a"], d["w"], d["out"], **kw)
    if device.type == "cuda":
        torch.cuda.synchronize()
    ref_kw.pop("stats", None)
    ref, mag = gemm_reference(d["a"], d["w"], **ref_kw)
    fam = FAMILY["gemm"]
    eps = fam.c_acc * math.sqrt(d["K"]) * U24
    name = case_id(c)
    assert_conform(d["out"], ref, mag, eps, "gemm", name)
    # columns of a strided output outside the view: untouched
    lo = d["out"].storage_offset() - d["obuf"].storage_offset()
    assert torch.equal(d["obuf"][:, :lo], obuf_before[:, :lo]), f"{name}: wrote left of the output view"
    assert torch.equal(d["obuf"][:, lo + d["n_out"]:], obuf_before[:, lo + d["n_out"]:]), f"{name}: wrote right of the view"
    if "stats" in kw:
        check_stats(kw["stats"], d["out"], name)
    return ref


def check_stats(stats, stored, name):
    """Fused GroupNorm partials against the values the kernel stored (the output, itself held to fp64 by the caller):
    per (128-token tile, 32-row quarter) of `stored` [M, N] in tile order, the column sum s and the sum of squared
    deviations from the quarter's mean.  Bound: fp32 sums of n <= 32 terms (n U24 of sum |x|, 2^-24 per term of the
    deviation sum); the kernel's mean fl(s / n) may differ from the exact one by the sum's error / n and half an fp32
    ulp, which adds n dm^2 to the deviation sum.  No term grows with mean^2: a partial that sums raw squares fails a
    column whose mean is large next to its spread."""
    v, n = quarters(stored)
    s_ref = v.sum(1)
    m = s_ref / n.clamp_min(1)
    valid = (torch.arange(32, device=v.device)[None, :] < n)[..., None]
    q_ref = torch.where(valid, (v - m[:, None]) ** 2, torch.zeros_like(v)).sum(1)
    s_tol = 32 * U24 * v.abs().sum(1) + 1e-30
    dm = s_tol / n.clamp_min(1) + ulp(m, torch.float32)
    q_tol = 36 * U24 * q_ref + n * dm * dm + 1e-30
    got = stats[: v.shape[0]].double()
    bad_s = ~((got[..., 0] - s_ref).abs() <= s_tol)
    bad_q = ~((got[..., 1] - q_ref).abs() <= q_tol)
    assert not bool(bad_s.any()), f"{name}: {int(bad_s.sum())} column-sum partials wrong"
    assert not bool(bad_q.any()), f"{name}: {int(bad_q.sum())} deviation-sum partials wrong"


def quarters(stored):
    """fp64 [quarters, 32, N] of `stored` [M, N] (zero rows past M) and the valid-row count [quarters, 1] of each."""
    M, N = stored.shape
    pad = (-M) % 128
    v = F.pad(stored.double(), (0, 0, 0, pad)).reshape(-1, 32, N)
    n = (M - 32 * torch.arange(v.shape[0], device=v.device)).clamp(0, 32).double()[:, None]
    return v, n


# ==================================================================================================================
# Attention
# ==================================================================================================================
def attention_reference(q, k, v, p_normalised: bool, scale: float = 0.125):
    """fp64 softmax(q k^T * scale) v over the last two dims (scale 1/8 for head dim 64) and its magnitude for the P
    rounding term (FAMILY['attn'], eps = 2 * 2^-12): P.|V| for the relative half-ulp of every weight, plus 2^-13 sum|V| / d
    for the absolute 2^-25 of a weight in fp16's subnormal range.  ``p_normalised``: the kernel rounds the normalised
    weights (temporal, d = 1); otherwise it rounds exp(s - running max) <= 1 and divides by the row sum afterwards
    (spatial and CLIP, d = l = sum exp(s - max), the fp64 row sum)."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.transpose(-1, -2) * scale
    e = torch.exp(s - s.max(-1, keepdim=True).values)
    l = e.sum(-1, keepdim=True)
    p = e / l
    small = 2.0 ** -13 * v.abs().sum(-2, keepdim=True)
    return p @ v, p @ v.abs() + (small if p_normalised else small / l)


ATTN_EPS = FAMILY["attn"].c_acc * 2.0 ** -12

SPATIAL_CASES = [(2, 1, 1), (2, 64, 2), (1, 127, 1), (3, 128, 1), (2, 129, 2), (1, 257, 3), (2, 576, 5)]
TEMPORAL_T = (1, 2, 8, 9, 24, 25, 31, 32)


def spatial_inputs(frames, seq, heads, device, seed):
    """Separate q / k / v buffers with different row strides (and column offsets)."""
    C = heads * 64
    q = padded(frames * seq, C, 64, seed, device, offset=64)
    k = padded(frames * seq, C, 128, seed + 1, device, offset=0)
    v = padded(frames * seq, C, 8, seed + 2, device, offset=8)
    return q, k, v


def spatial_ref(q, k, v, frames, seq, heads, rows=None):
    sp = lambda t: t.double().reshape(frames, seq, heads, 64).permute(0, 2, 1, 3)
    qq = sp(q)
    if rows is not None:
        qq = qq[:, :, rows]
    o, m = attention_reference(qq, sp(k), sp(v), p_normalised=False)
    n = o.shape[2]
    return o.permute(0, 2, 1, 3).reshape(frames * n, heads * 64), m.permute(0, 2, 1, 3).reshape(frames * n, heads * 64)


def temporal_ref(q, k, v, nb, T, S, heads):
    tp = lambda t: t.double().reshape(nb, T, S, heads, 64).permute(0, 2, 3, 1, 4)
    o, m = attention_reference(tp(q), tp(k), tp(v), p_normalised=True)
    back = lambda t: t.permute(0, 3, 1, 2, 4).reshape(nb * T * S, heads * 64)
    return back(o), back(m)


def sharded_kv(k, v, nb, T, S, C, shards, device):
    """The gathered K|V buffer of ShardedUNetRuntime: rank r's slab holds its clips' local frames, padded to T_pad frames
    (padding rows are NaN: a table entry pointing at one poisons the output), and the frame table that maps (clip, frame)
    to the first row of that frame."""
    W = len(shards)
    T_pad = max(e - s for s, e in shards)
    kv = torch.full((W * nb * T_pad * S, 2 * C), float("nan"), dtype=torch.float16, device=device)
    k4, v4 = k.reshape(nb, T, S, C), v.reshape(nb, T, S, C)
    rows = []
    for b in range(nb):
        for t in range(T):
            r = next(i for i, (s0, e) in enumerate(shards) if s0 <= t < e)
            row = ((r * nb + b) * T_pad + t - shards[r][0]) * S
            rows.append(row)
            kv[row:row + S, :C] = k4[b, t]
            kv[row:row + S, C:] = v4[b, t]
    return kv, torch.tensor(rows, dtype=torch.int64, device=device)


# ==================================================================================================================
# Norms, softmax, im2col
# ==================================================================================================================
def layernorm_reference(x, gamma, beta, eps, addvec=None, av_div=1, av_mod=1, rows=None, terms=None):
    """fp64 LayerNorm of x [tokens, >= C] (of the token subset ``rows``) and its magnitude.  ``terms`` receives the
    normalised values times gamma as 'norm' and 'beta' (tests/bias.py)."""
    C = gamma.numel()
    tok = torch.arange(x.shape[0], device=x.device) if rows is None else rows
    v = x[tok, :C].double()
    if addvec is not None:
        v = v + addvec.double()[(tok // av_div) % av_mod][:, :C]
    mean = v.mean(1, keepdim=True)
    rstd = torch.rsqrt(v.var(1, unbiased=False, keepdim=True) + eps)
    g, b = gamma.double(), beta.double()
    nrm = (v - mean) * rstd * g
    ref = nrm + b
    mag = (v.abs() + mean.abs()) * rstd * g.abs() + b.abs()
    if terms is not None:
        terms.update(norm=nrm, beta=b.expand_as(nrm))
    return ref, mag


def groupnorm_reference(x, frames, tpf, gamma, beta, eps, silu, fps, groups=32, stat_x=None, rows=None, moments=None,
                        terms=None):
    """fp64 GroupNorm of x [frames * tpf, C] with statistics over fps consecutive frames (over `stat_x` if given), its
    magnitude and an extra absolute term (assert_conform's ``mag`` and ``extra``).  ``rows`` with ``moments`` = fp64
    (mean, rstd) [frames / fps, groups]: the token subset ``rows`` only, normalised with those statistics (computed
    elsewhere over the whole frame set).

    The bound is GroupNorm's, not a kernel's: mag = |x - mean| rstd |gamma| + |beta| (times eps = c sqrt(n) U24: the
    statistics and the normalisation in fp32), extra = 4 ulp32(mean) rstd |gamma| (the fp32 mean, and the fp32 terms
    x rstd gamma and beta - mean rstd gamma of an fp32 apply, each of size |mean| rstd |gamma|, rounded: a few ulps of
    the mean, scaled); SiLU's slope is below 1.2.  Nothing grows with |mean| / std: a kernel
    that loses the variance of an offset or near-flat group to E x^2 - mean^2 in fp32 fails it.

    ``terms`` receives what the output is the sum of (tests/bias.py): 'norm' (the normalised values times gamma) and
    'beta'; with SiLU the whole output as 'ref'."""
    C = gamma.numel()
    g, b = gamma.double(), beta.double()
    if rows is not None:
        mean, rstd = (m[rows // (fps * tpf)].repeat_interleave(C // groups, dim=1) for m in moments)
        xs = x[rows, :C].double()
        nrm = (xs - mean) * rstd * g
        mag = (xs - mean).abs() * rstd * g.abs() + b.abs()
        extra = 4 * ulp(mean, torch.float32) * rstd * g.abs()
    else:
        xs = x[:, :C].double().reshape(frames // fps, fps * tpf, groups, C // groups)
        sx = xs if stat_x is None else stat_x[:, :C].double().reshape(xs.shape)
        mean = sx.mean(dim=(1, 3), keepdim=True)
        rstd = torch.rsqrt(sx.var(dim=(1, 3), unbiased=False, keepdim=True) + eps)
        nrm = ((xs - mean) * rstd).reshape(-1, C) * g
        mag = ((xs - mean).abs() * rstd).reshape(-1, C) * g.abs() + b.abs()
        extra = (4 * ulp(mean, torch.float32) * rstd).expand(xs.shape).reshape(-1, C) * g.abs()
    pre = nrm + b
    if silu:
        if terms is not None:
            terms["ref"] = F.silu(pre)
        return F.silu(pre), 1.2 * mag, 1.2 * extra
    if terms is not None:
        terms.update(norm=nrm, beta=b.expand_as(nrm))
    return pre, mag, extra


def softmax_reference(x):
    x = x.double()
    y = torch.softmax(x, dim=-1)
    return y, y * (1 + (x - x.max(-1, keepdim=True).values).abs())


def im2col_asym_reference(x, NB, H, W, C):
    """F.pad by one on the right / bottom, then a 3x3 stride-2 unfold, tap-major columns."""
    img = x[:, :C].reshape(NB, H, W, C).permute(0, 3, 1, 2).float()
    u = F.unfold(F.pad(img, (0, 1, 0, 1)), kernel_size=3, stride=2)            # (NB, C*9, L): channel-major
    L = u.shape[-1]
    return u.reshape(NB, C, 9, L).permute(0, 3, 2, 1).reshape(NB * L, 9 * C).to(x.dtype)


LN_CASES = [(1, 320), (3, 320), (5, 320), (20001, 320), (1, 640), (3, 640), (9217, 640), (1, 1280), (5, 1280),
            (333, 1280), (77, 64), (129, 512), (33, 768), (65, 1024), (17, 2560)]
GN_CASES = [(4, 9, 64, 1), (3, 13, 320, 3), (2, 300, 2560, 1), (5, 144, 640, 5)]
SOFTMAX_CASES = [(3, 4), (5, 1028), (4, 9216)]
IM2COL_CASES = [(2, 5, 7, 64), (1, 6, 8, 64), (3, 7, 6, 128), (1, 8, 9, 64)]


# ==================================================================================================================
# CPU run: the twins on the case tables
# ==================================================================================================================
CPU = torch.device("cpu")


@pytest.mark.parametrize("case", gemm_cases(small=True), ids=case_id)
def test_gemm_twin_sweep(case):
    """The tap-GEMM twin on every sweep case (bias scaled by s_acc, row vectors, residuals in place, GEGLU tile halves,
    erf-GELU, halo rows, fused statistics): a twin that drops a term is off by that term, O(1) against a tolerance of
    one fp16 ulp."""
    check_gemm_case(case, fake_ops.gemm, CPU)


def launcher_variant(d) -> int:
    """The epilogue variant b200v_gemm (gemm_tc.cu) selects for the arguments of one case."""
    kw = d["kw"]
    bf16, f32o = d["a"].dtype == torch.bfloat16, d["out"].dtype == torch.float32
    if kw.get("stats") is not None:
        return 9 + (2 if kw.get("rowvec") is not None else 1 if kw.get("res1") is not None else 0)
    if bf16:
        return 12
    if f32o:
        return 7
    nres = (kw.get("res1") is not None) + (kw.get("res2") is not None)
    act, rv = kw["act"], kw.get("rowvec") is not None
    if act == 0 and not rv:
        return nres
    if act == 0 and nres <= 1:
        return 3 + nres
    if act == 1 and not rv and nres == 0:
        return 5
    return {2: 6, 3: 8}.get(act, 7)


def test_gemm_sweep_reaches_every_instantiation():
    """The table reaches every (tile width, epilogue variant) pair the launcher can select — by the arguments each case
    really passes, not by its label — and the 'many' geometry has a K-chunk count that is not a multiple of the ring
    depth on at least three widths (the stage / phase carry between tiles)."""
    got = set()
    for c in gemm_cases(small=True):
        v = launcher_variant(make_gemm_case(c, CPU))
        assert v == c["variant"], (case_id(c), v)
        got.add((c["tn"], v))
    assert got == expected_instantiations() and len(got) == 100
    carry = {c["tn"] for c in gemm_cases() if c["geom"] == "many" and 9 % nstages(c["tn"])}
    assert len(carry) >= 3, carry


@pytest.mark.parametrize("frames,seq,heads", SPATIAL_CASES)
def test_attention_spatial_twin(frames, seq, heads):
    """Spatial attention twin with separate, differently strided q / k / v: a wrong head split or frame stride mixes
    unrelated rows (O(1) errors)."""
    q, k, v = spatial_inputs(frames, seq, heads, CPU, seed=7)
    out = torch.empty(frames * seq, heads * 64, dtype=torch.float16)
    fake_ops.attention_spatial(q, k, v, out, frames, seq, heads)
    ref, mag = spatial_ref(q, k, v, frames, seq, heads)
    assert_conform(out, ref, mag, ATTN_EPS, "attn", "spatial twin")


@pytest.mark.parametrize("T", TEMPORAL_T)
def test_attention_temporal_twin(T):
    """Temporal attention twin over frames of one pixel: a wrong (clip, frame, pixel) order attends across pixels."""
    nb, S, heads = 2, 6, 2
    C = heads * 64
    qkv = rnd((nb * T * S, 3 * C), 11 + T, CPU)
    out = torch.empty(nb * T * S, C, dtype=torch.float16)
    fake_ops.attention_temporal(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, nb, T, S, heads)
    ref, mag = temporal_ref(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], nb, T, S, heads)
    assert_conform(out, ref, mag, ATTN_EPS, "attn", f"temporal twin T={T}")


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_attention_temporal_sharded_twin(world):
    """The sharded temporal attention twin through the frame table of a gathered, T_pad-padded K|V (NaN padding): each
    simulated rank's output equals its rows of the unsharded attention."""
    from vista_b200.parallel import frame_shards
    nb, T, S, heads = 2, 7, 5, 1
    C = heads * 64
    qkv = rnd((nb * T * S, 3 * C), 21, CPU)
    ref, mag = temporal_ref(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], nb, T, S, heads)
    shards = frame_shards(T, world)
    kv, tab = sharded_kv(qkv[:, C:2 * C], qkv[:, 2 * C:], nb, T, S, C, shards, CPU)
    q4 = qkv[:, :C].reshape(nb, T, S, C)
    for s0, e in shards:
        Tq = e - s0
        q = q4[:, s0:e].reshape(nb * Tq * S, C)
        out = torch.empty(nb * Tq * S, C, dtype=torch.float16)
        fake_ops.attention_temporal_sharded(q, kv[:, :C], kv[:, C:], out, nb, Tq, T, S, heads, tab)
        rows = lambda t: t.reshape(nb, T, S, C)[:, s0:e].reshape(-1, C)
        assert_conform(out, rows(ref), rows(mag), ATTN_EPS, "attn", f"sharded twin W={world} [{s0},{e})")


@pytest.mark.parametrize("tokens,C", LN_CASES)
def test_layernorm_twin(tokens, C):
    """LayerNorm twin with strided x / y and a row-indexed add vector."""
    x = padded(tokens, C, 16, 31, CPU, scale=1.5, offset=8)
    assert x.stride(0) == C + 16
    gamma = rnd((C,), 32, CPU, dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 33, CPU, dtype=torch.float32) * 0.1
    add = rnd((5, C), 34, CPU, dtype=torch.float32)
    y = torch.empty(tokens, C, dtype=torch.float16)
    fake_ops.layernorm(x, y, gamma, beta, 1e-5, addvec=add, av_div=3, av_mod=5)
    ref, mag = layernorm_reference(x, gamma, beta, 1e-5, add, 3, 5)
    assert_conform(y, ref, mag, FAMILY["norm"].c_acc * math.sqrt(C) * U24, "norm", "layernorm twin")


@pytest.mark.parametrize("frames,tpf,C,fps", GN_CASES)
def test_groupnorm_twin(frames, tpf, C, fps):
    """GroupNorm twin, clip-wide statistics, an input with |mean| / std ~ 30."""
    x = (rnd((frames * tpf, C), 41, CPU, dtype=torch.float32) + 30).half()
    gamma = rnd((C,), 42, CPU, dtype=torch.float32) * 0.1 + 1
    beta = rnd((C,), 43, CPU, dtype=torch.float32) * 0.1
    y = torch.empty_like(x)
    fake_ops.groupnorm(x, y, frames, tpf, gamma, beta, 1e-5, True, frames_per_stat=fps)
    ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, 1e-5, True, fps)
    n = fps * tpf * C // 32
    assert_conform(y, ref, mag, FAMILY["norm"].c_acc * math.sqrt(n) * U24, "norm", "groupnorm twin", extra=extra)


@pytest.mark.parametrize("rows,cols", SOFTMAX_CASES)
def test_softmax_twin(rows, cols):
    x = rnd((rows, cols), 51, CPU, dtype=torch.float32)
    x[0] *= 40.0                                            # a row of large logits
    y = torch.empty(rows, cols, dtype=torch.float16)
    fake_ops.softmax_rows(x, y)
    ref, mag = softmax_reference(x)
    assert_conform(y, ref, mag, FAMILY["softmax"].c_acc * math.sqrt(cols) * U24, "softmax", "softmax twin")


@pytest.mark.parametrize("NB,H,W,C", IM2COL_CASES)
def test_im2col_s2_asym_twin(NB, H, W, C):
    """Exact: the twin of the encoder's Downsample gather against pad + unfold, odd and even H and W."""
    x = rnd((NB * H * W, C), 61, CPU)
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    out = torch.empty(NB * Ho * Wo, 9 * C, dtype=torch.float16)
    fake_ops.im2col_s2_asym(x, out, NB, H, W, C)
    assert torch.equal(out, im2col_asym_reference(x, NB, H, W, C))
