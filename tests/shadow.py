"""Shadow conformance checks of every launch a run makes: a context manager that wraps the vista_b200.ops entry points
(as fake_ops.patched_ops() swaps them) and holds the first launch of every distinct launch configuration to an fp64
reference on the inputs that launch really received.

The runtimes call ``ops.<name>(...)`` at call time, so with fused.USE_GRAPH = False every launch of the single-GPU path
passes through the wrappers.  For each call the wrapper forms a configuration key: the op, the shapes, dtypes and row
strides, whatever the launcher derives from them (the GEMM's tile width and token box, the GroupNorm chunk), the
optional operands present and whether the output overlaps an input.  The first ``first_n`` calls of a key are checked:
the reference is computed from the operands before the launch (so in-place residuals and aliased outputs are read as
the kernel read them), the kernel runs and is synchronised, and sampled outputs are compared under the rule of
tests/test_conformance_cpu.py (assert_conform with FAMILY's factors, eps from K or the row length).  Later calls pass
straight through.  Every reference is O(sample): rows, (frame, head) pairs, whole 128-token tiles, and GroupNorm
statistics reduced over the whole frame set in fp64 chunk by chunk.

Sample rows hold every boundary class: the four image borders of the first, a middle and the last frame, the first and
last token, the whole last m-tile of the box the launcher chose, and ``random_rows`` random rows.

Failures are collected (key -> message) so that one run reports every failing configuration; ``assert_ok()`` raises
with all of them.  An entry point that launches a kernel and has neither a checker nor a SHADOW_EXEMPT reason fails
the run when it is called, and so does an entry point exempted only because nothing calls it (UNCALLED)."""
import hashlib
import inspect
import math

import torch
import torch.nn.functional as F

from test_conformance_cpu import (ATTN_EPS, FAMILY, U24, assert_conform, attention_reference, check_stats,
                                  gemm_reference, layernorm_reference, groupnorm_reference, rel_l2, softmax_reference,
                                  ulp)
from test_conformance_small_cpu import (PREP_EPS, UPDATE_EPS, c_noise_reference, check_reward, check_u8_bytes,
                                        conv_eps, conv_reference, d80_reference, prepare_reference,
                                        rollout_advance_reference, timestep_embedding_reference, tmix_reference,
                                        update_reference, u8_path, BLEND_EPS, TMIX_EPS)
from fake_ops import partials_raw_sums
from vista_b200 import lib as _lib
from vista_b200 import ops as _ops

# the real entry points, captured before any test swaps twins in: their signatures name the arguments
_REAL = {n: f for n, f in vars(_ops).items() if inspect.isfunction(f) and f.__module__ == _ops.__name__}

SHADOW_EXEMPT = {
    "frames_u8_resize": "test_ingest_gpu.py holds it bit-exact at 1600 x 900 -> 576 x 1024",
    "peer_put": "peer-memory transport: frame-sharded runs on two or more GPUs only",
    "peer_wait": "peer-memory transport: frame-sharded runs on two or more GPUs only",
    "peer_allreduce_f64": "peer-memory transport: frame-sharded runs on two or more GPUs only",
    "groupnorm_sums": "first half of the frame-sharded GroupNorm: multi-GPU runs only",
    "groupnorm_finalize_apply": "second half of the frame-sharded GroupNorm: multi-GPU runs only",
    "attention_temporal_sharded": "frame-sharded temporal attention: multi-GPU runs only",
    "conv3x3_small_cout": "no caller on the product path",
}
# exempt only because nothing calls them: the harness installs the failing wrapper, so that a new caller is noticed
UNCALLED = {"conv3x3_small_cout"}


def launches_kernel(fn) -> bool:
    """An ops entry point launches a kernel when it hands a C-ABI call to lib.check."""
    return inspect.isfunction(fn) and "_lib.check(" in inspect.getsource(fn)


def overlaps(a, b) -> bool:
    """Whether two tensors share bytes of one storage."""
    if a is None or b is None or a.device != b.device:
        return False
    if a.untyped_storage().data_ptr() != b.untyped_storage().data_ptr():
        return False
    span = lambda t: (t.data_ptr(), t.data_ptr() + ((t.shape[0] - 1) * t.stride(0) + t.shape[-1]) * t.element_size())
    (a0, a1), (b0, b1) = span(a), span(b)
    return a0 < b1 and b0 < a1


def _ld(t):
    return None if t is None else (t.stride(0) if t.dim() >= 1 else 0)


def _dt(t):
    return None if t is None else str(t.dtype).replace("torch.", "")


def _sync(t):
    if t is not None and t.is_cuda:
        torch.cuda.synchronize()


class Entry:
    def __init__(self, op):
        self.op, self.calls, self.checked, self.ratio, self.rel_floor, self.family = op, 0, 0, 0.0, 0.0, None


class Check:
    """One checked launch: compares and records the worst error / bound and rel-L2 / floor of the key."""

    def __init__(self, shadow, key, entry):
        self.shadow, self.key, self.entry = shadow, key, entry
        self.gen = torch.Generator().manual_seed(int(hashlib.sha1(repr(key).encode()).hexdigest()[:8], 16))

    @property
    def name(self):
        return f"{self.key[0]} {self.key[1:]}"

    def rand(self, n, hi):
        return torch.randint(0, max(hi, 1), (n,), generator=self.gen)

    def _note(self, family, ratio, rel_floor=0.0):
        e = self.entry
        e.family = e.family or family
        e.ratio = max(e.ratio, ratio)
        e.rel_floor = max(e.rel_floor, rel_floor)

    def conform(self, out, ref, mag, eps, family, what="", extra=None, factor=None):
        o = out.double()
        tol = ulp(ref, out.dtype) + eps * mag + (0 if extra is None else extra)
        ratio = float(((o - ref).abs() / tol.clamp_min(1e-300)).max()) if o.numel() else 0.0
        r16 = torch.bfloat16 if out.dtype == torch.bfloat16 else torch.float16
        floor = rel_l2(ref.to(r16), ref)
        self._note(family, ratio, rel_l2(o, ref) / floor if floor > 0 else 0.0)
        assert_conform(out, ref, mag, eps, family, f"{self.name}{what}", factor=factor, extra=extra)

    def elements(self, out, ref, tol, family, what=""):
        err = (out.double() - ref).abs()
        ratio = float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0
        self._note(family, ratio)
        bad = ~(err <= tol)
        if bool(bad.any()):
            i = int(torch.argmax(torch.where(bad, err - tol, torch.zeros_like(err))))
            raise AssertionError(f"{self.name}{what}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; worst "
                                 f"flat index {i}: out {float(out.flatten()[i]):.9g} ref {float(ref.flatten()[i]):.9g} "
                                 f"tol {float(tol.flatten()[i]):.3g}")

    def exact(self, ok, what=""):
        self._note("exact", 0.0 if ok else math.inf)
        assert ok, f"{self.name}{what}: not bit-equal to its torch restatement"


# ==================================================================================================================
# Sample rows
# ==================================================================================================================
def tile_tokens(a_mode, geom, box, m_blk, tokens):
    """The output tokens of m-tile ``m_blk`` in the kernel's row order (gemm_tc.cuh's epilogue), valid ones only."""
    r = torch.arange(128)
    if a_mode == 0:
        t = m_blk * 128 + r
        return t[t < tokens]
    W, H, NB = geom
    bw, bh, bb = box
    tw_n, th_n = -(-W // bw), -(-H // bh)
    bx = m_blk >> 2 if a_mode == 2 else m_blk
    tw, th, tb = bx % tw_n, (bx // tw_n) % th_n, bx // (tw_n * th_n)
    w, h, b = tw * bw + r % bw, th * bh + (r // bw) % bh, tb * bb + r // (bw * bh)
    ok = (w < W) & (h < H) & (b < NB)
    if a_mode == 2:
        t = (2 * (b * H + h) + ((m_blk >> 1) & 1)) * 2 * W + 2 * w + (m_blk & 1)
    else:
        t = (b * H + h) * W + w
    return t[ok]


def n_tiles(a_mode, geom, box, tokens):
    if a_mode == 0:
        return -(-tokens // 128)
    W, H, NB = geom
    n = -(-W // box[0]) * -(-H // box[1]) * -(-NB // box[2])
    return 4 * n if a_mode == 2 else n


def border_rows(W, H, NB):
    """Tokens of the four borders of the first, a middle and the last frame of a W x H x NB geometry."""
    out = []
    for b in sorted({0, NB // 2, NB - 1}):
        base = b * H * W
        w, h = torch.arange(W), torch.arange(H)
        out += [base + w, base + (H - 1) * W + w, base + h * W, base + h * W + W - 1]
    return torch.cat(out)


def sample_rows(chk, tokens, n_random, geom=None, extra=()):
    parts = [torch.tensor([0, tokens - 1]), chk.rand(n_random, tokens)] + [torch.as_tensor(e) for e in extra]
    if geom is not None:
        parts.append(border_rows(*geom))
    return torch.unique(torch.cat(parts).long())


# ==================================================================================================================
# Checkers: each gets the bound arguments, computes its reference before the launch, and returns the comparison
# ==================================================================================================================
def _gemm(chk, A, n):
    a, w, out = A["a"], A["w"], A["out"]
    taps, geom, up, h_pad, act = list(A["taps"]), A["geom"], A.get("upsample", False), A["h_pad"], A["act"]
    N, K = w.shape
    tokens = geom[0] * geom[1] * geom[2] if geom is not None else a.shape[0]
    out_tokens = 4 * tokens if up else tokens
    tile_n = A["tile_n"] if A["tile_n"] is not None else _ops.pick_tile_n(N, act == 2)
    a_mode, box = gemm_box(A)
    n_out = N // 2 if act == 2 else N
    last = tile_tokens(a_mode, geom, box, n_tiles(a_mode, geom, box, tokens) - 1, tokens)
    out_geom = None if geom is None else ((2 * geom[0], 2 * geom[1], geom[2]) if up else geom)
    rows = sample_rows(chk, out_tokens, n, out_geom, [last])
    stats = A["stats"]
    tiles = []
    if stats is not None:                     # whole 128-token tiles: the first, the last and a few random ones
        nt = n_tiles(a_mode, geom, box, tokens)
        tiles = sorted({0, nt - 1} | set(chk.rand(max(2, n // 256), nt).tolist()))
        tile_rows = [tile_tokens(a_mode, geom, box, m, tokens) for m in tiles]
        rows = torch.unique(torch.cat([rows] + tile_rows))
    dev_rows = rows.to(a.device)
    kw = dict(taps=taps, geom=geom, h_pad=h_pad, bias=A["bias"], rowvec=A["rowvec"], rv_div=A["rv_div"],
              rv_mod=A["rv_mod"], s_acc=A["s_acc"], act=act, tile_n=tile_n, rows=dev_rows, upsample=up)
    ref, mag = gemm_reference(a, w, **kw)
    for r, s in ((A["res1"], A["s_res1"]), (A["res2"], A["s_res2"])):   # residuals as the kernel reads them: now
        if r is not None:
            v = s * r[dev_rows, :n_out].double()
            ref, mag = ref + v, mag + v.abs()
    eps = FAMILY["gemm"].c_acc * math.sqrt(K) * U24

    def compare():
        chk.conform(out[dev_rows, :n_out], ref, mag, eps, "gemm")
        if stats is not None:
            pos = {int(t): i for i, t in enumerate(rows.tolist())}
            for m, tr in zip(tiles, tile_rows):
                idx = torch.tensor([pos[int(t)] for t in tr.tolist()], device=a.device)
                check_stats(stats[4 * m:4 * m + 4, :n_out], out[dev_rows[idx], :n_out], f"{chk.name} stats tile {m}")
    return compare


def gemm_box(A):
    """(a_mode, token box) exactly as ops.gemm derives them."""
    geom = A["geom"]
    if geom is None:
        return 0, None
    if A.get("upsample", False):
        return 2, (_ops.upsample_stats_box(geom[0], geom[1]) if A["stats"] is not None else _ops.pick_box(*geom))
    return 1, (_ops.pick_box(*geom) if A["stats"] is None else _ops.stats_box(*geom))


# the fields of a gemm key after the op name (gemm_field reads one by name)
GEMM_KEY_FIELDS = ("a_dtype", "out_dtype", "rows", "lda", "ldo", "N", "K", "taps", "geom", "h_pad", "a_mode", "box",
                   "tile_n", "act")


def gemm_field(key, name):
    """Field ``name`` of a gemm key, with or without the leading op name."""
    return key[GEMM_KEY_FIELDS.index(name) + (key[0] == "gemm")]


def _gemm_key(A):
    a, w, out = A["a"], A["w"], A["out"]
    a_mode, box = gemm_box(A)
    N, K = w.shape
    act = A["act"]
    tile_n = A["tile_n"] if A["tile_n"] is not None else _ops.pick_tile_n(N, act == 2)
    flags = tuple(k for k in ("bias", "rowvec", "res1", "res2", "stats") if A[k] is not None)
    if A["s_acc"] != 1.0:
        flags += ("s_acc",)
    if any(overlaps(out, A[k]) for k in ("a", "res1", "res2")):
        flags += ("inplace",)
    # the tap offsets decide which border rows read zero padding: (-1, 0) / (1, 0) and (0, -1) / (0, 1) are different
    # boundary behaviours at equal tap counts
    taps = tuple(tuple(t) for t in A["taps"])
    return (_dt(a), _dt(out), a.shape[0], _ld(a), _ld(out), N, K, taps, A["geom"], A["h_pad"], a_mode, box, tile_n,
            act) + flags


def moments64(x, frames, tpf, C, fps, groups, chunk_rows=1 << 16):
    """fp64 (mean, var, E|x|, E x^2) [frames / fps, groups] of x [frames tpf, >= C], reduced chunk by chunk."""
    n_stat, per = frames // fps, fps * tpf
    cpg = C // groups
    acc = torch.zeros(4, n_stat, groups, dtype=torch.float64, device=x.device)
    for s in range(n_stat):
        for r0 in range(0, per, chunk_rows):
            v = x[s * per + r0: s * per + min(per, r0 + chunk_rows), :C].double().reshape(-1, groups, cpg)
            acc[0, s] += v.sum((0, 2))
            acc[1, s] += (v * v).sum((0, 2))
            acc[2, s] += v.abs().sum((0, 2))
    n = float(per * cpg)
    mean, ex2, eabs = acc[0] / n, acc[1] / n, acc[2] / n
    var = (ex2 - mean * mean).clamp_min(0.0)
    return mean, var, eabs, ex2


def gn_stats_accumulation(frames, tpf, C):
    """Relative error of gn_stats_kernel's fp32 sums, derived from its launch: a block walks one chunk of the frame
    (b200v_groupnorm_chunk_for), its 256 threads form rows = 256 / L token rows (L threads cover the C / 8 channel
    vectors, in J passes when C / 8 > 256), and each thread adds ceil(chunk / rows) tokens into fp32 sums (one more
    rounding for the square of x^2); rows, chunks and groups are then added in fp64.  Each fp32 addition rounds by at
    most U24 of the running sum; independent roundings grow as the square root of their number, and the norm family's
    c_acc is the margin over that random walk (FAMILY['norm'], the rule eps = c_acc sqrt(n) U24 of the norm tests)."""
    nvec = C // 8
    L, J = nvec, 1
    while L > 256:
        J += 1
        L = -(-nvec // J)
    rows = 256 // L
    chunk = _lib.load().b200v_groupnorm_chunk_for(frames, tpf)
    n_add = -(-min(chunk, tpf) // rows) + 1
    return FAMILY["norm"].c_acc * math.sqrt(n_add) * U24


# GEMM-fused partials (check_stats): fp32 sums of deviations over the 32 rows of one tile quarter, then fp64
PARTIALS_ACCUMULATION = FAMILY["norm"].c_acc * math.sqrt(32) * U24


def check_mean_rstd(chk, got, mean, var, eps, acc, what):
    """(mean, rstd) written by a kernel against the fp64 statistics of the tensor it normalises.  The bound is the
    operation's: fp32 sums of n_add terms (``acc`` = c sqrt(n_add) U24: gn_stats_accumulation, PARTIALS_ACCUMULATION)
    off relative to the spread, |d mean| <= ulp32(mean) + acc std, and rstd within acc + 4 U24 (the fp32 store and
    rsqrt) relative.  No term grows with |mean| / std, so statistics that cancel E x^2 - mean^2 in fp32 fail it."""
    tol_m = ulp(mean, torch.float32) + acc * var.sqrt()
    rstd = torch.rsqrt(var + eps)
    tol_r = rstd * (acc + 4 * U24)
    chk.elements(got[..., 0], mean, tol_m, "norm", f"{what} mean")
    chk.elements(got[..., 1], rstd, tol_r, "norm", f"{what} rstd")


def _gn_rows(chk, frames, tpf, n, fps):
    last = torch.arange(max(0, frames * tpf - 128), frames * tpf)
    firsts = torch.arange(0, frames * tpf, tpf)
    return sample_rows(chk, frames * tpf, n, None, [last, firsts, firsts + tpf - 1])


def _groupnorm(chk, A, n):
    x, y, frames, tpf = A["x"], A["y"], A["frames"], A["tokens_per_frame"]
    gamma, beta, eps, silu, fps, groups = A["gamma"], A["beta"], A["eps"], A["silu"], A["frames_per_stat"], A["groups"]
    C = gamma.numel()
    mean, var, eabs, ex2 = moments64(x, frames, tpf, C, fps, groups)
    rows = _gn_rows(chk, frames, tpf, n, fps).to(x.device)
    ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, eps, silu, fps, groups, rows=rows,
                                          moments=(mean, torch.rsqrt(var + eps)))
    stats = A["stats"]
    eps_n = FAMILY["norm"].c_acc * math.sqrt(fps * tpf * C // groups) * U24

    def compare():
        chk.conform(y[rows, :C], ref, mag, eps_n, "norm", extra=extra)
        if stats is not None:
            check_mean_rstd(chk, stats.double(), mean, var, eps, gn_stats_accumulation(frames, tpf, C), " stats")
    return compare


def _gn_key(A):
    return (A["frames"], A["tokens_per_frame"], A["gamma"].numel(), A["groups"], A["frames_per_stat"], bool(A["silu"]),
            _ld(A["x"]), _ld(A["y"]), overlaps(A["x"], A["y"]), A.get("stats") is not None,
            _lib.load().b200v_groupnorm_chunk_for(A["frames"], A["tokens_per_frame"]))


def _gn_from_partials(chk, A, n):
    """(mean, rstd) against the fp64 reduction of the partials it reads (the GroupNorm apply that follows holds them
    against the fp64 statistics of the stored tensor)."""
    p, frames, tpf, Cc, eps, stats = A["partials"], A["frames"], A["tokens_per_frame"], A["Cc"], A["eps"], A["stats"]
    fps, groups, raw = A["frames_per_stat"], A["groups"], A["raw_sums"]
    n_stat, rows = frames // fps, fps * (tpf // 128) * 4
    s = partials_raw_sums(p[: n_stat * rows, :Cc]).reshape(n_stat, rows, groups, Cc // groups, 2).sum(dim=(1, 3))
    count = float(Cc // groups) * tpf * fps
    mean = s[..., 0] / count
    var = (s[..., 1] / count - mean * mean).clamp_min(0.0)

    def compare():
        if raw is not None:
            chk.elements(raw.reshape(s.shape).double(), s, 1e-12 * s.abs() + 1e-300, "norm", " raw sums")
            return
        got = stats.double()
        chk.elements(got[..., 0], mean, ulp(mean, torch.float32) + 1e-12 * mean.abs(), "norm", " mean")
        r = torch.rsqrt(var + eps)
        # var from fp64 sums: relative error ~2^-52 E x^2 / var, then rsqrtf (2 ulp) and the store
        tol = r * (4 * U24 + 2.0 ** -50 * (s[..., 1] / count) / (var + eps))
        chk.elements(got[..., 1], r, tol, "norm", " rstd")
    return compare


def _gn_apply(chk, A, n):
    x, y, frames, tpf = A["x"], A["y"], A["frames"], A["tokens_per_frame"]
    gamma, beta, silu, stats, fps, groups = A["gamma"], A["beta"], A["silu"], A["stats"], A["frames_per_stat"], A["groups"]
    C = gamma.numel()
    mean, var, _, _ = moments64(x, frames, tpf, C, fps, groups)
    got = stats.double().clone()
    rows = _gn_rows(chk, frames, tpf, n, fps).to(x.device)
    eps_n = FAMILY["norm"].c_acc * math.sqrt(fps * tpf * C // groups) * U24
    # the eps the statistics were taken with: that of the groupnorm_from_partials call that wrote them
    eps_gn = chk.shadow.stats_eps.get(stats.data_ptr())
    assert eps_gn is not None, f"{chk.name}: statistics not written by groupnorm_from_partials"
    # the output against GroupNorm of the stored tensor with its own fp64 statistics, not the kernel's
    ref, mag, extra = groupnorm_reference(x, frames, tpf, gamma, beta, eps_gn, silu, fps, groups, rows=rows,
                                          moments=(mean, torch.rsqrt(var + eps_gn)))

    def compare():
        # the statistics describe the stored values the producing GEMM(s) summed
        check_mean_rstd(chk, got, mean, var, eps_gn, PARTIALS_ACCUMULATION, " statistics")
        chk.conform(y[rows, :C], ref, mag, eps_n, "norm", extra=extra)
    return compare


def _layernorm(chk, A, n):
    x, y, gamma, beta, eps = A["x"], A["y"], A["gamma"], A["beta"], A["eps"]
    C = gamma.numel()
    rows = sample_rows(chk, x.shape[0], n).to(x.device)
    ref, mag = layernorm_reference(x, gamma, beta, eps, A["addvec"], A["av_div"], A["av_mod"], rows=rows)
    return lambda: chk.conform(y[rows, :C], ref, mag, FAMILY["norm"].c_acc * math.sqrt(C) * U24, "norm")


def _attn_spatial(chk, A, n):
    q, k, v, out, frames, seq, heads = (A[s] for s in ("q", "k", "v", "out", "frames", "seq", "heads"))
    pairs = sorted({(0, 0), (frames - 1, heads - 1)} | set(zip(chk.rand(2, frames).tolist(), chk.rand(2, heads).tolist())))
    qrows = sample_rows(chk, seq, max(64, n // len(pairs)), None, [torch.arange(max(0, seq - 128), seq)]).to(q.device)
    refs = []
    for f, hd in pairs:
        sl = lambda t, r=None: t[f * seq + (torch.arange(seq, device=q.device) if r is None else r), hd * 64:(hd + 1) * 64]
        o, m = attention_reference(sl(q, qrows), sl(k), sl(v), p_normalised=False)
        refs.append((f * seq + qrows, hd, o, m))

    def compare():
        for i, (r, hd, o, m) in enumerate(refs):
            chk.conform(out[r, hd * 64:(hd + 1) * 64], o, m, ATTN_EPS, "attn", f" (frame, head) {pairs[i]}")
    return compare


def _attn_temporal(chk, A, n):
    q, k, v, out, nb, T, S, heads = (A[s] for s in ("q", "k", "v", "out", "nb", "T", "S", "heads"))
    pix = sample_rows(chk, nb * S, max(16, n // T), None, [torch.arange(max(0, nb * S - 64), nb * S), torch.tensor([S - 1])])
    b, s = pix // S, pix % S
    idx = ((b[:, None] * T + torch.arange(T)[None]) * S + s[:, None]).to(q.device)          # [P, T] token rows
    g = lambda t: t[idx.reshape(-1), :heads * 64].double().reshape(len(pix), T, heads, 64).permute(0, 2, 1, 3)
    o, m = attention_reference(g(q), g(k), g(v), p_normalised=True)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(-1, heads * 64)
    return lambda: chk.conform(out[idx.reshape(-1), :heads * 64], back(o), back(m), ATTN_EPS, "attn")


def _attn_d80(chk, A, n):
    q, k, v, out, batch, seq, heads = (A[s] for s in ("q", "k", "v", "out", "batch", "seq", "heads"))
    imgs = sorted({0, batch - 1} | set(chk.rand(1, batch).tolist()))
    refs = []
    for i in imgs:
        r = slice(i * seq, (i + 1) * seq)
        refs.append((r,) + d80_reference(q[r], k[r], v[r], 1, seq, heads))

    def compare():
        for i, (r, o, m) in zip(imgs, refs):
            chk.conform(out[r, :heads * 80], o, m, ATTN_EPS, "attn", f" image {i}")
    return compare


def _softmax(chk, A, n):
    x, y = A["x"], A["y"]
    rows = sample_rows(chk, x.shape[0], min(n, 1024)).to(x.device)
    ref, mag = softmax_reference(x[rows])
    cols = x.shape[1]
    return lambda: chk.conform(y[rows, :cols], ref, mag, FAMILY["softmax"].c_acc * math.sqrt(cols) * U24, "softmax")


def _conv_small_cin(chk, A, n):
    x8, cin, w, bias, out, NB, H, W = (A[s] for s in ("x8", "cin", "w", "bias", "out", "NB", "H", "W"))
    rows = sample_rows(chk, NB * H * W, n, (W, H, NB)).to(x8.device)
    ref, mag = conv_reference(x8, w, bias, NB, H, W, rows=rows)
    return lambda: chk.conform(out[rows, :w.shape[0]], ref, mag, conv_eps(cin), "gemm")


def _taps_gather(x, rows, NB, H, W, Cc, Ho, Wo, off):
    """Rows of a 3x3 stride-2 gather: out row (b, oy, ox), tap (kh, kw) reads x[b, 2 oy + kh - off, 2 ox + kw - off],
    zero outside the frame."""
    ox, oy, b = rows % Wo, (rows // Wo) % Ho, rows // (Wo * Ho)
    parts = []
    for kh in range(3):
        for kw in range(3):
            hs, ws = 2 * oy + kh - off, 2 * ox + kw - off
            ok = (hs >= 0) & (hs < H) & (ws >= 0) & (ws < W)
            src = torch.where(ok, (b * H + hs) * W + ws, torch.zeros_like(rows))
            parts.append(torch.where(ok[:, None], x[src, :Cc], torch.zeros_like(x[src, :Cc])))
    return torch.cat(parts, 1)


def _im2col(off):
    def checker(chk, A, n):
        x, out, NB, H, W, Cc = (A[s] for s in ("x", "out", "NB", "H", "W", "Cc"))
        Ho, Wo = ((H - 1) // 2 + 1, (W - 1) // 2 + 1) if off else ((H - 2) // 2 + 1, (W - 2) // 2 + 1)
        rows = sample_rows(chk, NB * Ho * Wo, n, (Wo, Ho, NB)).to(x.device)
        want = _taps_gather(x, rows, NB, H, W, Cc, Ho, Wo, off)
        return lambda: chk.exact(torch.equal(out[rows, :9 * Cc], want))
    return checker


def _upsample2x(chk, A, n):
    x, out, NB, H, W, Cc = (A[s] for s in ("x", "out", "NB", "H", "W", "Cc"))
    rows = sample_rows(chk, NB * 4 * H * W, n, (2 * W, 2 * H, NB)).to(x.device)
    xx, yy, b = rows % (2 * W), (rows // (2 * W)) % (2 * H), rows // (4 * H * W)
    want = x[(b * H + yy // 2) * W + xx // 2, :Cc].clone()
    return lambda: chk.exact(torch.equal(out[rows, :Cc], want))


def _nchw_to_tokens(chk, A, n):
    x, out, NB, Cc, H, W = (A[s] for s in ("x", "out", "NB", "Cc", "H", "W"))
    rows = sample_rows(chk, NB * H * W, n, (W, H, NB)).to(x.device)
    want = x.reshape(NB, Cc, H * W).permute(0, 2, 1).reshape(-1, Cc)[rows].to(out.dtype)
    return lambda: chk.exact(torch.equal(out[rows, :Cc], want))


def _tokens_to_nchw(chk, A, n):
    x, out, NB, Cc, H, W = (A[s] for s in ("x", "out", "NB", "Cc", "H", "W"))
    rows = sample_rows(chk, NB * H * W, n, (W, H, NB)).to(x.device)
    want = x[rows, :Cc].float()
    return lambda: chk.exact(torch.equal(out.reshape(NB, Cc, H * W).permute(0, 2, 1).reshape(-1, Cc)[rows], want))


def _time_mix(u8):
    def checker(chk, A, n):
        x, w, bias, out, blend, T, HW, Cc = (A[s] for s in ("x", "w", "bias", "out", "blend", "T", "HW", "Cc"))
        f0, skip = A["out_frame0"], A["skip_frames"]
        keep = A["keep_f32_from"] if u8 else -1
        pix = sample_rows(chk, HW, max(64, n // T), None, [torch.arange(max(0, HW - 256), HW)]).to(x.device)
        P, F_ = len(pix), out.shape[0]
        xs = x[(torch.arange(T, device=x.device)[:, None] * HW + pix[None]).reshape(-1)]
        prev = out.reshape(F_, Cc, HW)[:, :, pix].clone()
        ref, mag, extra = tmix_reference(xs, w, bias, T, P, prev, f0, blend, skip)
        lo, hi = f0 + skip, f0 + T
        k0 = lo if keep < 0 else max(lo, f0 + keep)

        def compare():
            got = out.reshape(F_, Cc, HW)[:, :, pix]
            if k0 < hi:
                chk.conform(got[k0:hi], ref[k0 - lo:], mag[k0 - lo:], TMIX_EPS, "elementwise", " fp32 frames",
                            extra=extra[k0 - lo:])
            if u8:
                b = A["out_u8"].reshape(-1, HW, Cc)[lo:hi, pix].permute(0, 2, 1)
                tol = ulp(ref, torch.float32) + TMIX_EPS * mag + extra
                check_u8_bytes(b, ref, tol, f"{chk.name} bytes")
                chk.exact(torch.equal(b[k0 - lo:], u8_path(got[k0:hi])), " bytes vs the output path of the fp32 frames")
        return compare
    return checker


def _tmix_key(A):
    return (A["T"], A["HW"], A["Cc"], _ld(A["x"]), tuple(A["out"].shape), A["out_frame0"], A["skip_frames"],
            A["blend"] is not None and int(A["blend"].sum()), A.get("keep_f32_from", -1), A["bias"] is not None)


def _sampler_d(A, net_key="net_out"):
    d = dict(T=A["T"], h=A["h"], w=A["w"], x=A["x"].clone(), mask=A["mask"], cond_frame=A["cond_frame"],
             sigmas=A["sigmas"], scales=A.get("scales"))
    if net_key in A:
        d["net"] = A[net_key]
    return d


def _prepare(chk, A, n):
    d = _sampler_d(A)
    d["concat_u"], d["concat_c"] = A["concat_u"], A["concat_c"]
    step = int(A["step_idx"][0])
    sigma = A["sigmas"][step]
    x_ref, in_ref, cat_ref = prepare_reference(d, sigma)
    rows = 2 * A["T"] * A["h"] * A["w"]
    cn = A["c_noise"]

    def compare():
        chk.exact(torch.equal(A["x"], x_ref), " masked x")
        un = A["unet_in"][:rows]
        chk.conform(un[:, :4], in_ref, in_ref.abs(), PREP_EPS, "elementwise", " unet_in")
        chk.exact(torch.equal(un[:, 4:8], cat_ref), " concat columns")
        if cn is not None:
            ref, tol = c_noise_reference(sigma, cn.numel(), cn.device)
            chk.elements(cn, ref, tol, "elementwise", " c_noise")
    return compare


def _update(kind):
    def checker(chk, A, n):
        from test_dpmpp2m_cpu import update_2m_reference
        from test_action_cfg_cpu import update_action_reference
        d = _sampler_d(A)
        x0, step, num_steps = d["x"], int(A["step_idx"][0]), A["num_steps"]
        dp = A.get("d_prev")
        dp0 = None if dp is None else dp.clone()
        if kind == "euler":
            xn, mag, _ = update_reference(x0, d, step, num_steps)
            bound, den, den_bound = UPDATE_EPS * mag, None, None
        elif kind == "2m":
            xn, den, bound, den_bound = update_2m_reference(x0, d, step, A["coefs"], dp0, num_steps)
        else:
            d["net_img"], d["action_scales"] = A["net_img"], A["action_scales"]
            xn, den, bound, den_bound = update_action_reference(x0, d, step, num_steps, A["coefs"], dp0)

        def compare():
            x = A["x"]
            chk.exact(int(A["step_idx"][0]) == step + 1, " step_idx")
            chk.elements(x, xn, bound + U24 * xn.abs(), "elementwise", f" x (step {step})")
            if den is not None and dp is not None:
                chk.elements(dp, den, den_bound + U24 * den.abs(), "elementwise", " D_prev")
        return compare
    return checker


def _update_key(A):
    coefs = A.get("coefs")
    order = None if coefs is None else float(coefs[int(A["step_idx"][0]), 3]) != 0.0
    return (A["T"], A["h"], A["w"], _ld(A["net_out"]), A["mask"] is not None, A.get("net_img") is not None, order,
            int(A["step_idx"][0]) + 1 == A["num_steps"])


def _rollout_advance(chk, A, n):
    sample, z0, sz, filled = A["sample"], A["z0"], A["samples_z"], A["filled"]
    want = rollout_advance_reference(sample, z0, sz, filled, A["dst_frame0"], A["src_frame0"], A["n_cond"])

    def compare():
        s_ref, sz_ref, f_ref = want
        chk.exact(torch.equal(sample, s_ref) and torch.equal(sz, sz_ref) and (filled is None or torch.equal(filled, f_ref)))
    return compare


class _Reward:
    """ensemble_reward returns its output: the check runs on it after the launch."""


def _timestep_embedding(chk, A, n):
    t, out, dim = A["t"], A["out"], A["dim"]
    ref, mag = timestep_embedding_reference(t, dim, A["max_period"])
    return lambda: chk.conform(out[:t.numel(), :dim], ref, mag, U24, "elementwise")


def _blend_emb(chk, A, n):
    e_plain, e_cond, label, mask, emb, semb = (A[s] for s in ("e_plain", "e_cond", "label", "mask", "emb", "silu_emb"))
    rows = e_plain.shape[0]
    m = torch.zeros(rows, 1, dtype=torch.float64, device=e_plain.device) if mask is None else mask.double().reshape(-1, 1)
    ref, mag = e_plain.double() * (1 - m), e_plain.double().abs() * (1 - m).abs()
    if e_cond is not None:
        ref, mag = ref + e_cond.double() * m, mag + e_cond.double().abs() * m.abs()
    if label is not None:
        ref, mag = ref + label.double(), mag + label.double().abs()

    def compare():
        if emb is not None:
            chk.conform(emb, ref, mag, BLEND_EPS, "elementwise", " emb")
        if semb is not None:      # the silu bound of test_conformance_small_cpu.check_blend_emb
            s = F.silu(ref)
            chk.conform(semb, s, 1.1 * BLEND_EPS / U24 * mag + (ref.abs() + 8) * s.abs(), U24, "elementwise", " silu_emb")
    return compare


def _sinusoid(chk, A, n):
    values, slots, freqs, out = A["values"], A["slots"], A["freqs"], A["out"]
    rows = out.shape[0]
    parts = []
    for vc, nf, od, dc, zero, fo in slots:
        half = od // 2
        if zero:
            ref = torch.zeros(rows, nf * od, dtype=torch.float64, device=out.device)
        else:          # the fp32 product of value and host frequency, as the kernel forms it; cos / sin in fp64
            a = (values[:, vc:vc + nf].reshape(rows * nf, 1) * freqs[fo:fo + half].reshape(1, half)).double()
            e = [torch.cos(a), torch.sin(a)] + ([torch.zeros_like(a[:, :1])] if od % 2 else [])
            ref = torch.cat(e, 1).reshape(rows, nf * od)
        parts.append((dc, nf * od, ref))

    def compare():
        for dc, width, ref in parts:      # the bound of test_conditioner_gpu.test_sinusoid_embed_matches_formula
            chk.elements(out[:, dc:dc + width], ref, torch.full_like(ref, 1e-6), "elementwise", f" slot at column {dc}")
    return compare


def _clip_preprocess(chk, A, n):
    from oracle import clip_oracle
    x, out = A["x"], A["out"]
    want = clip_oracle.preprocess(x.float().cpu(), A["antialias"]).double()
    nimg = x.shape[0]

    def compare():
        r = out.double().cpu().reshape(nimg, 257, -1)
        chk.exact(bool((r[:, 0] == 0).all()) and bool((r[:, :, 588:] == 0).all()), " class-token row and pad columns")
        got = r[:, 1:, :588].reshape(nimg, 16, 16, 3, 14, 14).permute(0, 3, 1, 4, 2, 5).reshape(nimg, 3, 224, 224)
        # the bound of test_clip_gpu.test_preprocess_matches_oracle, plus the fp16 store when the rows are fp16
        chk.elements(got, want, 1e-5 + ulp(want, out.dtype), "elementwise")
    return compare


CHECKERS = {
    # op: (checker(chk, bound arguments, n_random) -> compare(), key(bound arguments) -> tuple)
    "gemm": (_gemm, _gemm_key),
    "groupnorm": (_groupnorm, _gn_key),
    "groupnorm_from_partials": (_gn_from_partials, lambda A: (A["frames"], A["tokens_per_frame"], A["Cc"],
                                                              A["frames_per_stat"], A["groups"], _ld(A["partials"]),
                                                              A["raw_sums"] is not None)),
    "groupnorm_apply": (_gn_apply, lambda A: _gn_key(dict(A, eps=None, stats=None)) + ("apply",)),
    "layernorm": (_layernorm, lambda A: (A["x"].shape[0], A["gamma"].numel(), _ld(A["x"]), _ld(A["y"]),
                                         A["addvec"] is not None, A["av_div"], A["av_mod"], overlaps(A["x"], A["y"]))),
    "attention_spatial": (_attn_spatial, lambda A: (A["frames"], A["seq"], A["heads"], _ld(A["q"]), _ld(A["k"]),
                                                    _ld(A["v"]), _ld(A["out"]), A["impl"])),
    "attention_temporal": (_attn_temporal, lambda A: (A["nb"], A["T"], A["S"], A["heads"], _ld(A["q"]), _ld(A["out"]))),
    "attention_d80": (_attn_d80, lambda A: (A["batch"], A["seq"], A["heads"], _ld(A["q"]), _ld(A["out"]))),
    "softmax_rows": (_softmax, lambda A: (tuple(A["x"].shape), _ld(A["x"]), _ld(A["y"]))),
    "conv3x3_small_cin": (_conv_small_cin, lambda A: (A["cin"], tuple(A["w"].shape), A["bias"] is not None, _ld(A["out"]),
                                                      A["NB"], A["H"], A["W"])),
    "im2col_s2": (_im2col(1), lambda A: (A["NB"], A["H"], A["W"], A["Cc"], _ld(A["x"]))),
    "im2col_s2_asym": (_im2col(0), lambda A: (A["NB"], A["H"], A["W"], A["Cc"], _ld(A["x"]))),
    "upsample2x": (_upsample2x, lambda A: (A["NB"], A["H"], A["W"], A["Cc"], _ld(A["x"]), _ld(A["out"]))),
    "nchw_to_tokens": (_nchw_to_tokens, lambda A: (A["NB"], A["Cc"], A["H"], A["W"], _ld(A["out"]))),
    "tokens_to_nchw": (_tokens_to_nchw, lambda A: (A["NB"], A["Cc"], A["H"], A["W"], _ld(A["x"]), _dt(A["x"]))),
    "time_mix_small": (_time_mix(False), _tmix_key),
    "time_mix_small_u8": (_time_mix(True), _tmix_key),
    "sampler_prepare": (_prepare, lambda A: (A["T"], A["h"], A["w"], _ld(A["unet_in"]), A["mask"] is not None,
                                             A["concat_u"] is not None, A["concat_c"] is not None,
                                             A["c_noise"] is not None)),
    "sampler_update": (_update("euler"), _update_key),
    "sampler_update_2m": (_update("2m"), _update_key),
    "sampler_update_action": (_update("action"), _update_key),
    "rollout_advance": (_rollout_advance, lambda A: (tuple(A["sample"].shape), A["z0"] is not None,
                                                     A["filled"] is not None, A["src_frame0"], A["n_cond"])),
    "ensemble_reward": (_Reward, lambda A: (len(A["members"]), A["members"][0].numel())),
    "timestep_embedding": (_timestep_embedding, lambda A: (A["t"].numel(), A["dim"], _ld(A["out"]))),
    "blend_emb": (_blend_emb, lambda A: (tuple(A["e_plain"].shape),) + tuple(A[s] is not None for s in
                                                                             ("e_cond", "label", "mask", "emb", "silu_emb"))),
    "sinusoid_embed": (_sinusoid, lambda A: (A["out"].shape[0], _ld(A["out"]), A["values"] is not None,
                                             tuple(tuple(s) for s in A["slots"]))),
    "clip_preprocess": (_clip_preprocess, lambda A: (tuple(A["x"].shape), _dt(A["out"]), _ld(A["out"]),
                                                     bool(A["antialias"]))),
}


def kernel_entry_points():
    """Every public entry point of vista_b200.ops that launches a kernel."""
    return {n for n, f in _REAL.items() if not n.startswith("_") and launches_kernel(f)}


class Shadow:
    """``with Shadow() as sh: ...`` checks every new launch configuration of the block; ``sh.census`` maps key ->
    Entry(calls, checked, worst error / bound, worst rel-L2 / floor); ``sh.assert_ok()`` raises with every failure."""

    def __init__(self, first_n: int = 1, random_rows: int = 2048, ops_module=None):
        self.first_n, self.random_rows = first_n, random_rows
        self.ops = ops_module or _ops
        self.census, self.failures, self._saved = {}, {}, {}
        self.stats_eps = {}       # (mean, rstd) buffer -> eps of the groupnorm_from_partials call that wrote it

    def __enter__(self):
        for name in sorted(kernel_entry_points()):
            if name in SHADOW_EXEMPT and name not in UNCALLED:
                continue
            self._saved[name] = getattr(self.ops, name)
            setattr(self.ops, name, self._wrap(name, self._saved[name]) if name in CHECKERS else self._unknown(name))
        return self

    def __exit__(self, *exc):
        for name, fn in self._saved.items():
            setattr(self.ops, name, fn)
        self._saved = {}
        return False

    def _unknown(self, name):
        why = ("is exempt only because nothing called it; give it a checker before calling it" if name in UNCALLED else
               "has no checker (add one to CHECKERS or a reason to SHADOW_EXEMPT)")

        def call(*a, **k):
            raise AssertionError(f"shadow: ops.{name} launches a kernel and {why}")
        return call

    def _wrap(self, name, real):
        sig = inspect.signature(_REAL[name])
        checker, keyer = CHECKERS[name]

        def call(*args, **kwargs):
            ba = sig.bind(*args, **kwargs)
            ba.apply_defaults()
            A = ba.arguments
            key = (name,) + tuple(keyer(A))
            if name == "groupnorm_from_partials" and A["stats"] is not None:
                self.stats_eps[A["stats"].data_ptr()] = A["eps"]
            e = self.census.setdefault(key, Entry(name))
            e.calls += 1
            if e.checked >= self.first_n:
                return real(*args, **kwargs)
            e.checked += 1
            chk = Check(self, key, e)
            if checker is _Reward:
                ref_members = [m.clone() for m in A["members"]]
                out = real(*args, **kwargs)
                _sync(out)
                self._run(chk, lambda: self._reward(chk, out, ref_members))
                return out
            compare = checker(chk, A, self.random_rows)
            out = real(*args, **kwargs)
            _sync(next((t for t in A.values() if isinstance(t, torch.Tensor)), None))
            self._run(chk, compare)
            return out
        return call

    def _reward(self, chk, out, members):
        check_reward(out, members, chk.name)
        chk._note("elementwise", 0.0)

    def _run(self, chk, compare):
        try:
            compare()
        except AssertionError as err:
            self.failures[chk.key] = f"{chk.key[0]} key {chk.key[1:]}: {err}"

    def assert_ok(self):
        assert not self.failures, f"{len(self.failures)} launch configuration(s) failed:\n" + "\n".join(self.failures.values())

    def families(self):
        """op -> (distinct keys, checked keys, worst error / bound, worst rel-L2 / floor)."""
        out = {}
        for e in self.census.values():
            k, c, r, f = out.get(e.op, (0, 0, 0.0, 0.0))
            out[e.op] = (k + 1, c + (e.checked > 0), max(r, e.ratio), max(f, e.rel_floor))
        return out

    def report(self) -> str:
        lines = [f"{'op':<26}{'keys':>6}{'checked':>9}{'worst err/bound':>17}{'worst rel/floor':>17}"]
        for op, (k, c, r, f) in sorted(self.families().items()):
            lines.append(f"{op:<26}{k:>6}{c:>9}{r:>17.3f}{f:>17.3f}")
        lines.append(f"{len(self.census)} keys, {sum(e.calls for e in self.census.values())} calls, "
                     f"{len(self.failures)} failing")
        return "\n".join(lines)

    def checked_ops(self):
        return {e.op for e in self.census.values() if e.checked}
