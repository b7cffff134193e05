"""Python-side call wrappers over the C-ABI (include/vista_b200.h).

torch is used only for device memory and streams: every function takes CUDA tensors, hands their
raw pointers and the current stream to the library, and returns the (pre-allocated) output.
Activations are token-major fp16 ``[tokens, C]`` views (row stride = ``tensor.stride(0)``).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence, Tuple

import torch

from . import lib as _lib

TAPS_3X3 = [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]   # tap index = kh*3 + kw
TAPS_T3 = [(-1, 0), (0, 0), (1, 0)]                              # (3,1,1) conv: taps along frames
TAPS_1 = [(0, 0)]


LAUNCHES = 0   # kernels of this library launched so far (bench.py reports the per-step delta)


def _count(n: int = 1):
    global LAUNCHES
    LAUNCHES += n


TRACE = None   # debugging aid: set to a list to record (op, shape, checksum) after every launch (synchronises)


def _trace(name: str, out: torch.Tensor):
    if TRACE is not None:
        torch.cuda.synchronize()
        o = out.double()
        TRACE.append((name, tuple(out.shape), float(o.sum()), float(o.abs().sum())))


PROFILE = None   # set to a list: every launch is bracketed by CUDA events -> (family, detail, flops, bytes, ev0, ev1)
_prof_open = None


def _prof_begin(family: str, detail: str, flops: float, nbytes: float):
    global _prof_open
    if PROFILE is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        _prof_open = (family, detail, flops, nbytes, e0, e1)


def _prof_end():
    global _prof_open
    if PROFILE is not None and _prof_open is not None:
        _prof_open[5].record()
        PROFILE.append(_prof_open)
        _prof_open = None


def profile_summary(records):
    """Aggregates PROFILE records (after a synchronize) -> {family: dict(ms, launches, tflops, gbs)}, rows by detail."""
    fam, det = {}, {}
    for family, detail, flops, nbytes, e0, e1 in records:
        ms = e0.elapsed_time(e1)
        for table, key in ((fam, family), (det, (family, detail))):
            r = table.setdefault(key, dict(ms=0.0, launches=0, flops=0.0, bytes=0.0))
            r["ms"] += ms
            r["launches"] += 1
            r["flops"] += flops
            r["bytes"] += nbytes
    for table in (fam, det):
        for r in table.values():
            r["tflops"] = r["flops"] / (r["ms"] * 1e-3) / 1e12 if r["ms"] > 0 else 0.0
            r["gbs"] = r["bytes"] / (r["ms"] * 1e-3) / 1e9 if r["ms"] > 0 else 0.0
    return fam, det


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _rows(t: torch.Tensor) -> Tuple[int, int]:
    assert t.dim() == 2 and t.stride(1) == 1, "token-major 2-D view with unit channel stride expected"
    # launches go to the CURRENT device's current stream: a tensor living elsewhere would be dereferenced on the wrong GPU
    if t.is_cuda and t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"vista_b200: tensor on cuda:{t.device.index} but the current device is cuda:{torch.cuda.current_device()}; "
                           "wrap the call in torch.cuda.device(tensor.device)")
    return t.shape[0], t.stride(0)


def pick_box(W: int, H: int, NB: int) -> Tuple[int, int, int]:
    """Token tile (box_w, box_h, box_b) with product 128 minimising padded work."""
    best, best_cost = None, None
    for bw in (128, 64, 32, 16, 8, 4, 2, 1):
        for bh in (1, 2, 4, 8, 16, 32, 64, 128):
            if bw * bh > 128:
                continue
            bb = 128 // (bw * bh)
            tiles = -(-W // bw) * -(-H // bh) * -(-NB // bb)
            cost = (tiles, -bw)
            if best_cost is None or cost < best_cost:
                best, best_cost = (bw, bh, bb), cost
    return best


def stats_box(W: int, H: int, NB: int) -> Optional[Tuple[int, int, int]]:
    """Token tile of 128 CONSECUTIVE tokens (whole image rows, or a segment of one row) — what the fused GroupNorm
    statistics need so that tile i covers tokens [128 i, 128 i + 128) in every producer of a tensor; None if the geometry
    has no such tiling (then the statistics take their own pass)."""
    if W >= 128:
        return (128, 1, 1) if W % 128 == 0 else None
    if 128 % W == 0 and H % (128 // W) == 0:
        return (W, 128 // W, 1)
    return None


def upsample_stats_box(W: int, H: int) -> Optional[Tuple[int, int, int]]:
    """Low-resolution box (box_w, box_h, 1) of the upsampling tap-GEMM (``gemm(..., upsample=True)``) that tiles every
    frame exactly — what fused statistics need there; None if the geometry has none."""
    for bw in (128, 64, 32, 16, 8, 4, 2, 1):
        if W % bw == 0 and H % (128 // bw) == 0:
            return (bw, 128 // bw, 1)
    return None


def pick_tile_n(N: int, geglu: bool = False) -> int:
    """tile_n <= 256 (multiple of 32, of 64 for GEGLU) minimising the time of one row of n-tiles under a cost model
    with a fixed per-tile part (pipeline fill, epilogue set-up) and a part linear in the width above 128 columns,
    t(n) = 61 + 0.22 * max(n, 128): wide tiles win even when the last one is partly empty (every tile re-reads its A
    operand, so fewer tiles also mean less A traffic)."""
    step = 64 if geglu else 32
    best, best_cost = None, None
    for tn in range(256, step - 1, -step):
        if geglu and N % tn:
            continue
        tiles = -(-N // tn)
        cost = (round(tiles * (61.0 + 0.22 * max(tn, 128)), 3), tiles, tiles * tn - N)
        if best_cost is None or cost < best_cost:
            best, best_cost = tn, cost
    if best is None:
        raise ValueError(f"no tile_n for N={N} geglu={geglu}")
    return best


def gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, taps: Sequence[Tuple[int, int]] = TAPS_1,
         geom: Optional[Tuple[int, int, int]] = None, bias: Optional[torch.Tensor] = None,
         rowvec: Optional[torch.Tensor] = None, rv_div: int = 1, rv_mod: int = 1,
         res1: Optional[torch.Tensor] = None, s_res1: float = 1.0,
         res2: Optional[torch.Tensor] = None, s_res2: float = 1.0,
         s_acc: float = 1.0, act: int = 0, tile_n: Optional[int] = None, cin: Optional[int] = None,
         stats: Optional[torch.Tensor] = None, h_pad: int = 0, upsample: bool = False) -> torch.Tensor:
    """out = epilogue(tap-GEMM(a, w)).  ``a``: [tokens, >=cin] fp16 view; ``w``: [N, ntaps*cin] fp16;
    ``geom`` = (W, H, NB) turns on image taps (zero padded); act 1 = SiLU, act 2 = GEGLU (out has N/2 columns),
    act 3 = erf-GELU.
    ``stats`` = partials [tokens/128*4, N, 2] fp32 (may be a column slice of a wider matrix): the epilogue also writes,
    per 32-row quarter of each token tile, the column sum of the stored output and its sum of squared deviations from
    the quarter's mean (GroupNorm statistics of the consumer without a pass over the tensor, exact for groups whose
    mean is large next to their spread); the token tiles are then the 128-consecutive-token ones of stats_box().
    ``h_pad``: ``a`` holds h_pad extra rows of H before and after the H rows of ``geom`` (halo frames of the frame-sharded
    (3,1,1) convolution): ``a`` is the extended [(NB (H + 2 h_pad) W), C] tensor, the output has NB H W rows.
    ``upsample``: the taps run over the nearest-2x upsampled view of ``a`` (``geom`` is the geometry of ``a``; ``out`` and
    ``stats`` cover the 4x as many tokens of NB x 2H x 2W), without writing the upsampled tensor; bias and ``stats``
    are the only epilogue features, and the statistics boxes are upsample_stats_box()'s.
    ``bias`` / ``rowvec`` are fp32; ``res1`` / ``res2`` have the operand dtype whatever the output dtype (the kernel reads
    them as 16-bit values); GEGLU takes a bias only (no ``s_acc``)."""
    assert bias is None or bias.dtype == torch.float32, f"gemm: bias must be fp32, got {bias.dtype}"
    assert rowvec is None or rowvec.dtype == torch.float32, f"gemm: rowvec must be fp32, got {rowvec.dtype}"
    for r in (res1, res2):
        assert r is None or r.dtype == a.dtype, f"gemm: residual dtype {r.dtype} != operand dtype {a.dtype}"
    assert act != 2 or s_acc == 1.0, "gemm: the GEGLU epilogue does not scale by s_acc"
    tokens, lda = _rows(a)
    if h_pad:
        assert geom is not None and tokens == geom[2] * (geom[1] + 2 * h_pad) * geom[0]
        tokens = geom[0] * geom[1] * geom[2]
    N, K = w.shape
    ntaps = len(taps)
    cin = cin if cin is not None else K // ntaps
    assert K == ntaps * cin and w.is_contiguous()
    d = _lib.GemmDesc()
    d.a, d.lda, d.tokens = a.data_ptr(), lda, tokens
    out_tokens = 4 * tokens if upsample else tokens
    if geom is None:
        assert ntaps == 1 and not upsample
        d.a_mode = 0
    else:
        d.a_mode = 2 if upsample else 1
        d.W, d.H, d.NB = geom
        assert geom[0] * geom[1] * geom[2] == tokens
        if upsample and stats is not None:
            box = upsample_stats_box(geom[0], geom[1])
            assert box is not None, f"gemm: no box tiles the frames of {geom} for fused statistics"
        else:
            box = pick_box(*geom) if stats is None else stats_box(*geom)
        d.box_w, d.box_h, d.box_b = box
    d.cin, d.ntaps = cin, ntaps
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i] = dh, dw
    d.b, d.N = w.data_ptr(), N
    d.tile_n = tile_n if tile_n is not None else pick_tile_n(N, act == 2)
    d.bf16 = 1 if a.dtype == torch.bfloat16 else 0
    _, ldo = _rows(out)
    d.out, d.ldo, d.out_f32, d.act = out.data_ptr(), ldo, int(out.dtype == torch.float32), act
    d.bias = _ptr(bias)
    if rowvec is not None:
        d.rowvec, d.ld_rowvec, d.rv_div, d.rv_mod = rowvec.data_ptr(), rowvec.stride(0), rv_div, rv_mod
    if res1 is not None:
        d.res1, d.ld_res1, d.s_res1 = res1.data_ptr(), res1.stride(0), s_res1
    if res2 is not None:
        d.res2, d.ld_res2, d.s_res2 = res2.data_ptr(), res2.stride(0), s_res2
    d.s_acc = s_acc
    if stats is not None:      # [tokens/128*4, >= N, 2] fp32 view (possibly a column slice of a wider partial matrix)
        assert stats.dtype == torch.float32 and stats.dim() == 3 and stats.shape[2] == 2 and stats.stride(2) == 1 \
            and stats.stride(1) == 2 and stats.stride(0) % 2 == 0 and stats.shape[1] >= (N // 2 if act == 2 else N)
        assert stats.shape[0] >= -(-out_tokens // 128) * 4
        d.stats, d.stats_ld, d.stats_col0 = stats.data_ptr(), stats.stride(0) // 2, 0
    assert not upsample or out.shape[0] >= out_tokens
    d.h_pad = h_pad
    _count()
    n_out = N // 2 if act == 2 else N
    _prof_begin("gemm", f"M={out_tokens} N={N} K={K} taps={ntaps} act={act}{' up2x' if upsample else ''}",
                2.0 * out_tokens * N * K,
                2.0 * tokens * cin + 2.0 * N * K + out.element_size() * out_tokens * n_out
                + (2.0 * tokens * n_out if res1 is not None else 0) + (2.0 * tokens * n_out if res2 is not None else 0))
    _lib.check(_lib.load().b200v_gemm(C.byref(d), _stream()), "b200v_gemm")
    _prof_end()
    _trace(f"gemm taps={ntaps} act={act} N={N} K={K}", out)
    return out




def attention_spatial(q, k, v, out, frames: int, seq: int, heads: int, impl: Optional[int] = None):
    l = _lib.load()
    # both C-ABI entry points run the one wgmma kernel of csrc/attn_tc.cu; `impl=3` calls the `_v3` symbol (tests check both)
    fn = l.b200v_attention_spatial_v3 if impl == 3 else l.b200v_attention_spatial_v7
    _count(1)
    _prof_begin("attn_spatial", f"frames={frames} seq={seq} heads={heads}", 4.0 * 64 * heads * frames * seq * seq,
                2.0 * 4 * frames * seq * heads * 64)
    _lib.check(fn(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                  out.stride(0), frames, seq, heads, _stream()), "b200v_attention_spatial")
    _prof_end()
    _trace("attn_spatial", out)
    return out


def attention_d80(q, k, v, out, batch: int, seq: int, heads: int):
    """softmax(Q K^T / sqrt(80)) V per (image, head): q / k / v / out are [batch*seq, >= heads*80] fp16 views (column
    blocks of the CLIP tower's fused in-proj output), the output holds the merged heads."""
    for t in (q, k, v, out):
        _rows(t)
    _count(1)
    _prof_begin("attn_d80", f"batch={batch} seq={seq} heads={heads}", 4.0 * 80 * heads * batch * seq * seq,
                2.0 * 4 * batch * seq * heads * 80)
    _lib.check(_lib.load().b200v_attention_d80(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
                                               v.stride(0), out.data_ptr(), out.stride(0), batch, seq, heads, _stream()),
               "b200v_attention_d80")
    _prof_end()
    _trace("attn_d80", out)
    return out


def clip_preprocess(x, out, antialias: bool = True):
    """FrozenOpenCLIPImageEmbedder.preprocess + 14x14 patchify: x (n,3,H,W) fp32 in [-1, 1] -> out [n*257, K_pad] fp16
    (or fp32) patch rows (row b*257 is the zero class-token slot, columns 588.. are zero padding)."""
    n, c, H, W = x.shape
    assert c == 3 and x.dtype == torch.float32 and x.is_contiguous()
    _, ldo = _rows(out)
    assert out.shape[0] == n * 257 and out.dtype in (torch.float16, torch.float32)
    _count(1)
    _prof_begin("other", f"clip_preprocess n={n} {H}x{W}", 0.0, 4.0 * x.numel() + 2.0 * out.numel())
    _lib.check(_lib.load().b200v_clip_preprocess(x.data_ptr(), n, H, W, int(bool(antialias)), out.data_ptr(), ldo,
                                                 int(out.dtype == torch.float32), _stream()), "b200v_clip_preprocess")
    _prof_end()
    _trace("clip_preprocess", out)
    return out


def attention_temporal(q, k, v, out, nb: int, T: int, S: int, heads: int):
    _count(1)
    _prof_begin("attn_temporal", f"nb={nb} T={T} S={S} heads={heads}", 4.0 * 64 * heads * nb * S * T * T,
                2.0 * 4 * nb * T * S * heads * 64)
    _lib.check(_lib.load().b200v_attention_temporal(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0),
                                                    v.data_ptr(), v.stride(0), out.data_ptr(), out.stride(0),
                                                    nb, T, S, heads, _stream()), "b200v_attention_temporal")
    _prof_end()
    _trace("attn_temporal", out)
    return out


def groupnorm_scratch(frames: int, tokens_per_frame: int, groups: int = 32) -> int:
    """Doubles of partial-sum scratch b200v_groupnorm_stats needs for this shape."""
    chunk = _lib.load().b200v_groupnorm_chunk_for(frames, tokens_per_frame)
    return frames * (-(-tokens_per_frame // chunk)) * groups * 2


class GNWorkspace:
    """Scratch for the two-phase GroupNorm: partial sums (grown on demand) and self-resetting ticket counters."""

    def __init__(self, device, max_stats: int = 4096):
        self.device = device
        self.partials = torch.empty(1 << 16, dtype=torch.float64, device=device)
        self.counters = torch.zeros(max_stats, dtype=torch.int32, device=device)
        self._retired = []     # outgrown buffers stay alive: captured CUDA graphs / launch tapes hold their raw pointers

    def reserve(self, n_doubles: int):
        if self.partials.numel() < n_doubles:
            self._retired.append(self.partials)
            self.partials = torch.empty(n_doubles, dtype=torch.float64, device=self.device)


_default_ws = {}


def groupnorm(x, y, frames: int, tokens_per_frame: int, gamma, beta, eps: float, silu: bool,
              stats: Optional[torch.Tensor] = None, frames_per_stat: int = 1, groups: int = 32,
              ws: Optional[GNWorkspace] = None):
    """Two-phase GroupNorm; ``stats`` ([frames/frames_per_stat, groups, 2] fp32) receives (mean, rstd)."""
    Cc = gamma.numel()
    l = _lib.load()
    if ws is None:
        ws = _default_ws.setdefault(x.device, GNWorkspace(x.device))
    if stats is None:
        stats = torch.empty(frames // frames_per_stat, groups, 2, dtype=torch.float32, device=x.device)
    ws.reserve(groupnorm_scratch(frames, tokens_per_frame, groups))
    assert frames // frames_per_stat <= ws.counters.numel()
    _count(2)
    _prof_begin("groupnorm", f"tokens={frames * tokens_per_frame} C={Cc} fps={frames_per_stat}", 0.0,
                2.0 * 3 * frames * tokens_per_frame * Cc)
    _lib.check(l.b200v_groupnorm_stats(x.data_ptr(), x.stride(0), frames, tokens_per_frame, Cc, groups,
                                       frames_per_stat, eps, ws.partials.data_ptr(), ws.counters.data_ptr(),
                                       stats.data_ptr(), _stream()), "b200v_groupnorm_stats")
    _lib.check(l.b200v_groupnorm_apply(x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0), frames,
                                       tokens_per_frame, Cc, groups, frames_per_stat, stats.data_ptr(),
                                       gamma.data_ptr(), beta.data_ptr(), int(silu), _stream()),
               "b200v_groupnorm_apply")
    _prof_end()
    _trace(f"groupnorm fps={frames_per_stat}", y)
    return y


def groupnorm_from_partials(partials, frames: int, tokens_per_frame: int, Cc: int, eps: float, stats: Optional[torch.Tensor],
                            frames_per_stat: int = 1, groups: int = 32, raw_sums: Optional[torch.Tensor] = None):
    """(mean, rstd) [frames/frames_per_stat, groups, 2] from the column partials the producing GEMM(s) wrote; raw_sums
    (fp64) instead for the frame-sharded GroupNorm."""
    _count(1)
    _prof_begin("groupnorm", f"from_partials tokens={frames * tokens_per_frame} C={Cc} fps={frames_per_stat}", 0.0,
                4.0 * 2 * (frames * tokens_per_frame // 32) * Cc)
    assert partials.stride(1) == 2 and partials.stride(2) == 1 and partials.shape[1] == Cc
    _lib.check(_lib.load().b200v_groupnorm_from_partials(partials.data_ptr(), partials.stride(0) // 2, frames // frames_per_stat,
                                                         frames_per_stat, tokens_per_frame, Cc, groups, eps, _ptr(stats),
                                                         _ptr(raw_sums), _stream()), "b200v_groupnorm_from_partials")
    _prof_end()
    return stats


def groupnorm_apply(x, y, frames: int, tokens_per_frame: int, gamma, beta, silu: bool, stats: torch.Tensor,
                    frames_per_stat: int = 1, groups: int = 32):
    """The apply half of GroupNorm alone (statistics already in ``stats``)."""
    Cc = gamma.numel()
    _count(1)
    _prof_begin("groupnorm", f"apply tokens={frames * tokens_per_frame} C={Cc} fps={frames_per_stat}", 0.0,
                2.0 * 2 * frames * tokens_per_frame * Cc)
    _lib.check(_lib.load().b200v_groupnorm_apply(x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0), frames,
                                                 tokens_per_frame, Cc, groups, frames_per_stat, stats.data_ptr(),
                                                 gamma.data_ptr(), beta.data_ptr(), int(silu), _stream()),
               "b200v_groupnorm_apply")
    _prof_end()
    _trace(f"groupnorm(apply) fps={frames_per_stat}", y)
    return y


def groupnorm_sums(x, frames: int, tokens_per_frame: int, Cc: int, sums: torch.Tensor, frames_per_stat: int,
                   groups: int = 32, ws: Optional[GNWorkspace] = None):
    """Raw per-statistic (sum, sum of squares) in fp64 — first half of the frame-sharded temporal GroupNorm."""
    l = _lib.load()
    if ws is None:
        ws = _default_ws.setdefault(x.device, GNWorkspace(x.device))
    ws.reserve(groupnorm_scratch(frames, tokens_per_frame, groups))
    _count(1)
    _prof_begin("groupnorm", f"sums tokens={frames * tokens_per_frame} C={Cc} fps={frames_per_stat}", 0.0,
                2.0 * frames * tokens_per_frame * Cc)
    _lib.check(l.b200v_groupnorm_sums(x.data_ptr(), x.stride(0), frames, tokens_per_frame, Cc, groups, frames_per_stat,
                                      ws.partials.data_ptr(), ws.counters.data_ptr(), sums.data_ptr(), _stream()),
               "b200v_groupnorm_sums")
    _prof_end()
    return sums


def groupnorm_finalize_apply(x, y, frames: int, tokens_per_frame: int, gamma, beta, eps: float, silu: bool,
                             sums: torch.Tensor, count: float, stats: torch.Tensor, frames_per_stat: int, groups: int = 32):
    """Second half: (mean, rstd) from globally reduced sums, then the apply kernel."""
    l = _lib.load()
    Cc = gamma.numel()
    _count(2)
    _prof_begin("groupnorm", f"finalize+apply tokens={frames * tokens_per_frame} C={Cc} fps={frames_per_stat}", 0.0,
                2.0 * 2 * frames * tokens_per_frame * Cc)
    _lib.check(l.b200v_groupnorm_finalize(sums.data_ptr(), sums.numel() // 2, float(count), eps, stats.data_ptr(), _stream()),
               "b200v_groupnorm_finalize")
    _lib.check(l.b200v_groupnorm_apply(x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0), frames, tokens_per_frame, Cc,
                                       groups, frames_per_stat, stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                       int(silu), _stream()), "b200v_groupnorm_apply")
    _prof_end()
    return y


def attention_temporal_sharded(q, k, v, out, nb: int, Tq: int, T: int, S: int, heads: int, kv_frame_tok: torch.Tensor):
    _count(1)
    _prof_begin("attn_temporal", f"sharded nb={nb} Tq={Tq} T={T} S={S} heads={heads}", 4.0 * 64 * heads * nb * S * Tq * T,
                2.0 * (2 * nb * Tq + 2 * nb * T) * S * heads * 64)
    _lib.check(_lib.load().b200v_attention_temporal_sharded(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0),
                                                            v.data_ptr(), v.stride(0), out.data_ptr(), out.stride(0),
                                                            nb, Tq, T, S, heads, kv_frame_tok.data_ptr(), _stream()),
               "b200v_attention_temporal_sharded")
    _prof_end()
    return out


def layernorm(x, y, gamma, beta, eps: float = 1e-5, addvec=None, av_div: int = 1, av_mod: int = 1):
    tokens, ldx = _rows(x)
    _count(1)
    _prof_begin("layernorm", f"tokens={tokens} C={gamma.numel()}", 0.0, 2.0 * 2 * tokens * gamma.numel())
    _lib.check(_lib.load().b200v_layernorm(x.data_ptr(), ldx, y.data_ptr(), y.stride(0), tokens, gamma.numel(),
                                           gamma.data_ptr(), beta.data_ptr(), eps, _ptr(addvec),
                                           addvec.stride(0) if addvec is not None else 0, av_div, av_mod,
                                           _stream()), "b200v_layernorm")
    _prof_end()
    _trace("layernorm", y)
    return y


def conv3x3_small_cin(x8, cin: int, w, bias, out, NB: int, H: int, W: int):
    """3x3 convolution (padding 1) of x8 [NB*H*W, 8] fp16 (channels >= cin ignored) with fp32 w [cout, cin, 3, 3] into
    out [NB*H*W, >= cout] fp16.  The kernel has no row-stride argument: it reads x8 as rows of exactly 8 halves."""
    _, ldx = _rows(x8)
    assert x8.dtype == torch.float16 and ldx == 8, \
        f"conv3x3_small_cin: x8 must be fp16 rows of stride 8, got {x8.dtype} with row stride {ldx}"
    _count(1)
    _prof_begin("other", "conv3x3_small_cin", 0.0, 0.0)
    _lib.check(_lib.load().b200v_conv3x3_small_cin(x8.data_ptr(), cin, w.data_ptr(), _ptr(bias), out.data_ptr(),
                                                   out.stride(0), NB, H, W, w.shape[0], _stream()),
               "b200v_conv3x3_small_cin")
    _prof_end()
    return out


def conv3x3_small_cout(x, w, bias, out, NB: int, H: int, W: int):
    _count(1)
    _prof_begin("other", "conv3x3_small_cout", 0.0, 0.0)
    _lib.check(_lib.load().b200v_conv3x3_small_cout(x.data_ptr(), x.stride(0), w.shape[1], w.data_ptr(), _ptr(bias),
                                                    out.data_ptr(), NB, H, W, w.shape[0], _stream()),
               "b200v_conv3x3_small_cout")
    _prof_end()
    return out


def im2col_s2(x, out, NB: int, H: int, W: int, Cc: int):
    _count(1)
    _prof_begin("other", "im2col_s2", 0.0, 0.0)
    _lib.check(_lib.load().b200v_im2col_s2(x.data_ptr(), x.stride(0), out.data_ptr(), NB, H, W, Cc, _stream()),
               "b200v_im2col_s2")
    _prof_end()
    return out


def im2col_s2_asym(x, out, NB: int, H: int, W: int, Cc: int):
    """VAE-encoder Downsample gather (zero pad right / bottom only)."""
    _count(1)
    _prof_begin("other", "im2col_s2_asym", 0.0, 0.0)
    _lib.check(_lib.load().b200v_im2col_s2_asym(x.data_ptr(), x.stride(0), out.data_ptr(), NB, H, W, Cc, _stream()),
               "b200v_im2col_s2_asym")
    _prof_end()
    return out


def upsample2x(x, out, NB: int, H: int, W: int, Cc: int):
    _count(1)
    _prof_begin("other", "upsample2x", 0.0, 0.0)
    _lib.check(_lib.load().b200v_upsample2x(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), NB, H, W, Cc,
                                            _stream()), "b200v_upsample2x")
    _prof_end()
    return out


def timestep_embedding(t, out, dim: int, max_period: float = 10000.0):
    _count(1)
    _prof_begin("other", "timestep_embedding", 0.0, 0.0)
    _lib.check(_lib.load().b200v_timestep_embedding(t.data_ptr(), t.numel(), dim, max_period, out.data_ptr(),
                                                    out.stride(0), _stream()), "b200v_timestep_embedding")
    _prof_end()
    return out


def sinusoid_embed(values: Optional[torch.Tensor], slots: Sequence[Tuple[int, int, int, int, bool, int]],
                   freqs: Optional[torch.Tensor], out: torch.Tensor):
    """Every sinusoidal-embedder slot of one conditioning tensor in one launch (csrc/cond.cu).  out: fp32 [rows, >= cols]
    (row stride out.stride(0)); values: fp32 [rows, n_values] or None when every slot is zero; slots: (value_col,
    num_features, outdim, dst_col, zero, freq_off); freqs: fp32 frequency table on the device."""
    rows, ldo = _rows(out)
    assert out.dtype == torch.float32 and 0 < len(slots) <= _lib.SINUSOID_MAX_SLOTS
    if values is not None:
        _, ldv = _rows(values)
        assert values.dtype == torch.float32 and values.shape[0] == rows
    else:
        ldv = 0
    assert freqs is None or (freqs.dtype == torch.float32 and freqs.is_contiguous())
    tab = _lib.SinusoidTable()
    tab.n_slots = len(slots)
    for i, (vc, nf, od, dc, zero, fo) in enumerate(slots):
        s = tab.slot[i]
        s.value_col, s.num_features, s.outdim, s.dst_col, s.zero, s.freq_off = vc, nf, od, dc, int(bool(zero)), fo
    _count(1)
    _prof_begin("other", f"sinusoid_embed rows={rows} slots={len(slots)}", 0.0, 4.0 * rows * out.shape[1])
    _lib.check(_lib.load().b200v_sinusoid_embed(_ptr(values), ldv, rows, C.byref(tab), _ptr(freqs), out.data_ptr(), ldo,
                                                _stream()), "b200v_sinusoid_embed")
    _prof_end()
    _trace("sinusoid_embed", out)
    return out


def blend_emb(e_plain, e_cond, label, mask, emb, silu_emb):
    rows, dim = e_plain.shape
    _count(1)
    _prof_begin("other", "blend_emb", 0.0, 0.0)
    _lib.check(_lib.load().b200v_blend_emb(e_plain.data_ptr(), _ptr(e_cond), _ptr(label), _ptr(mask), _ptr(emb),
                                           _ptr(silu_emb), rows, dim, _stream()), "b200v_blend_emb")
    _prof_end()


def sampler_prepare(x, cond_frame, mask, concat_u, concat_c, sigmas, step_idx, unet_in, c_noise, T, h, w):
    _count(1)
    _prof_begin("other", "sampler_prepare", 0.0, 0.0)
    _lib.check(_lib.load().b200v_sampler_prepare(x.data_ptr(), _ptr(cond_frame), _ptr(mask), _ptr(concat_u),
                                                 _ptr(concat_c), sigmas.data_ptr(), step_idx.data_ptr(), unet_in.data_ptr(),
                                                 unet_in.stride(0), _ptr(c_noise), T, h, w, _stream()), "b200v_sampler_prepare")
    _prof_end()


def sampler_update(x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w):
    _count(2)
    _prof_begin("other", "sampler_update", 0.0, 0.0)
    _lib.check(_lib.load().b200v_sampler_update(x.data_ptr(), net_out.data_ptr(), net_out.stride(0), _ptr(cond_frame), _ptr(mask),
                                                scales.data_ptr(), sigmas.data_ptr(), step_idx.data_ptr(), num_steps,
                                                T, h, w, _stream()), "b200v_sampler_update")
    _prof_end()


def sampler_update_2m(x, net_out, cond_frame, mask, scales, coefs, d_prev, sigmas, step_idx, num_steps, T, h, w):
    """The DPM-Solver++(2M) step: ``coefs`` is the fp32 (>= num_steps, 4) table of ``diffusion.dpmpp2m_coefficients``,
    ``d_prev`` the (T, 4, h, w) fp32 denoised value of the previous step (read only on second-order rows)."""
    _count(2)
    _prof_begin("other", "sampler_update_2m", 0.0, 0.0)
    _lib.check(_lib.load().b200v_sampler_update_2m(x.data_ptr(), net_out.data_ptr(), net_out.stride(0), _ptr(cond_frame),
                                                   _ptr(mask), scales.data_ptr(), coefs.data_ptr(), d_prev.data_ptr(),
                                                   sigmas.data_ptr(), step_idx.data_ptr(), num_steps, T, h, w, _stream()),
               "b200v_sampler_update_2m")
    _prof_end()


def sampler_update_action(x, net_out, net_img, cond_frame, mask, scales, action_scales, coefs, d_prev, sigmas, step_idx,
                          num_steps, T, h, w):
    """The step under action guidance: ``net_img`` is the [T h w, >= 4] fp32 output of the conditional rows with the
    action slots zeroed, ``action_scales`` the (T,) device array of s_act.  ``coefs`` / ``d_prev`` as in
    ``sampler_update_2m`` for the 2M step, both None for the Euler step."""
    _count(2)
    _prof_begin("other", "sampler_update_action", 0.0, 0.0)
    _lib.check(_lib.load().b200v_sampler_update_action(x.data_ptr(), net_out.data_ptr(), net_out.stride(0),
                                                       net_img.data_ptr(), net_img.stride(0), _ptr(cond_frame), _ptr(mask),
                                                       scales.data_ptr(), action_scales.data_ptr(), _ptr(coefs),
                                                       _ptr(d_prev), sigmas.data_ptr(), step_idx.data_ptr(), num_steps, T,
                                                       h, w, _stream()),
               "b200v_sampler_update_action")
    _prof_end()


def _sampler_update_cond(x, net_c, cond_frame, mask, coefs, d_prev, sigmas, step_idx, num_steps, T, h, w):
    """The unguided step, for the fused loop of vista_b200.fused (its one caller), so not part of the public ops surface
    that the production-path launch checks enumerate; tests/test_interval_cfg_gpu.py holds the kernel to fp64.
    ``net_c`` is the [T h w, >= 4] fp32 output of the T conditional rows only, D = D_c.
    ``coefs`` / ``d_prev`` as in ``sampler_update_2m`` for the 2M step (D is written to ``d_prev``), both None for the
    Euler step."""
    _count(2)
    _prof_begin("other", "sampler_update_cond", 0.0, 0.0)
    _lib.check(_lib.load().b200v_sampler_update_cond(x.data_ptr(), net_c.data_ptr(), net_c.stride(0), _ptr(cond_frame),
                                                     _ptr(mask), _ptr(coefs), _ptr(d_prev), sigmas.data_ptr(),
                                                     step_idx.data_ptr(), num_steps, T, h, w, _stream()),
               "b200v_sampler_update_cond")
    _prof_end()


def nchw_to_tokens(x, out, NB, Cc, H, W):
    _count(1)
    _prof_begin("other", "nchw_to_tokens", 0.0, 0.0)
    _lib.check(_lib.load().b200v_nchw_to_tokens(x.data_ptr(), out.data_ptr(), out.stride(0), NB, Cc, H, W, _stream()),
               "b200v_nchw_to_tokens")
    _prof_end()
    return out


def tokens_to_nchw(x, out, NB, Cc, H, W):
    _count(1)
    _prof_begin("other", "tokens_to_nchw", 0.0, 0.0)
    _lib.check(_lib.load().b200v_tokens_to_nchw(x.data_ptr(), int(x.dtype == torch.float32), x.stride(0),
                                                out.data_ptr(), NB, Cc, H, W, _stream()), "b200v_tokens_to_nchw")
    _prof_end()
    return out


def softmax_rows(x, y):
    rows, cols = x.shape
    _count(1)
    _prof_begin("other", "softmax_rows", 0.0, 0.0)
    _lib.check(_lib.load().b200v_softmax_rows(x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0), rows, cols, _stream()),
               "b200v_softmax_rows")
    _prof_end()
    return y


def time_mix_small(x, w, bias, out, blend, T, HW, Cc, out_frame0=0, skip_frames=0):
    _count(1)
    _prof_begin("other", "time_mix_small", 0.0, 0.0)
    _lib.check(_lib.load().b200v_time_mix_small(x.data_ptr(), x.stride(0), w.data_ptr(), _ptr(bias), out.data_ptr(), _ptr(blend),
                                                T, HW, Cc, out_frame0, skip_frames, _stream()), "b200v_time_mix_small")
    _prof_end()
    return out


def time_mix_small_u8(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0=0, skip_frames=0, keep_f32_from=-1):
    """time_mix_small that also writes the uint8 NHWC frames of the reference's output path (sample_utils.py:96-126,374)."""
    assert out_u8.dtype == torch.uint8 and out_u8.is_contiguous()
    _count(1)
    _prof_begin("other", "time_mix_small_u8", 0.0, 0.0)
    _lib.check(_lib.load().b200v_time_mix_small_u8(x.data_ptr(), x.stride(0), w.data_ptr(), _ptr(bias), out.data_ptr(),
                                                   out_u8.data_ptr(), _ptr(blend), T, HW, Cc, out_frame0, skip_frames,
                                                   keep_f32_from, _stream()), "b200v_time_mix_small_u8")
    _prof_end()
    return out_u8


def rollout_advance(sample, z0, samples_z, filled, dst_frame0: int, src_frame0: int, n_cond: int):
    """sample_utils.py:335-337,350,362 as one launch (see include/vista_b200.h)."""
    T = sample.shape[0]
    E = sample[0].numel()
    assert sample.is_contiguous() and samples_z.is_contiguous() and sample.dtype == torch.float32
    assert filled is None or (filled.is_contiguous() and filled.shape == sample.shape)
    assert samples_z.shape[0] >= dst_frame0 + T
    _count(1)
    _lib.check(_lib.load().b200v_rollout_advance(sample.data_ptr(), _ptr(z0), samples_z.data_ptr(), _ptr(filled), T, E,
                                                 dst_frame0, src_frame0, n_cond, _stream()), "b200v_rollout_advance")
    return samples_z


def frames_u8_resize(frames, box, out, xtab, ytab, y_first: int, y_rows: int, scratch=None):
    """load_img's crop + LANCZOS resize + ToTensor + ``* 2 - 1`` (csrc/ingest/ingest.cu): frames (T, Hs, Ws, 3) uint8 with
    adjacent channels, box = (left, top, crop_w, crop_h) -> out (T, 3, H, W) fp32.  xtab / ytab = (bounds, weights, ksize)
    on the device (vista_b200.ingest.device_tables), None for an axis whose size is unchanged; scratch holds
    (T, y_rows, W, 3) uint8 when the width changes."""
    T, Hs, Ws, _ = frames.shape
    _, _, H, W = out.shape
    left, top, cw, ch = box
    assert frames.dtype == torch.uint8 and frames.stride(3) == 1 and frames.stride(2) == 3
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape[:2] == (T, 3)
    assert scratch is None or (scratch.dtype == torch.uint8 and scratch.numel() >= T * y_rows * W * 3)
    xb, xw, xk = xtab if xtab is not None else (None, None, 0)
    yb, yw, yk = ytab if ytab is not None else (None, None, 0)
    _count(1 + (xtab is not None))
    mid = T * y_rows * W * 3 if xtab is not None else 0
    _prof_begin("other", f"frames_u8_resize T={T} {Ws}x{Hs}->{W}x{H}", 0.0, float(T * ch * cw * 3 + 2 * mid + out.numel() * 4))
    _lib.check(_lib.load().b200v_frames_u8_resize(frames.data_ptr(), frames.stride(0), frames.stride(1), T, Hs, Ws, left, top,
                                                  cw, ch, H, W, _ptr(xb), _ptr(xw), xk, _ptr(yb), _ptr(yw), yk, y_first,
                                                  y_rows, _ptr(scratch), out.data_ptr(), _stream()),
               "b200v_frames_u8_resize")
    _prof_end()
    _trace("frames_u8_resize", out)
    return out


_reward_ws = {}


def ensemble_reward(members: Sequence[torch.Tensor]) -> torch.Tensor:
    """[mean variance, reward = exp(-mean variance)] of an ensemble of equally shaped fp32 samples (reward_utils.py:327-333)."""
    K, n, dev = len(members), members[0].numel(), members[0].device
    assert all(m.is_contiguous() and m.dtype == torch.float32 and m.numel() == n for m in members)
    l = _lib.load()
    ws = _reward_ws.get(dev)
    if ws is None:
        ws = _reward_ws[dev] = (torch.empty(l.b200v_ensemble_reward_scratch(), dtype=torch.float64, device=dev),
                                torch.zeros(1, dtype=torch.int32, device=dev))
    ptrs = torch.tensor([m.data_ptr() for m in members], dtype=torch.int64).to(dev)
    out = torch.empty(2, dtype=torch.float32, device=dev)
    _count(1)
    _lib.check(l.b200v_ensemble_reward(ptrs.data_ptr(), K, n, ws[0].data_ptr(), ws[1].data_ptr(), out.data_ptr(), _stream()),
               "b200v_ensemble_reward")
    out._keepalive = (ptrs, tuple(members))      # the launch is asynchronous
    return out


# ------------------------------------------------------------------------------------------------------------------
# Peer-memory collectives (csrc/peer.cu): thin wrappers; the window bookkeeping lives in vista_b200/peer.py
# ------------------------------------------------------------------------------------------------------------------
def peer_allreduce_f64(data: torch.Tensor, windows_dev: torch.Tensor, slot_off: int, flag_off: int, rank: int, world: int,
                       counter: torch.Tensor):
    assert data.dtype == torch.float64 and data.is_contiguous()
    _count(1)
    _prof_begin("peer", f"allreduce_f64 n={data.numel()}", 0.0, 8.0 * data.numel() * world)
    _lib.check(_lib.load().b200v_peer_allreduce_f64(data.data_ptr(), data.numel(), windows_dev.data_ptr(), slot_off, flag_off,
                                                    rank, world, counter.data_ptr(), _stream()), "b200v_peer_allreduce_f64")
    _prof_end()
    return data


def peer_put(src_ptr: int, src_pitch: int, rows: int, row_bytes: int, dsts_dev: torch.Tensor, dst_pitch: int,
             flags_dev: torch.Tensor, n_dst: int, counter: torch.Tensor, ticket: torch.Tensor, detail: str = ""):
    _count(1)
    _prof_begin("peer", f"put {detail} bytes={rows * row_bytes} x{n_dst}", 0.0, float(rows * row_bytes * (n_dst + 1)))
    _lib.check(_lib.load().b200v_peer_put(src_ptr, src_pitch, rows, row_bytes, dsts_dev.data_ptr(), dst_pitch, flags_dev.data_ptr(),
                                          n_dst, counter.data_ptr(), ticket.data_ptr(), _stream()), "b200v_peer_put")
    _prof_end()


def peer_wait(flags_dev: torch.Tensor, n: int, counter: torch.Tensor, detail: str = ""):
    _count(1)
    _prof_begin("peer", f"wait {detail}", 0.0, 0.0)
    _lib.check(_lib.load().b200v_peer_wait(flags_dev.data_ptr(), n, counter.data_ptr(), _stream()), "b200v_peer_wait")
    _prof_end()
