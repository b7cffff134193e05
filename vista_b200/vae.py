"""B200 executor of the temporal VAE decoder and of the chunked ``decode_first_stage``.

Reference behaviour (paths relative to the reference root):
  VideoDecoder.forward ......... vwm/modules/diffusionmodules/model.py:664-694 + autoencoding/temporal_ae.py:105-151
  decoder VideoResBlock ........ temporal_ae.py:55-72 on model.py:116-135 (GN eps 1e-6, swish); temporal
                                 openaimodel.ResBlock with skip_t_emb (GN32 eps 1e-5); alpha*temporal + (1-alpha)*spatial
  AttnBlock (1 head, d = C) .... model.py:147-176
  AE3DConv ..................... temporal_ae.py:75-97
  decode_first_stage ........... vwm/models/diffusion.py:150-180 (14-frame chunks, 3-frame overlap averaged)

The reference runs this stage in fp32 (autocast disabled, configs/inference/vista.yaml:6); here the
convolutions run on fp16 tensor cores with fp32 accumulation and fp32/fp64 normalisation statistics —
the stated tolerance is in tests/test_decoder_gpu.py.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .modules import register_param_tree
from .spec import DecoderConfig, DecResBlockSpec, build_decoder_plan, decoder_param_specs
from .unet import Lin
from .weights import conv_weight_to_taps

_SCRATCH_ALIGN = 4096      # byte alignment of every role in the decoder's arena (TMA needs 16)


def _fuses(T: int, h: int, w: int) -> bool:
    """Whether the decoder's convolutions at this geometry write their output's GroupNorm partials (ops.stats_box)."""
    return ops.stats_box(w, h, T) is not None


class ScratchPlan(NamedTuple):
    """The decoder's scratch for one (T, h, w): ``roles`` maps each role to (byte offset, bytes) in one arena of ``total``
    bytes; ``uses`` lists every view DecoderRuntime.forward takes, in order, as (role, shape, dtype, first op, last op):
    the view lives from the op that writes it to the last op that reads it.  Roles whose views are never live at the same
    op may share storage."""
    roles: Dict[str, Tuple[int, int]]
    uses: List[Tuple[str, Tuple[int, ...], torch.dtype, int, int]]
    total: int


def _decoder_scratch_uses(cfg: DecoderConfig, T: int, h: int, w: int):
    """Replays DecoderRuntime.forward's scratch traffic op by op: the role (and shape) every op writes and the views it
    reads.  Must follow forward / _resblock / _attn; the CPU executor tests run the decoder on this plan."""
    uses, step = [], [0]
    f16, f32 = torch.float16, torch.float32

    def op(reads, *writes):
        for u in reads:
            if u is not None:
                u[4] = step[0]
        out = [None if wr is None else [wr[0], wr[1], wr[2] if len(wr) > 2 else f16, step[0], step[0]] for wr in writes]
        uses.extend(u for u in out if u is not None)
        step[0] += 1
        return out

    def part(role, M, Cc, fuse):
        return ("part." + role, (-(-M // 128) * 4, Cc, 2), f32) if fuse else None

    def resblock(rb: DecResBlockSpec, x, xp, h, w, name):
        M, fuse, co = T * h * w, _fuses(T, h, w), rb.cout
        a1, = op([x, xp], ("d.a1", (M, rb.cin)))
        h1, p1 = op([a1], ("d.h1", (M, co)), part("d.h1", M, co, fuse))
        a2, = op([h1, p1], ("d.a2", (M, co)))
        xs = op([x], ("d.xs", (M, co)))[0] if rb.has_skip else x
        xsp, p2 = op([a2, xs], ("d.xsp", (M, co)), part("d.xsp", M, co, fuse))
        a3, = op([xsp, p2], ("d.a1", (M, co)))
        h2, p1 = op([a3], ("d.h1", (M, co)), part("d.h1", M, co, fuse))
        a4, = op([h2, p1], ("d.a2", (M, co)))
        return op([a4, xsp], (name, (M, co)), part(name, M, co, fuse))

    def attn(x, xp, h, w, Cc):
        M, hw = T * h * w, h * w
        xn, = op([x, xp], ("d.a1", (M, Cc)))
        q, = op([xn], ("d.q", (M, Cc)))
        k, = op([xn], ("d.k", (M, Cc)))
        # the per-frame loop: V^T, S, P and O are all live until O is complete
        _, _, _, o = op([xn, q, k], ("d.vT", (Cc, hw)), ("d.s", (hw, hw), f32), ("d.p", (hw, hw)), ("d.o", (M, Cc)))
        return op([o, x], ("d.attn_y", (M, Cc)), part("d.attn_y", M, Cc, _fuses(T, h, w)))

    plan = build_decoder_plan(cfg)
    x, = op([], ("d.in", (T * h * w, plan.block_in)))
    x, xp = resblock(plan.mid[0], x, None, h, w, "d.r0")
    x, xp = attn(x, xp, h, w, plan.block_in)
    x, xp = resblock(plan.mid[1], x, xp, h, w, "d.r1")
    for blocks, up, ch in plan.levels:
        for bi, rb in enumerate(blocks):
            x, xp = resblock(rb, x, xp, h, w, f"d.r{bi % 2}")
        if up is not None:
            fuse = _fuses(T, 2 * h, 2 * w) and ops.upsample_stats_box(w, h) is not None
            h, w = 2 * h, 2 * w
            x, xp = op([x], ("d.upc", (T * h * w, ch)), part("d.upc", T * h * w, ch, fuse))
    M = T * h * w
    a, = op([x, xp], ("d.a1", (M, plan.final_ch)))
    y, = op([a], ("d.y", (M, 8), f32))
    op([y])
    return [tuple(u) for u in uses]


def decoder_scratch_plan(cfg: DecoderConfig, T: int, h: int, w: int) -> ScratchPlan:
    """Scratch of DecoderRuntime.forward for T frames of h x w latents: every role sized once for its largest view, and
    placed first-fit (largest role first) at the lowest offset clear of every role it is live together with at some op."""
    size: Dict[str, int] = {}
    live: Dict[str, list] = {}
    uses = _decoder_scratch_uses(cfg, T, h, w)
    for role, shape, dtype, first, last in uses:
        n = dtype.itemsize
        for s in shape:
            n *= s
        size[role] = max(size.get(role, 0), -(-n // _SCRATCH_ALIGN) * _SCRATCH_ALIGN)
        live.setdefault(role, []).append((first, last))

    def together(r1, r2):
        return any(a0 <= b1 and b0 <= a1 for a0, a1 in live[r1] for b0, b1 in live[r2])

    roles: Dict[str, Tuple[int, int]] = {}
    for role in sorted(size, key=lambda r: (-size[r], r)):
        off = 0
        for s, e in sorted((roles[o][0], roles[o][0] + roles[o][1]) for o in roles if together(role, o)):
            if off + size[role] <= s:
                break
            off = max(off, e)
        roles[role] = (off, size[role])
    return ScratchPlan(roles, uses, max(o + n for o, n in roles.values()))


class DecoderRuntime:
    # forward's scratch: one arena laid out by decoder_scratch_plan (roles: set while forward runs; the encoder and the
    # frame-sharded decoder keep per-name buffers, buf())
    _arena: Optional[torch.Tensor] = None
    _arena_key: Optional[Tuple[int, int, int]] = None
    _roles: Optional[Dict[str, Tuple[int, int]]] = None

    def __init__(self, cfg: DecoderConfig, sd: Dict[str, torch.Tensor], device):
        self.cfg, self.dev = cfg, torch.device(device)
        self.plan = build_decoder_plan(cfg)
        self._bufs = {}
        self._sd = sd
        self._pack()
        self._sd = None

    # ------------------------------------------------------------------ packing
    def _f32(self, name):
        return self._sd[name].detach().to(self.dev, torch.float32).contiguous()

    def _lin(self, prefix) -> Lin:
        w = self._sd[f"{prefix}.weight"].detach().to(self.dev, torch.float32)
        w = conv_weight_to_taps(w) if w.dim() > 2 else w
        return Lin(w.to(torch.float16).contiguous(), self._f32(f"{prefix}.bias"), ops.pick_tile_n(w.shape[0]))

    def _norm(self, prefix):
        return self._f32(f"{prefix}.weight"), self._f32(f"{prefix}.bias")

    def _pack(self):
        sd = self._sd
        self.n_gn = 0
        self.res: Dict[str, dict] = {}

        def pack_res(rb: DecResBlockSpec):
            p, t = rb.prefix, f"{rb.prefix}.time_stack"
            self.res[p] = dict(spec=rb, gn1=self._norm(f"{p}.norm1"), conv1=self._lin(f"{p}.conv1"),
                               gn2=self._norm(f"{p}.norm2"), conv2=self._lin(f"{p}.conv2"),
                               skip=self._lin(f"{p}.nin_shortcut") if rb.has_skip else None,
                               tgn1=self._norm(f"{t}.in_layers.0"), tconv1=self._lin(f"{t}.in_layers.2"),
                               tgn2=self._norm(f"{t}.out_layers.0"), tconv2=self._lin(f"{t}.out_layers.3"),
                               alpha=float(torch.sigmoid(sd[f"{p}.mix_factor"].float()).item()), gn_idx=self.n_gn)
            self.n_gn += 4

        self.conv_in_w, self.conv_in_b = self._f32("conv_in.weight"), self._f32("conv_in.bias")
        pack_res(self.plan.mid[0])
        a = "mid.attn_1"
        wq = self._lin(f"{a}.q")
        self.attn = dict(norm=self._norm(f"{a}.norm"), q=wq, k=self._lin(f"{a}.k"),
                         v_w=conv_weight_to_taps(sd[f"{a}.v.weight"].detach().to(self.dev, torch.float32)).to(torch.float16).contiguous(),
                         v_b=self._f32(f"{a}.v.bias"), proj=self._lin(f"{a}.proj_out"), gn_idx=self.n_gn)
        self.n_gn += 1
        pack_res(self.plan.mid[1])
        self.ups = {}
        for blocks, up, ch in self.plan.levels:
            for rb in blocks:
                pack_res(rb)
            if up is not None:
                self.ups[up] = self._lin(up)
        self.norm_out = self._norm("norm_out")
        self.norm_out_idx = self.n_gn
        self.n_gn += 1
        ow = conv_weight_to_taps(self._f32("conv_out.weight"))
        w8 = torch.zeros(8, ow.shape[1], dtype=torch.float16, device=self.dev)
        w8[: ow.shape[0]] = ow.to(torch.float16)
        b8 = torch.zeros(8, dtype=torch.float32, device=self.dev)
        b8[: ow.shape[0]] = self._f32("conv_out.bias")
        self.out_conv = Lin(w8.contiguous(), b8, 32)
        self.tmix_w = self._f32("conv_out.time_mix_conv.weight").reshape(self.cfg.out_ch, self.cfg.out_ch, 3).contiguous()
        self.tmix_b = self._f32("conv_out.time_mix_conv.bias")

    # ------------------------------------------------------------------ helpers
    def _scratch(self, role, shape, dtype):
        """View of ``role``'s storage in the planned arena (inside forward)."""
        off, size = self._roles[role]
        n = dtype.itemsize
        for s in shape:
            n *= s
        assert n <= size, f"decoder scratch: {role} {shape} exceeds its planned {size} bytes"
        return self._arena[off:off + n].view(dtype).view(*shape)

    def buf(self, name, rows, cols, dtype=torch.float16):
        if self._roles is not None:
            return self._scratch(name, (rows, cols), dtype)
        key = (name, rows, cols, dtype)
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = torch.empty(rows, cols, dtype=dtype, device=self.dev)
        return t

    def gemm(self, a, lin: Lin, out, **kw):
        return ops.gemm(a, lin.w, out, bias=lin.b, tile_n=lin.tile_n, **kw)

    def _gn(self, x, y, T, hw, norm, eps, idx, fps=1, part=None, silu=True):
        """GroupNorm (+ swish).  part: column partials of x from its producing GEMM (ops.gemm(stats=...)): the statistics
        are then one small reduction instead of a pass over x."""
        stats = self.gn_stats[idx, : T // fps]
        if part is None:
            return ops.groupnorm(x, y, T, hw, norm[0], norm[1], eps, silu, stats, frames_per_stat=fps,
                                 groups=self.cfg.num_groups, ws=self.gn_ws)
        ops.groupnorm_from_partials(part, T, hw, norm[0].numel(), eps, stats, fps, self.cfg.num_groups)
        return ops.groupnorm_apply(x, y, T, hw, norm[0], norm[1], silu, stats, fps, self.cfg.num_groups)

    def part(self, name: str, tokens: int, cols: int) -> torch.Tensor:
        if self._roles is not None:        # every partial the kernels read was written before (whole-frame tiles)
            return self._scratch("part." + name, (-(-tokens // 128) * 4, cols, 2), torch.float32)
        key = ("part." + name, tokens, cols)
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = torch.zeros(-(-tokens // 128) * 4, cols, 2, dtype=torch.float32, device=self.dev)
        return t

    def _fuse_stats(self, T, h, w) -> bool:
        return _fuses(T, h, w)

    def _upsample_in_gemm(self) -> bool:
        """The up-convolutions read the low-resolution tensor (tap-GEMM a_mode 2) on CUDA, the only device the kernels
        run on.  A runtime on another device only runs on the host-executor tests' CPU emulation of the operators, which
        covers upsample2x and the image-tap GEMM but not the upsampling mode: there the 2x upsample is materialised."""
        return self.dev.type == "cuda"

    def _resblock(self, L, x, T, h, w, name, xp=None):
        """Returns (output, its GroupNorm column partials or None); xp: those of x."""
        rb: DecResBlockSpec = L["spec"]
        hw, M, gi = h * w, T * h * w, L["gn_idx"]
        fuse = self._fuse_stats(T, h, w)
        p1 = self.part("d.h1", M, rb.cout) if fuse else None
        p2 = self.part("d.xsp", M, rb.cout) if fuse else None
        pd = self.part(name, M, rb.cout) if fuse else None
        a1 = self._gn(x, self.buf("d.a1", M, rb.cin), T, hw, L["gn1"], 1e-6, gi, part=xp)
        h1 = self.gemm(a1, L["conv1"], self.buf("d.h1", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, T), stats=p1)
        a2 = self._gn(h1, self.buf("d.a2", M, rb.cout), T, hw, L["gn2"], 1e-6, gi + 1, part=p1)
        xs = x if L["skip"] is None else self.gemm(x, L["skip"], self.buf("d.xs", M, rb.cout))
        xsp = self.gemm(a2, L["conv2"], self.buf("d.xsp", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, T), res1=xs, stats=p2)
        a3 = self._gn(xsp, self.buf("d.a1", M, rb.cout), T, hw, L["tgn1"], 1e-5, gi + 2, fps=T, part=p2)
        h2 = self.gemm(a3, L["tconv1"], self.buf("d.h1", M, rb.cout), taps=ops.TAPS_T3, geom=(hw, T, 1), stats=p1)
        a4 = self._gn(h2, self.buf("d.a2", M, rb.cout), T, hw, L["tgn2"], 1e-5, gi + 3, fps=T, part=p1)
        # alpha*(xsp + conv) + (1-alpha)*xsp = xsp + alpha*(conv + bias)            (temporal_ae.py:68-69)
        out = self.buf(name, M, rb.cout)
        self.gemm(a4, L["tconv2"], out, taps=ops.TAPS_T3, geom=(hw, T, 1), s_acc=L["alpha"], res1=xsp, stats=pd)
        return out, pd

    def _attn(self, x, T, h, w, xp=None):
        """GN -> q,k,v (1x1) -> softmax(q k^T / sqrt(C)) v -> proj_out -> + x, one head of dim C, per frame.
        Returns (output, its GroupNorm column partials or None)."""
        A = self.attn
        Cc, hw, M = x.shape[1], h * w, T * h * w
        assert hw % 64 == 0, "decoder attention needs h*w to be a multiple of 64"
        y = self.buf("d.attn_y", M, Cc)
        yp = self.part("d.attn_y", M, Cc) if self._fuse_stats(T, h, w) else None
        xn = self._gn(x, self.buf("d.a1", M, Cc), T, hw, A["norm"], 1e-6, A["gn_idx"], part=xp, silu=False)
        q = self.gemm(xn, A["q"], self.buf("d.q", M, Cc))
        k = self.gemm(xn, A["k"], self.buf("d.k", M, Cc))
        o = self.buf("d.o", M, Cc)
        s = self.buf("d.s", hw, hw, torch.float32)
        p = self.buf("d.p", hw, hw)
        vT = self.buf("d.vT", Cc, hw)
        for f in range(T):
            rows = slice(f * hw, (f + 1) * hw)
            ops.gemm(A["v_w"], xn[rows], vT)         # V^T = W_v x^T; v bias is added after PV (softmax rows sum to 1)
            ops.gemm(q[rows], k[rows], s, s_acc=float(Cc) ** -0.5)
            ops.softmax_rows(s, p)
            ops.gemm(p, vT, o[rows], bias=A["v_b"])
        self.gemm(o, A["proj"], y, res1=x, stats=yp)
        return y, yp

    # ------------------------------------------------------------------ forward
    def forward(self, z_tokens: torch.Tensor, T: int, h: int, w: int, out: torch.Tensor, out_frame0: int = 0,
                blend: Optional[torch.Tensor] = None, skip_frames: int = 0, out_u8: Optional[torch.Tensor] = None,
                keep_f32_from: int = -1) -> torch.Tensor:
        """z_tokens: [(T h w), 8] fp16 (channels >= z_channels zero).  Writes frames
        out[out_frame0 + skip_frames : out_frame0 + T] (NCHW fp32, (n,3,8h,8w)).  With ``out_u8`` ((F,8h,8w,3) uint8) the
        last kernel also stores the frames as the reference's output path does (ops.time_mix_small_u8) and keeps fp32 only
        for frames >= keep_f32_from of this call."""
        cfg = self.cfg
        if not hasattr(self, "gn_stats") or self.gn_stats.shape[1] < T:
            self._bufs.setdefault(("gn.retired",), []).append(getattr(self, "gn_stats", None))   # tapes may still point at it
            self.gn_stats = torch.zeros(self.n_gn, T, cfg.num_groups, 2, dtype=torch.float32, device=self.dev)
        if not hasattr(self, "gn_ws"):
            self.gn_ws = ops.GNWorkspace(self.dev)
        up_total = 2 ** (len(cfg.ch_mult) - 1)
        self.gn_ws.reserve(ops.groupnorm_scratch(T, h * w * up_total * up_total, cfg.num_groups))
        if self._arena_key != (T, h, w):
            plan = decoder_scratch_plan(cfg, T, h, w)
            if self._arena is None or self._arena.numel() < plan.total:
                # nothing captures the decoder's launches: the old arena can go back to the allocator (stream-ordered)
                self._arena = None
                self._arena = torch.empty(plan.total, dtype=torch.uint8, device=self.dev)
            self._arena_key, self._arena_roles = (T, h, w), plan.roles
        self._roles = self._arena_roles
        try:
            return self._forward(z_tokens, T, h, w, out, out_frame0, blend, skip_frames, out_u8, keep_f32_from)
        finally:
            self._roles = None

    def _forward(self, z_tokens, T, h, w, out, out_frame0, blend, skip_frames, out_u8, keep_f32_from):
        cfg = self.cfg
        M = T * h * w
        x = ops.conv3x3_small_cin(z_tokens, cfg.z_channels, self.conv_in_w, self.conv_in_b,
                                  self.buf("d.in", M, self.plan.block_in), T, h, w)
        x, xp = self._resblock(self.res[self.plan.mid[0].prefix], x, T, h, w, "d.r0")
        x, xp = self._attn(x, T, h, w, xp)
        x, xp = self._resblock(self.res[self.plan.mid[1].prefix], x, T, h, w, "d.r1", xp)
        for li, (blocks, up, ch) in enumerate(self.plan.levels):
            for bi, rb in enumerate(blocks):
                x, xp = self._resblock(self.res[rb.prefix], x, T, h, w, f"d.r{bi % 2}", xp)
            if up is not None:
                fuse = self._fuse_stats(T, 2 * h, 2 * w) and ops.upsample_stats_box(w, h) is not None
                xp = self.part("d.upc", T * 4 * h * w, ch) if fuse else None
                upc = self.buf("d.upc", T * 4 * h * w, ch)
                if self._upsample_in_gemm():    # nearest-2x upsample + 3x3 conv in one launch, reading x at low resolution
                    x = self.gemm(x, self.ups[up], upc, taps=ops.TAPS_3X3, geom=(w, h, T), upsample=True, stats=xp)
                else:
                    xu = ops.upsample2x(x, torch.empty(T * 4 * h * w, ch, dtype=x.dtype, device=self.dev), T, h, w, ch)
                    x = self.gemm(xu, self.ups[up], upc, taps=ops.TAPS_3X3, geom=(2 * w, 2 * h, T), stats=xp)
                h, w = 2 * h, 2 * w
        M = T * h * w
        a = self._gn(x, self.buf("d.a1", M, self.plan.final_ch), T, h * w, self.norm_out, 1e-6, self.norm_out_idx, part=xp)
        y = self.gemm(a, self.out_conv, self.buf("d.y", M, 8, torch.float32), taps=ops.TAPS_3X3, geom=(w, h, T))
        if out_u8 is not None:
            ops.time_mix_small_u8(y, self.tmix_w, self.tmix_b, out, out_u8, blend, T, h * w, cfg.out_ch, out_frame0,
                                  skip_frames, keep_f32_from)
        else:
            ops.time_mix_small(y, self.tmix_w, self.tmix_b, out, blend, T, h * w, cfg.out_ch, out_frame0, skip_frames)
        return out


def decode_first_stage(rt: DecoderRuntime, z: torch.Tensor, scale_factor: float = 0.18215, n_samples: Optional[int] = 14,
                       overlap: int = 3, u8: bool = False) -> torch.Tensor:
    """vwm/models/diffusion.py:150-180 on the B200 decoder.  z: (F,4,h,w) fp32 -> (F,3,8h,8w) fp32.
    ``u8``: return (F,8h,8w,3) uint8 instead — what do_sample's clamp((x+1)/2,0,1) (sample_utils.py:374) followed by
    perform_save_locally's (255*sample).astype(uint8) in "t h w c" order (sample_utils.py:96-126) makes of the same
    frames, written by the decoder's last kernel (SURVEY.md 8f rank 4: no fp32 frame tensor, 4x less D2H)."""
    F_, zc, h, w = z.shape
    n_samples = F_ if n_samples is None else n_samples
    up = 2 ** (len(rt.cfg.ch_mult) - 1)
    out = torch.empty(F_, rt.cfg.out_ch, h * up, w * up, dtype=torch.float32, device=z.device)
    zs = (z.float() / scale_factor).contiguous()
    if u8:
        out8 = torch.empty(F_, h * up, w * up, rt.cfg.out_ch, dtype=torch.uint8, device=z.device)
        chunks = _decode_chunks(F_, n_samples, overlap)
        for ci, (f0, n, o0, nov) in enumerate(chunks):
            # fp32 is kept only for the frames the NEXT chunk averages with (its first `nov` output frames)
            keep = n if ci + 1 == len(chunks) else max(0, chunks[ci + 1][2] - o0)
            decode_chunk_u8(rt, zs[f0:f0 + n], out, out8, o0, nov, keep)
        return out8

    def run(frames: torch.Tensor, out_frame0: int, n_overlap: int):
        T = frames.shape[0]
        tok = rt.buf("d.z", T * h * w, 8)
        tok.zero_()
        ops.nchw_to_tokens(frames.contiguous(), tok, T, zc, h, w)
        blend = None
        if n_overlap:
            blend = torch.zeros(T, dtype=torch.int32, device=z.device)
            blend[:n_overlap] = 1
        rt.forward(tok, T, h, w, out, out_frame0=out_frame0, blend=blend)

    for f0, n, o0, nov in _decode_chunks(F_, n_samples, overlap):
        run(zs[f0:f0 + n], o0, nov)
    return out


def decode_chunk_u8(rt: DecoderRuntime, zs: torch.Tensor, out: torch.Tensor, out8: torch.Tensor, out_frame0: int,
                    n_overlap: int, keep_f32_from: int) -> None:
    """One chunk of the uint8 decode.  zs: the chunk's (n,4,h,w) latents / scale_factor.  Writes out8[out_frame0 + t] for
    t < n; frames t < n_overlap are averaged with the fp32 frames out[out_frame0 + t] the previous chunk kept; the fp32 of
    frames t >= keep_f32_from is kept in out[out_frame0 + t] for the next chunk."""
    n, zc, h, w = zs.shape
    tok = rt.buf("d.z", n * h * w, 8)
    tok.zero_()
    ops.nchw_to_tokens(zs.contiguous(), tok, n, zc, h, w)
    blend = None
    if n_overlap:
        blend = torch.zeros(n, dtype=torch.int32, device=zs.device)
        blend[:n_overlap] = 1
    rt.forward(tok, n, h, w, out, out_frame0=out_frame0, blend=blend, out_u8=out8, keep_f32_from=keep_f32_from)


# ---------------------------------------------------------------------------------------------------------------
# VAE encoder (SURVEY.md §8f rank 1, the next row).  Host executor over the validated kernels (tap-GEMM, GroupNorm,
# GEMM-softmax-GEMM attention) plus one new gather (b200v_im2col_s2_asym).  Pinned by the oracle
# (tests/test_oracle_golden.py::test_encoder_matches_reference) and, on hardware, by tests/test_decoder_gpu.py against the
# real-reference fixtures (encode_first_stage rel-L2 ~1e-3).
# ---------------------------------------------------------------------------------------------------------------
class EncoderRuntime(DecoderRuntime):
    """``Encoder.forward`` (vwm/modules/diffusionmodules/model.py:527-557): conv_in, per level ResnetBlocks
    (model.py:116-135, temb = None) + Downsample (model.py:69-83), mid (res, attn, res), GN, swish, conv_out."""

    def __init__(self, cfg, sd: Dict[str, torch.Tensor], device, post=None):
        """post = (W [o, 2 z_channels], b [o]) fp32: a 1x1 convolution after conv_out (AutoencodingEngineLegacy.quant_conv,
        autoencoder.py:449-453,472), folded into conv_out's weights at packing time."""
        from .spec import build_encoder_plan
        self.cfg, self.dev = cfg, torch.device(device)
        self._post = post
        self.levels, self.mid_ch = build_encoder_plan(cfg)
        self._bufs = {}
        self._sd = sd
        self._pack()
        self._sd = None

    def _pack(self):
        self.n_gn = 0
        self.res = {}

        def pack_res(rb: DecResBlockSpec):
            p = rb.prefix
            self.res[p] = dict(spec=rb, gn1=self._norm(f"{p}.norm1"), conv1=self._lin(f"{p}.conv1"),
                               gn2=self._norm(f"{p}.norm2"), conv2=self._lin(f"{p}.conv2"),
                               skip=self._lin(f"{p}.nin_shortcut") if rb.has_skip else None, gn_idx=self.n_gn)
            self.n_gn += 2

        self.conv_in_w, self.conv_in_b = self._f32("conv_in.weight"), self._f32("conv_in.bias")
        self.downs = {}
        for blocks, down, ch in self.levels:
            for rb in blocks:
                pack_res(rb)
            if down is not None:
                self.downs[down] = self._lin(down)          # [C, 9 C] tap-major: K order of the im2col gather
        pack_res(DecResBlockSpec("mid.block_1", self.mid_ch, self.mid_ch))
        a, sd = "mid.attn_1", self._sd
        self.attn = dict(norm=self._norm(f"{a}.norm"), q=self._lin(f"{a}.q"), k=self._lin(f"{a}.k"),
                         v_w=conv_weight_to_taps(sd[f"{a}.v.weight"].detach().to(self.dev, torch.float32)).to(torch.float16).contiguous(),
                         v_b=self._f32(f"{a}.v.bias"), proj=self._lin(f"{a}.proj_out"), gn_idx=self.n_gn)
        self.n_gn += 1
        pack_res(DecResBlockSpec("mid.block_2", self.mid_ch, self.mid_ch))
        self.norm_out = self._norm("norm_out")
        self.norm_out_idx = self.n_gn
        self.n_gn += 1
        ow = conv_weight_to_taps(self._f32("conv_out.weight"))          # 2 z_channels = 8 output channels
        ob = self._f32("conv_out.bias")
        if getattr(self, "_post", None) is not None:                    # quant_conv o conv_out, composed in fp32
            pw, pb = (t.to(self.dev, torch.float32) for t in self._post)
            ow, ob = pw @ ow, pw @ ob + pb
        assert ow.shape[0] <= 8
        w8 = torch.zeros(8, ow.shape[1], dtype=torch.float16, device=self.dev)
        w8[: ow.shape[0]] = ow.to(torch.float16)
        b8 = torch.zeros(8, dtype=torch.float32, device=self.dev)
        b8[: ow.shape[0]] = ob
        self.out_conv = Lin(w8.contiguous(), b8, 32)
        self.n_moments = ow.shape[0]

    def _fuse_stats(self, n, h, w) -> bool:
        return False        # the encoder runs once per sample on one frame group: statistics keep their own pass

    def _enc_resblock(self, L, x, n, h, w, name):
        rb: DecResBlockSpec = L["spec"]
        hw, M, gi = h * w, n * h * w, L["gn_idx"]
        a1 = self._gn(x, self.buf("e.a1", M, rb.cin), n, hw, L["gn1"], 1e-6, gi)
        h1 = self.gemm(a1, L["conv1"], self.buf("e.h1", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, n))
        a2 = self._gn(h1, self.buf("e.a2", M, rb.cout), n, hw, L["gn2"], 1e-6, gi + 1)
        xs = x if L["skip"] is None else self.gemm(x, L["skip"], self.buf("e.xs", M, rb.cout))
        return self.gemm(a2, L["conv2"], self.buf(name, M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, n), res1=xs)

    def forward(self, x_tokens: torch.Tensor, n: int, h: int, w: int) -> torch.Tensor:
        """x_tokens: [(n h w), 8] fp16 image rows (channels >= in_channels zero) -> moments [(n h/8 w/8), 8] fp32
        (mean | logvar columns)."""
        cfg = self.cfg
        if not hasattr(self, "gn_stats") or self.gn_stats.shape[1] < n:
            self._bufs.setdefault(("gn.retired",), []).append(getattr(self, "gn_stats", None))
            self.gn_stats = torch.zeros(self.n_gn, n, cfg.num_groups, 2, dtype=torch.float32, device=self.dev)
        if not hasattr(self, "gn_ws"):
            self.gn_ws = ops.GNWorkspace(self.dev)
        self.gn_ws.reserve(ops.groupnorm_scratch(n, h * w, cfg.num_groups))
        x = ops.conv3x3_small_cin(x_tokens, cfg.in_channels, self.conv_in_w, self.conv_in_b,
                                  self.buf("e.in", n * h * w, cfg.ch), n, h, w)
        for blocks, down, ch in self.levels:
            for bi, rb in enumerate(blocks):
                x = self._enc_resblock(self.res[rb.prefix], x, n, h, w, f"e.r{bi % 2}")
            if down is not None:
                ho, wo = (h - 2) // 2 + 1, (w - 2) // 2 + 1
                col = ops.im2col_s2_asym(x, self.buf("e.col", n * ho * wo, 9 * ch), n, h, w, ch)
                h, w = ho, wo
                x = self.gemm(col, self.downs[down], self.buf("e.down", n * h * w, ch))
        x = self._enc_resblock(self.res["mid.block_1"], x, n, h, w, "e.m0")
        x, _ = self._attn(x, n, h, w)
        x = self._enc_resblock(self.res["mid.block_2"], x, n, h, w, "e.m1")
        M = n * h * w
        a = ops.groupnorm(x, self.buf("e.a1", M, self.mid_ch), n, h * w, self.norm_out[0], self.norm_out[1], 1e-6,
                          True, self.gn_stats[self.norm_out_idx, :n], groups=cfg.num_groups, ws=self.gn_ws)
        return self.gemm(a, self.out_conv, self.buf("e.y", M, 8, torch.float32), taps=ops.TAPS_3X3, geom=(w, h, n))


def encode_first_stage(rt: EncoderRuntime, x: torch.Tensor, scale_factor: float = 0.18215,
                       n_samples: Optional[int] = None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """DiffusionEngine.encode_first_stage (vwm/models/diffusion.py:183-195) over AutoencodingEngine.encode with the
    DiagonalGaussianRegularizer (autoencoder.py:190-203, regularizers/__init__.py:30-40, distributions.py:25-36):
    x (n,3,H,W) fp32 -> z (n,4,H/8,W/8) fp32 = (mean + exp(0.5 clamp(logvar,-30,20)) * noise) * scale_factor; the
    reference draws `noise` from the device RNG — pass it in for reproducible parity, None gives the mode."""
    n_all, cin, H, W = x.shape
    n_samples = n_all if n_samples is None else n_samples
    down = 2 ** (len(rt.cfg.ch_mult) - 1)
    zc = rt.cfg.z_channels
    out = torch.empty(n_all, zc, H // down, W // down, dtype=torch.float32, device=x.device)
    for i in range(0, n_all, n_samples):
        xs = x[i:i + n_samples].float().contiguous()
        n = xs.shape[0]
        tok = rt.buf("e.x", n * H * W, 8)
        tok.zero_()
        ops.nchw_to_tokens(xs, tok, n, cin, H, W)
        mom_tok = rt.forward(tok, n, H, W)
        mom = torch.empty(n, 8, H // down, W // down, dtype=torch.float32, device=x.device)
        ops.tokens_to_nchw(mom_tok, mom, n, 8, H // down, W // down)
        mean, logvar = mom[:, :zc], mom[:, zc:2 * zc]
        z = mean if noise is None else mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise[i:i + n].to(mean)
        out[i:i + n] = z * scale_factor
    return out


class Encoder(nn.Module):
    """``encoder_config.target`` stand-in for vwm.modules.diffusionmodules.model.Encoder: same keywords, same
    ``state_dict`` keys, ``forward(x)`` -> (n, 2 z_channels, H/8, W/8) moments."""

    def __init__(self, *, ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions=(), dropout=0.0, resamp_with_conv=True,
                 in_channels=3, resolution=256, z_channels=4, double_z=True, use_linear_attn=False, attn_type="vanilla",
                 **ignore_kwargs):
        super().__init__()
        from .spec import EncoderConfig, encoder_param_specs
        bad = [k for k, v in dict(attn_resolutions=len(list(attn_resolutions)) != 0, dropout=dropout != 0.0,
                                  resamp_with_conv=not resamp_with_conv, use_linear_attn=use_linear_attn,
                                  attn_type=attn_type != "vanilla", double_z=not double_z).items() if v]
        if bad:
            raise NotImplementedError(f"vista_b200.Encoder: unsupported option(s) {bad}")
        self.b200_config = EncoderConfig(ch=ch, in_channels=in_channels, ch_mult=tuple(ch_mult),
                                         num_res_blocks=num_res_blocks, z_channels=z_channels, double_z=double_z)
        register_param_tree(self, encoder_param_specs(self.b200_config))
        self._runtime = None
        self.register_load_state_dict_post_hook(lambda module, keys: setattr(module, "_runtime", None))

    def _apply(self, fn, *args, **kwargs):     # keep the packed runtime unless a parameter moved / changed dtype
        before = tuple((p.device, p.dtype) for p in self.parameters())
        out = super()._apply(fn, *args, **kwargs)
        if tuple((p.device, p.dtype) for p in self.parameters()) != before:
            self._runtime = None
        return out

    def runtime(self, device) -> EncoderRuntime:
        if torch.device(device).type != "cuda":
            raise RuntimeError("vista_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self._runtime is None:
            self._runtime = EncoderRuntime(self.b200_config, self.state_dict(), device)
        return self._runtime

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        rt = self.runtime(x.device)
        n, cin, H, W = x.shape
        down = 2 ** (len(rt.cfg.ch_mult) - 1)
        tok = rt.buf("e.x", n * H * W, 8)
        tok.zero_()
        ops.nchw_to_tokens(x.float().contiguous(), tok, n, cin, H, W)
        mom_tok = rt.forward(tok, n, H, W)
        mom = torch.empty(n, 8, H // down, W // down, dtype=torch.float32, device=x.device)
        ops.tokens_to_nchw(mom_tok, mom, n, 8, H // down, W // down)
        return mom[:, : rt.n_moments]


def _decode_chunks(F_: int, n_samples: int, overlap: int):
    """Chunk plan of decode_first_stage (vwm/models/diffusion.py:150-180): (first input frame, frame count,
    first output frame, overlapping frames that are averaged with the previous chunk's output)."""
    chunks = []
    if overlap == 0 and n_samples < F_:
        # previous_z = current_z[-0:] is the WHOLE previous chunk in the reference (diffusion.py:178): not a usable mode
        raise NotImplementedError("decode_first_stage: overlap = 0 with more than one chunk is ill-defined in the reference")
    if overlap < n_samples:
        pos, first, prev_len = overlap, True, overlap
        while pos < F_:
            cur = min(n_samples - overlap, F_ - pos)
            # context = the last prev_len frames before pos (prev = cur[-overlap:] of the previous chunk) + cur
            chunks.append((pos - prev_len, prev_len + cur, pos - overlap, 0 if first else overlap))
            pos += cur
            prev_len = min(overlap, cur)
            first = False
    else:
        pos = 0
        while pos < F_:
            cur = min(n_samples, F_ - pos)
            chunks.append((pos, cur, pos, 0))
            pos += cur
    return chunks


def decode_first_stage_parallel(rt: DecoderRuntime, z: torch.Tensor, scale_factor: float = 0.18215,
                                n_samples: Optional[int] = 14, overlap: int = 3, group=None) -> torch.Tensor:
    """decode_first_stage with the chunks dealt out over the ranks of `group`: the chunks are independent up to the
    overlap rule (out = (previous + new) / 2 on the first `overlap` frames of a chunk), so rank r decodes chunks
    r, r + W, ... unblended, the owners broadcast them, and every rank assembles the clip in chunk order with the
    same arithmetic as the serial path (bit-identical result on every rank).  Every rank passes the same z."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    F_, zc, h, w = z.shape
    n_samples = F_ if n_samples is None else n_samples
    up = 2 ** (len(rt.cfg.ch_mult) - 1)
    out = torch.empty(F_, rt.cfg.out_ch, h * up, w * up, dtype=torch.float32, device=z.device)
    zs = (z.float() / scale_factor).contiguous()
    chunks = _decode_chunks(F_, n_samples, overlap)
    if any(nov > n or o0 != f0 for f0, n, o0, nov in chunks):
        raise NotImplementedError("decode_first_stage_parallel: chunks shorter than the overlap")
    to_global = (lambda r: r) if group is None else (lambda r: dist.get_global_rank(group, r))
    bufs = []
    for i, (f0, n, o0, nov) in enumerate(chunks):
        cb = rt.__dict__.setdefault("_chunk_out", {}).get((i, n))
        if cb is None:
            cb = rt._chunk_out[(i, n)] = torch.empty(n, rt.cfg.out_ch, h * up, w * up, dtype=torch.float32, device=z.device)
        bufs.append(cb)
        if i % world == rank:
            tok = rt.buf("d.z", n * h * w, 8)
            tok.zero_()
            ops.nchw_to_tokens(zs[f0:f0 + n].contiguous(), tok, n, zc, h, w)
            rt.forward(tok, n, h, w, cb)
    for i, (f0, n, o0, nov) in enumerate(chunks):
        if world > 1:
            dist.broadcast(bufs[i], src=to_global(i % world), group=group)
        if nov:
            out[o0:o0 + nov] = 0.5 * (out[o0:o0 + nov] + bufs[i][:nov])
        out[o0 + nov:o0 + n] = bufs[i][nov:]
    return out


class VideoDecoder(nn.Module):
    """``decoder_config.target`` stand-in for vwm.modules.autoencoding.temporal_ae.VideoDecoder: same keywords,
    same ``state_dict`` keys, ``forward(z, timesteps=...)`` -> (n,3,8h,8w)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions=(), dropout=0.0,
                 resamp_with_conv=True, in_channels=3, resolution=256, z_channels=4, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", video_kernel_size=3, alpha: float = 0.0,
                 merge_strategy: str = "learned", time_mode: str = "conv-only", **ignorekwargs):
        super().__init__()
        vks = [3, 1, 1] if video_kernel_size is None else video_kernel_size
        bad = [n for n, v in dict(attn_resolutions=len(list(attn_resolutions)) != 0, dropout=dropout != 0.0,
                                  resamp_with_conv=not resamp_with_conv, give_pre_end=give_pre_end, tanh_out=tanh_out,
                                  use_linear_attn=use_linear_attn, attn_type=attn_type != "vanilla",
                                  video_kernel_size=isinstance(vks, int) or list(vks) != [3, 1, 1],
                                  merge_strategy=merge_strategy != "learned", time_mode=time_mode != "conv-only").items() if v]
        if bad:
            raise NotImplementedError(f"vista_b200.VideoDecoder: unsupported option(s) {bad}")
        self.b200_config = DecoderConfig(ch=ch, out_ch=out_ch, ch_mult=tuple(ch_mult), num_res_blocks=num_res_blocks,
                                         z_channels=z_channels)
        register_param_tree(self, decoder_param_specs(self.b200_config))
        self._runtime = None
        self.register_load_state_dict_post_hook(lambda module, keys: setattr(module, "_runtime", None))

    def _apply(self, fn, *args, **kwargs):     # keep the packed runtime unless a parameter moved / changed dtype
        before = tuple((p.device, p.dtype) for p in self.parameters())
        out = super()._apply(fn, *args, **kwargs)
        if tuple((p.device, p.dtype) for p in self.parameters()) != before:
            self._runtime = None
        return out

    def runtime(self, device) -> DecoderRuntime:
        if torch.device(device).type != "cuda":
            raise RuntimeError("vista_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self._runtime is None:
            self._runtime = DecoderRuntime(self.b200_config, self.state_dict(), device)
        return self._runtime

    def forward(self, z: torch.Tensor, timesteps: Optional[int] = None, **kwargs) -> torch.Tensor:
        rt = self.runtime(z.device)
        T, zc, h, w = z.shape
        assert timesteps in (None, T), "one clip per call (decode_first_stage passes timesteps == batch)"
        up = 2 ** (len(rt.cfg.ch_mult) - 1)
        out = torch.empty(T, rt.cfg.out_ch, h * up, w * up, dtype=torch.float32, device=z.device)
        tok = rt.buf("d.z", T * h * w, 8)
        tok.zero_()
        ops.nchw_to_tokens(z.float().contiguous(), tok, T, zc, h, w)
        return rt.forward(tok, T, h, w, out)

    def get_last_layer(self, skip_time_mix=False, **kwargs):
        return self.conv_out.time_mix_conv.weight if not skip_time_mix else self.conv_out.weight
