"""B200 executor of the Vista ``VideoUNet`` forward (vwm/modules/diffusionmodules/video_model.py:442-503).

Python only orchestrates: it owns device buffers (torch tensors), repacks the reference weights
once, and issues C-ABI calls (vista_b200/ops.py) — every FLOP of the forward runs in the
hand-written kernels.  Design points (DESIGN.md has the full list):

  * activations are token-major fp16 ``[(b t) h w, C]`` everywhere; the reference's NCHW <-> token
    ``rearrange``/``contiguous`` copies (video_attention.py:116,140,266,292) do not exist;
  * skip connections are never concatenated: the producer of a skip tensor writes straight into
    the channel slice of its consumer's input buffer (``torch.cat`` at video_model.py:493);
  * every conv / linear is one tap-GEMM launch with bias, time-embedding row vector, residual(s),
    AlphaBlender mix and GEGLU fused in the epilogue;
  * both cross-attentions (attn2) have ONE key (encoders/modules.py:514-516, video_attention.py:256),
    so softmax == 1 and attn2(x) == to_out(to_v(ctx) + v_adapter(ctx_action)) — a per-frame constant
    computed once per sample in ``set_conditioning`` and added as a row vector in the epilogue of the
    preceding projection (SURVEY.md §0, verified bit-exact there);
  * all 44 ``emb_layers`` projections of a step are one batched GEMM.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .spec import ConvSpec, ResBlockSpec, SVTSpec, UNetConfig, build_unet_plan
from .weights import conv_weight_to_taps, permute_geglu


@dataclass
class Lin:
    w: torch.Tensor                   # fp16 [N, K]
    b: Optional[torch.Tensor]         # fp32 [N]
    tile_n: int
    geglu: bool = False


IN_PAD = 64   # token rows of the network input: 8 channels used, zero padded to one 64-channel K chunk


def padded_input_rows(rows: int, device) -> torch.Tensor:
    """[rows, 8] fp16 view (row stride IN_PAD) of a zeroed buffer: what UNetRuntime.forward wants as x_tokens so
    that the input convolution is a tap-GEMM; the pad columns must stay zero."""
    return torch.zeros(rows, IN_PAD, dtype=torch.float16, device=device)[:, :8]


class UNetRuntime:
    """Device-resident, repacked VideoUNet.  One instance per (weights, num_frames)."""
    has_collectives = False       # a step is a fixed sequence of local launches: CUDA-graph capturable

    def __init__(self, cfg: UNetConfig, sd: Dict[str, torch.Tensor], device, num_frames: int = 25):
        self.cfg, self.dev, self.T = cfg, torch.device(device), num_frames
        self.plan = build_unet_plan(cfg)
        self._bufs: Dict[Tuple, torch.Tensor] = {}
        self._sd = sd
        self._pack()
        self._sd = None
        self.cond = None
        self.conds: Dict[int, dict] = {}      # batch size -> its conditioning; forward(B rows) uses conds[B]
        # (B, h, w) -> per output block, whether the last full forward left GroupNorm partials of its input's h half
        self._h_filled: Dict[Tuple[int, int, int], List[bool]] = {}

    # ------------------------------------------------------------------ weight packing
    def _f32(self, name):
        return self._sd[name].detach().to(self.dev, torch.float32).contiguous()

    def _lin(self, prefix, geglu=False, bias=True, tile_n=None) -> Lin:
        w = self._sd[f"{prefix}.weight"].detach().to(self.dev, torch.float32)
        b = self._f32(f"{prefix}.bias") if bias and f"{prefix}.bias" in self._sd else None
        if w.dim() > 2:
            w = conv_weight_to_taps(w)
        tn = tile_n or ops.pick_tile_n(w.shape[0], geglu)
        if geglu:
            w, b = permute_geglu(w, b, tn)
        return Lin(w.to(torch.float16).contiguous(), b, tn, geglu)

    def _norm(self, prefix):
        return self._f32(f"{prefix}.weight"), self._f32(f"{prefix}.bias")

    def _attn2_weights(self, p):
        return dict(v=self._lin(f"{p}.to_v", bias=False),
                    va=self._lin(f"{p}.v_adapter_action_control", bias=False) if f"{p}.v_adapter_action_control.weight" in self._sd else None,
                    out=self._lin(f"{p}.to_out.0"))

    def _pack(self):
        cfg, sd = self.cfg, self._sd
        self.time_embed = (self._lin("time_embed.0"), self._lin("time_embed.2"))
        self.cond_embed = (self._lin("cond_time_stack_embed.0"), self._lin("cond_time_stack_embed.2"))
        self.label_emb = (self._lin("label_emb.0.0"), self._lin("label_emb.0.2"))
        self.layers: Dict[str, dict] = {}
        emb_w, emb_b, off = [], [], 0
        self.n_gn = 0
        for layer in self.plan.all_layers():
            if isinstance(layer, ResBlockSpec):
                p = layer.prefix
                L = dict(spec=layer, gn1=self._norm(f"{p}.in_layers.0"), conv1=self._lin(f"{p}.in_layers.2"),
                         gn2=self._norm(f"{p}.out_layers.0"), conv2=self._lin(f"{p}.out_layers.3"),
                         skip=self._lin(f"{p}.skip_connection") if layer.has_skip else None,
                         tgn1=self._norm(f"{p}.time_stack.in_layers.0"), tconv1=self._lin(f"{p}.time_stack.in_layers.2"),
                         tgn2=self._norm(f"{p}.time_stack.out_layers.0"), tconv2=self._lin(f"{p}.time_stack.out_layers.3"),
                         alpha=float(torch.sigmoid(sd[f"{p}.time_mixer.mix_factor"].float()).item()),
                         gn_idx=self.n_gn)
                self.n_gn += 4
                for key, q in (("emb_off", f"{p}.emb_layers.1"), ("embt_off", f"{p}.time_stack.emb_layers.1")):
                    L[key] = off
                    emb_w.append(sd[f"{q}.weight"].detach().to(self.dev, torch.float32))
                    emb_b.append(sd[f"{q}.bias"].detach().to(self.dev, torch.float32))
                    off += layer.cout
                self.layers[p] = L
            elif isinstance(layer, SVTSpec):
                p, s, m = layer.prefix, f"{layer.prefix}.transformer_blocks.0", f"{layer.prefix}.time_stack.0"

                def qkv(a):
                    w = torch.cat([sd[f"{a}.to_q.weight"], sd[f"{a}.to_k.weight"], sd[f"{a}.to_v.weight"]], 0)
                    w = w.detach().to(self.dev, torch.float16).contiguous()
                    return Lin(w, None, ops.pick_tile_n(w.shape[0]))

                L = dict(spec=layer, norm=self._norm(f"{p}.norm"), proj_in=self._lin(f"{p}.proj_in"),
                         ln1=self._norm(f"{s}.norm1"), qkv=qkv(f"{s}.attn1"), out=self._lin(f"{s}.attn1.to_out.0"),
                         attn2=self._attn2_weights(f"{s}.attn2"),
                         ln3=self._norm(f"{s}.norm3"), ff1=self._lin(f"{s}.ff.net.0.proj", geglu=True), ff2=self._lin(f"{s}.ff.net.2"),
                         ln_in=self._norm(f"{m}.norm_in"), ffin1=self._lin(f"{m}.ff_in.net.0.proj", geglu=True),
                         ffin2=self._lin(f"{m}.ff_in.net.2"),
                         tln1=self._norm(f"{m}.norm1"), tqkv=qkv(f"{m}.attn1"), tout=self._lin(f"{m}.attn1.to_out.0"),
                         tattn2=self._attn2_weights(f"{m}.attn2"),
                         tln3=self._norm(f"{m}.norm3"), tff1=self._lin(f"{m}.ff.net.0.proj", geglu=True), tff2=self._lin(f"{m}.ff.net.2"),
                         pos=(self._lin(f"{p}.time_pos_embed.0"), self._lin(f"{p}.time_pos_embed.2")),
                         alpha=float(torch.sigmoid(sd[f"{p}.time_mixer.mix_factor"].float()).item()),
                         proj_out=self._lin(f"{p}.proj_out"), gn_idx=self.n_gn)
                self.n_gn += 1
                self.layers[p] = L
            elif isinstance(layer, ConvSpec):
                if layer.kind == "conv_in":
                    # two forms: fp32 [Cout, Cin, 3, 3] for the thin direct kernel (8-wide token rows), and a tap-GEMM
                    # weight with Cin zero-padded to 64 for callers that hand in IN_PAD-wide, zero-padded rows
                    w = self._f32(f"{layer.prefix}.weight")
                    wp = torch.zeros(w.shape[0], IN_PAD, 3, 3, dtype=torch.float32, device=self.dev)
                    wp[:, :w.shape[1]] = w
                    b = self._f32(f"{layer.prefix}.bias")
                    self.layers[layer.prefix] = dict(spec=layer, w=w, b=b,
                                                     conv=Lin(conv_weight_to_taps(wp).to(torch.float16).contiguous(), b,
                                                              ops.pick_tile_n(w.shape[0])))
                else:
                    self.layers[layer.prefix] = dict(spec=layer, conv=self._lin(layer.prefix))
        self.emb_all = Lin(torch.cat(emb_w, 0).to(torch.float16).contiguous(), torch.cat(emb_b, 0).contiguous(),
                           ops.pick_tile_n(off))
        self.emb_total = off
        self.out_norm = self._norm("out.0")
        self.out_gn_idx = self.n_gn
        self.n_gn += 1
        # out[2]: conv3x3 320 -> 4 as a tap-GEMM with N padded to 8 (fp32 output, 4 channels used)
        ow = conv_weight_to_taps(self._f32("out.2.weight"))
        oc = ow.shape[0]
        assert oc <= 8
        w8 = torch.zeros(8, ow.shape[1], dtype=torch.float16, device=self.dev)
        w8[:oc] = ow.to(torch.float16)
        b8 = torch.zeros(8, dtype=torch.float32, device=self.dev)
        b8[:oc] = self._f32("out.2.bias")
        self.out_conv = Lin(w8.contiguous(), b8, 32)

    # ------------------------------------------------------------------ buffers
    def buf(self, name: str, rows: int, cols: int, dtype=torch.float16) -> torch.Tensor:
        key = (name, rows, cols, dtype)
        t = self._bufs.get(key)
        if t is None:
            t = torch.empty(rows, cols, dtype=dtype, device=self.dev)
            self._bufs[key] = t
        return t

    def gemm(self, a, lin: Lin, out, **kw):
        return ops.gemm(a, lin.w, out, bias=lin.b, tile_n=lin.tile_n, act=2 if lin.geglu else kw.pop("act", 0), **kw)

    def _gn(self, x, y, B, hw, norm, eps, silu, idx, fps=1, part=None):
        """GroupNorm32 (+ SiLU).  ``part``: column partials of x written by its producing GEMM(s) — the statistics then
        cost one small reduction instead of a pass over x (util.py:214-216 reads x three times in the reference)."""
        if fps != 1:
            return self._gn_temporal(x, y, B, hw, norm, eps, silu, idx, fps, part)
        stats = self.gn_stats[idx, : B // fps]
        if part is None:
            return ops.groupnorm(x, y, B, hw, norm[0], norm[1], eps, silu, stats, frames_per_stat=fps,
                                 groups=self.cfg.num_groups, ws=self.gn_ws)
        ops.groupnorm_from_partials(part, B, hw, norm[0].numel(), eps, stats, fps, self.cfg.num_groups)
        return ops.groupnorm_apply(x, y, B, hw, norm[0], norm[1], silu, stats, fps, self.cfg.num_groups)

    def _gn_temporal(self, x, y, B, hw, norm, eps, silu, idx, fps, part=None):
        """GroupNorm whose statistic spans the frames of a clip (video_model.py:67-72)."""
        stats = self.gn_stats[idx, : B // fps]
        if part is None:
            return ops.groupnorm(x, y, B, hw, norm[0], norm[1], eps, silu, stats, frames_per_stat=fps,
                                 groups=self.cfg.num_groups, ws=self.gn_ws)
        ops.groupnorm_from_partials(part, B, hw, norm[0].numel(), eps, stats, fps, self.cfg.num_groups)
        return ops.groupnorm_apply(x, y, B, hw, norm[0], norm[1], silu, stats, fps, self.cfg.num_groups)

    def part(self, name: str, tokens: int, cols: int) -> torch.Tensor:
        """Persistent [tokens/128*4, cols, 2] fp32 matrix of GroupNorm column partials (ops.gemm(stats=...))."""
        key = ("part." + name, tokens, cols)
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = torch.zeros(-(-tokens // 128) * 4, cols, 2, dtype=torch.float32, device=self.dev)
        return t

    def _ln(self, x, y, norm, **kw):
        return ops.layernorm(x, y, norm[0], norm[1], 1e-5, **kw)

    # ------------------------------------------------------------------ per-sample constants
    def _mlp(self, x16, l0: Lin, l2: Lin, name: str) -> torch.Tensor:
        rows = x16.shape[0]
        hmid = self.buf(f"{name}.mid", rows, l0.w.shape[0])
        self.gemm(x16, l0, hmid, act=1)
        out = self.buf(f"{name}.out", rows, l2.w.shape[0], torch.float32)
        self.gemm(hmid, l2, out)
        return out

    def _attn2_const(self, W: dict, ctx16: torch.Tensor, name: str) -> torch.Tensor:
        """to_out(to_v(ctx[:, :D]) + v_adapter(ctx[:, D:])) for a single-token context (attention.py:342-353,421)."""
        rows, D = ctx16.shape[0], self.cfg.context_dim
        Cc = W["v"].w.shape[0]
        v = self.buf("a2.v", rows, Cc)
        self.gemm(ctx16[:, :D], W["v"], v)
        if W["va"] is not None:
            v2 = self.buf("a2.v2", rows, Cc)
            self.gemm(ctx16[:, D:], W["va"], v2, res1=v)
            v = v2
        out = self.buf(name, rows, Cc, torch.float32)   # persistent: captured CUDA graphs read it
        self.gemm(v, W["out"], out)
        return out

    def set_conditioning(self, context: torch.Tensor, y: torch.Tensor, slot: str = ""):
        """context (B,1,3456) / y (B,768): everything that does not depend on sigma or the step.  One conditioning is
        kept per batch size B (its constants are buffers of B rows), so that the CFG pair's 2T rows and action guidance's
        T image rows are conditioned side by side; setting B again replaces only B's.  A named ``slot`` keeps one more
        conditioning of B rows in buffers of its own, which ``forward(..., slot=slot)`` reads: the unguided steps of
        interval guidance condition their T rows on the full ``c`` beside action guidance's action-free T rows."""
        T = self.T
        B = context.shape[0]
        p = f"{slot}." if slot else ""
        # both cross-attentions are folded to per-frame constants, which is exact for ONE key token only
        # (encoders/modules.py:514-516, video_attention.py:256-257): refuse anything else instead of using token 0
        from .spec import ACTION_DIM
        want = self.cfg.context_dim + (ACTION_DIM if self.cfg.action_control else 0)
        if context.dim() != 3 or context.shape[1] != 1 or context.shape[2] != want:
            raise NotImplementedError(f"vista_b200: crossattn context must be (B, 1, {want}); got {tuple(context.shape)}")
        ctx16 = self.buf("cond.ctx", B, context.numel() // B)
        ctx16.copy_(context.reshape(B, -1))
        y16 = self.buf("cond.y", B, y.shape[-1])
        y16.copy_(y)
        cond = dict(B=B, label=self._mlp(y16, *self.label_emb, p + "label"), sp={}, tm={}, pos={})
        tctx16 = self.buf("cond.tctx", B // T, ctx16.shape[1])
        tctx16.copy_(ctx16[::T])                                   # video_attention.py:256
        frames = torch.arange(T, dtype=torch.float32, device=self.dev)
        for t in self.plan.transformers():
            L = self.layers[t.prefix]
            cond["sp"][t.prefix] = self._attn2_const(L["attn2"], ctx16, f"{p}cond.sp.{t.prefix}")
            cond["tm"][t.prefix] = self._attn2_const(L["tattn2"], tctx16, f"{p}cond.tm.{t.prefix}")
            temb = self.buf("cond.temb", T, t.ch)
            ops.timestep_embedding(frames, temb, t.ch)
            cond["pos"][t.prefix] = self._mlp(temb, *L["pos"], f"{p}cond.pos.{t.prefix}")
        self.cond = self.conds[(B, slot) if slot else B] = cond

    # ------------------------------------------------------------------ layers
    def _fuse_stats(self, B, h, w) -> bool:
        """GroupNorm statistics come out of the producing GEMM's epilogue where the token tiles are runs of 128 consecutive
        tokens (ops.stats_box): 72 x 128 and 36 x 64 of the BASELINE shape, every level of the decoder."""
        return ops.stats_box(w, h, B) is not None

    def _resblock(self, L, x, dst, B, h, w, xp=None, dp=None):
        """xp: column partials of x (None: the statistics of x take their own pass); dp: where to put those of dst."""
        rb: ResBlockSpec = L["spec"]
        T, hw, M, nb = self.T, h * w, B * h * w, B // self.T
        gi = L["gn_idx"]
        fuse = self._fuse_stats(B, h, w)
        p1 = self.part("rb.h1", M, rb.cout) if fuse else None
        p2 = self.part("rb.xsp", M, rb.cout) if fuse else None
        a1 = self._gn(x, self.buf("rb.a1", M, rb.cin), B, hw, L["gn1"], 1e-5, True, gi, part=xp)
        h1 = self.gemm(a1, L["conv1"], self.buf("rb.h1", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, B),
                       rowvec=self.emb_out[:, L["emb_off"]:L["emb_off"] + rb.cout], rv_div=hw, rv_mod=B, stats=p1)
        a2 = self._gn(h1, self.buf("rb.a2", M, rb.cout), B, hw, L["gn2"], 1e-5, True, gi + 1, part=p1)
        xs = x if L["skip"] is None else self.gemm(x, L["skip"], self.buf("rb.xs", M, rb.cout))
        xsp = self.gemm(a2, L["conv2"], self.buf("rb.xsp", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, B), res1=xs,
                        stats=p2)
        # temporal ResBlock: GroupNorm over (C/32, T, H, W), (3,1,1) conv over frames, AlphaBlender
        a3 = self._gn(xsp, self.buf("rb.a1", M, rb.cout), B, hw, L["tgn1"], 1e-5, True, gi + 2, fps=T, part=p2)
        h2 = self._tconv(a3, L["tconv1"], self.buf("rb.h1", M, rb.cout), hw, nb,
                         rowvec=self.emb_out[:, L["embt_off"]:L["embt_off"] + rb.cout], rv_div=hw, rv_mod=B, stats=p1)
        a4 = self._gn(h2, self.buf("rb.a2", M, rb.cout), B, hw, L["tgn2"], 1e-5, True, gi + 3, fps=T, part=p1)
        # out = alpha*xsp + (1-alpha)*(xsp + conv) = xsp + (1-alpha)*(conv + bias)      (util.py:317)
        self._tconv(a4, L["tconv2"], dst, hw, nb, s_acc=1.0 - L["alpha"], res1=xsp, stats=dp if fuse else None)
        return dst

    def _tconv(self, a, lin: Lin, out, hw: int, nb: int, **epi):
        """(3,1,1) convolution over the frames of each clip (zero padded at the clip ends)."""
        return self.gemm(a, lin, out, taps=ops.TAPS_T3, geom=(hw, self.T, nb), **epi)

    def _svt_tqkv(self, n, L, M: int, Cc: int, nb: int, hw: int):
        """Fused q|k|v projection of the temporal attention (a hook: the frame-sharded runtime splits it)."""
        return self.gemm(n, L["tqkv"], self.buf("tr.qkv", M, 3 * Cc))

    def _attn_temporal(self, qkv, o, nb: int, hw: int, heads: int, Cc: int):
        return ops.attention_temporal(qkv[:, :Cc], qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:], o, nb, self.T, hw, heads)

    def _svt(self, L, x, dst, B, h, w, xp=None, dp=None):
        t: SVTSpec = L["spec"]
        T, hw, M, nb, Cc = self.T, h * w, B * h * w, B // self.T, t.ch
        p = t.prefix
        al = L["alpha"]
        xn = self._gn(x, self.buf("tr.n", M, Cc), B, hw, L["norm"], 1e-6, False, L["gn_idx"], part=xp)
        t0 = self.gemm(xn, L["proj_in"], self.buf("tr.t0", M, Cc))
        # spatial block: self-attn, (constant) cross-attn, GEGLU FF           (attention.py:514-524)
        n = self._ln(t0, self.buf("tr.n", M, Cc), L["ln1"])
        qkv = self.gemm(n, L["qkv"], self.buf("tr.qkv", M, 3 * Cc))
        o = self.buf("tr.o", M, Cc)
        ops.attention_spatial(qkv[:, :Cc], qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:], o, B, hw, t.heads)
        t1 = self.gemm(o, L["out"], self.buf("tr.t1", M, Cc), res1=t0, rowvec=self.cond["sp"][p], rv_div=hw, rv_mod=B)
        n = self._ln(t1, self.buf("tr.n", M, Cc), L["ln3"])
        g = self.gemm(n, L["ff1"], self.buf("tr.g", M, 4 * Cc))
        t2 = self.gemm(g, L["ff2"], self.buf("tr.t2", M, Cc), res1=t1)
        # temporal block on x_mix = t2 + pos_emb[frame]                        (video_attention.py:284-288,111-141)
        pos = self.cond["pos"][p]
        n = self._ln(t2, self.buf("tr.n", M, Cc), L["ln_in"], addvec=pos, av_div=hw, av_mod=T)
        g = self.gemm(n, L["ffin1"], self.buf("tr.g", M, 4 * Cc))
        u1 = self.gemm(g, L["ffin2"], self.buf("tr.u1", M, Cc), res1=t2, rowvec=pos, rv_div=hw, rv_mod=T)
        n = self._ln(u1, self.buf("tr.n", M, Cc), L["tln1"])
        qkv = self._svt_tqkv(n, L, M, Cc, nb, hw)
        self._attn_temporal(qkv, o, nb, hw, t.heads, Cc)
        u2 = self.gemm(o, L["tout"], self.buf("tr.t1", M, Cc), res1=u1, rowvec=self.cond["tm"][p], rv_div=T * hw, rv_mod=nb)
        n = self._ln(u2, self.buf("tr.n", M, Cc), L["tln3"])
        g = self.gemm(n, L["tff1"], self.buf("tr.g", M, 4 * Cc))
        # x = alpha*t2 + (1-alpha)*(ff(...) + u2)                               (util.py:317)
        x3 = self.gemm(g, L["tff2"], self.buf("tr.u1", M, Cc), s_acc=1.0 - al, res1=u2, s_res1=1.0 - al, res2=t2, s_res2=al)
        self.gemm(x3, L["proj_out"], dst, res1=x, stats=dp if self._fuse_stats(B, h, w) else None)
        return dst

    def _down(self, L, x, dst, B, h, w, dp=None):
        c: ConvSpec = L["spec"]
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        col = self.buf("down.col", B * ho * wo, 9 * c.cin)
        ops.im2col_s2(x, col, B, h, w, c.cin)
        self.gemm(col, L["conv"], dst, stats=dp if self._fuse_stats(B, ho, wo) else None)
        return dst

    def _up(self, L, x, dst, B, h, w, dp=None):
        c: ConvSpec = L["spec"]
        up = self.buf("up.x", B * 4 * h * w, c.cin)
        ops.upsample2x(x, up, B, h, w, c.cin)
        self.gemm(up, L["conv"], dst, taps=ops.TAPS_3X3, geom=(2 * w, 2 * h, B),
                  stats=dp if self._fuse_stats(B, 2 * h, 2 * w) else None)
        return dst

    # ------------------------------------------------------------------ forward
    def forward(self, x_tokens: torch.Tensor, c_noise: torch.Tensor, cond_mask: Optional[torch.Tensor],
                h: int, w: int, net_out: Optional[torch.Tensor] = None, slot: str = "", cache_branch: int = 0,
                cached: bool = False) -> torch.Tensor:
        """x_tokens: [(B h w), 8] fp16 (x*c_in | concat), either contiguous or a view of zero-padded IN_PAD-wide rows
        (padded_input_rows); c_noise: [B] fp32; returns [(B h w), 8] fp32 whose first out_channels columns are the
        network output.  ``slot``: which conditioning of B rows to use (set_conditioning).

        ``cached`` (feature caching, Ma et al. 2024, DeepCache): run input blocks 0..b and output blocks n-1-b..n-1 only,
        b = ``cache_branch``.  Output block n-1-b reads the h half of its skip-concat buffer, and that half's GroupNorm
        column partials, as the last full forward of B rows at (h, w) left them: the feature is never copied, and a cached
        forward launches a subsequence of the full forward's launches."""
        cfg, T = self.cfg, self.T
        B = c_noise.numel()
        if cached:
            n_in = len(self.plan.input_blocks)
            if not 0 <= cache_branch < n_in or len(self.plan.output_blocks) != n_in:
                raise ValueError(f"cache_branch must be in [0, {n_in - 1}]; got {cache_branch}")
            if (B, h, w) not in self._h_filled:
                raise RuntimeError(f"a cached forward of {B} rows at {h} x {w} needs a full forward of them first")
        ckey = (B, slot) if slot else B
        assert ckey in self.conds, f"call set_conditioning() with {B} rows first" + (f" (slot {slot!r})" if slot else "")
        self.cond = self.conds[ckey]
        assert B % T == 0 and x_tokens.shape[0] == B * h * w
        mc, ed = cfg.model_channels, cfg.time_embed_dim
        # GroupNorm statistics / scratch are persistent per batch size (never replaced or freed): CUDA graphs and launch
        # tapes captured for another (B, h, w) keep replaying against the buffers they were captured with
        key = ("gn.stats", B)
        if key not in self._bufs:
            self._bufs[key] = torch.zeros(self.n_gn, B, cfg.num_groups, 2, dtype=torch.float32, device=self.dev)
        self.gn_stats = self._bufs[key]
        if not hasattr(self, "gn_ws"):
            self.gn_ws = ops.GNWorkspace(self.dev)
        self.gn_ws.reserve(ops.groupnorm_scratch(B, h * w, cfg.num_groups))
        # --- embeddings (video_model.py:456-471) + all emb_layers of the step in one GEMM
        temb = ops.timestep_embedding(c_noise, self.buf("emb.t", B, mc), mc)
        e_plain = self._mlp_step(temb, self.time_embed, "emb.plain")
        e_cond = self._mlp_step(temb, self.cond_embed, "emb.cond") if cond_mask is not None else None
        semb = self.buf("emb.silu", B, ed)
        ops.blend_emb(e_plain, e_cond, self.cond["label"], cond_mask, None, semb)
        self.emb_out = self.gemm(semb, self.emb_all, self.buf("emb.out", B, self.emb_total, torch.float32))

        plan = self.plan
        # geometry per input block + skip-concat buffers
        hs: List[Tuple[torch.Tensor, int, int]] = []
        n_out = len(plan.output_blocks)
        # channel count of `h` entering every output block
        ch_in_h = []
        ch = plan.middle_block.layers[-1].cout
        for blk in plan.output_blocks:
            ch_in_h.append(ch)
            ch = blk.layers[0].cout
        # spatial size of every output block's input
        sizes = []
        hh, ww = h, w
        in_sizes = []
        for blk in plan.input_blocks:
            if isinstance(blk.layers[0], ConvSpec) and blk.layers[0].kind == "down":
                hh, ww = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
            in_sizes.append((hh, ww))
        cat_bufs = []
        for j, blk in enumerate(plan.output_blocks):
            sh, sw = in_sizes[len(in_sizes) - 1 - j]
            cskip = plan.skip_channels[len(in_sizes) - 1 - j]
            cat_bufs.append(self.buf(f"cat{j}", B * sh * sw, ch_in_h[j] + cskip))
            sizes.append((sh, sw))

        def run_block(blk, x, dst, bh, bw, xp=None, dp=None):
            """xp: GroupNorm column partials of x (or None); dp: partial view to fill for dst (or None).  Returns
            (dst tensor, True if dp was filled)."""
            n_layers = len(blk.layers)
            filled = False
            for li, layer in enumerate(blk.layers):
                last = li == n_layers - 1
                L = self.layers[layer.prefix]
                if isinstance(layer, ResBlockSpec) or isinstance(layer, SVTSpec):
                    cch = layer.cout if isinstance(layer, ResBlockSpec) else layer.ch
                    fuse = self._fuse_stats(B, bh, bw)
                    d = dst if last else self.buf("blk.tmp%d" % li, B * bh * bw, cch)
                    p_out = (dp if last else self.part("blk.tmp%d" % li, B * bh * bw, cch)) if fuse else None
                    fn = self._resblock if isinstance(layer, ResBlockSpec) else self._svt
                    x = fn(L, x, d, B, bh, bw, xp=xp, dp=p_out)
                    xp = p_out
                    filled = p_out is not None
                elif layer.kind == "down":
                    ho, wo = (bh - 1) // 2 + 1, (bw - 1) // 2 + 1
                    x = self._down(L, x, dst, B, bh, bw, dp=dp)
                    filled = dp is not None and self._fuse_stats(B, ho, wo)
                elif layer.kind == "up":
                    x = self._up(L, x, dst, B, bh, bw, dp=dp)
                    filled = dp is not None and self._fuse_stats(B, 2 * bh, 2 * bw)
                elif layer.kind == "conv_in":
                    if x.stride(0) == IN_PAD:      # zero-padded rows: the input conv runs on the tensor cores
                        a = x.as_strided((x.shape[0], IN_PAD), (IN_PAD, 1))
                        fuse = dp is not None and self._fuse_stats(B, bh, bw)
                        x = self.gemm(a, L["conv"], dst, taps=ops.TAPS_3X3, geom=(bw, bh, B), stats=dp if fuse else None)
                        filled = fuse
                    else:
                        x = ops.conv3x3_small_cin(x, layer.cin, L["w"], L["b"], dst, B, bh, bw)
            return x, filled

        # GroupNorm column partials of the skip-concat buffers: two producers (h half, skip half) fill one matrix
        cat_parts = [self.part(f"cat{j}", cat_bufs[j].shape[0], cat_bufs[j].shape[1]) if self._fuse_stats(B, *sizes[j]) else None
                     for j in range(n_out)]
        cat_ok = [[False, False] for _ in range(n_out)]
        # --- input blocks: block i writes into the skip slice of output block (n-1-i)
        cur, cur_p = x_tokens, None
        hh, ww = h, w                      # size of the tensor entering the block
        for i, blk in enumerate(plan.input_blocks):
            if cached and i > cache_branch:
                break
            j = n_out - 1 - i
            dp = cat_parts[j][:, ch_in_h[j]:] if cat_parts[j] is not None else None
            cur, cat_ok[j][1] = run_block(blk, cur, cat_bufs[j][:, ch_in_h[j]:], hh, ww, xp=cur_p, dp=dp)
            cur_p = dp if cat_ok[j][1] else None
            hh, ww = in_sizes[i]
        # --- middle block -> h slice of output block 0
        j0 = n_out - 1 - cache_branch if cached else 0
        if cached:       # the h half of cat{j0} and its partials are the last full forward's: whether those were filled
            cat_ok[j0][0] = self._h_filled[(B, h, w)][j0]
        else:
            dp = cat_parts[0][:, :ch_in_h[0]] if cat_parts[0] is not None else None
            cur, cat_ok[0][0] = run_block(plan.middle_block, cur, cat_bufs[0][:, :ch_in_h[0]], hh, ww, xp=cur_p, dp=dp)
        # --- output blocks
        last_p = None
        for j, blk in enumerate(plan.output_blocks):
            if j < j0:
                continue
            bh, bw = sizes[j]
            if j + 1 < n_out:
                dst = cat_bufs[j + 1][:, :ch_in_h[j + 1]]
                dp = cat_parts[j + 1][:, :ch_in_h[j + 1]] if cat_parts[j + 1] is not None else None
            else:
                cl = blk.layers[-1].cout if not isinstance(blk.layers[-1], SVTSpec) else blk.layers[-1].ch
                dst = self.buf("unet.last", B * bh * bw, cl)
                dp = self.part("unet.last", B * bh * bw, cl) if self._fuse_stats(B, bh, bw) else None
            xp = cat_parts[j] if (cat_parts[j] is not None and all(cat_ok[j])) else None
            cur, ok = run_block(blk, cat_bufs[j], dst, bh, bw, xp=xp, dp=dp)
            if j + 1 < n_out:
                cat_ok[j + 1][0] = ok
            else:
                last_p = dp if ok else None
        if not cached:
            self._h_filled[(B, h, w)] = [ok[0] for ok in cat_ok]
        # --- out: GroupNorm32 -> SiLU -> conv3x3(320 -> 4)                      (video_model.py:434-440,502-503)
        M = B * h * w
        a = self._gn(cur, self.buf("out.a", M, mc), B, h * w, self.out_norm, 1e-5, True, self.out_gn_idx, part=last_p)
        if net_out is None:
            net_out = self.buf("unet.out", M, 8, torch.float32)
        self.gemm(a, self.out_conv, net_out, taps=ops.TAPS_3X3, geom=(w, h, B))
        return net_out

    def _mlp_step(self, temb, mlp, name):
        l0, l2 = mlp
        B = temb.shape[0]
        mid = self.gemm(temb, l0, self.buf(name + ".mid", B, l0.w.shape[0]), act=1)
        return self.gemm(mid, l2, self.buf(name + ".out", B, l2.w.shape[0], torch.float32))
