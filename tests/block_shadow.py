"""Layer-level shadow conformance, one level above tests/shadow.py: a context manager that wraps the runtimes' layer
methods (UNetRuntime._resblock / _svt / _down / _up, DecoderRuntime._resblock / _attn, EncoderRuntime._enc_resblock and
the _attn it inherits) and their forwards, and holds every layer of a run to the fp64 oracle (oracle/vista_oracle.py)
evaluated on the fp16 input that layer really read.

tests/shadow.py checks that each kernel launch computed the right thing from what it was given; this harness checks
what happens between launches:

  * layers: each hooked call clones its input before and its output after the call (torch copies only: the launch
    sequence is the runtime's own), synchronises, and compares the output with the oracle function of the same spec
    object (ResBlockSpec -> video_res_block, SVTSpec -> spatial_video_transformer, down / up -> the F.conv2d forms of
    unet_forward, decoder resblock -> dec_video_res_block, decoder / encoder attention -> dec_attn_block, encoder
    resblock -> enc_res_block), per clip of T frames;
  * segments: the pieces that have no method of their own (the input convolutions, the encoder's Downsample, the
    decoder's up-convolutions and the three heads) read the last captured output (or the network input) and write the
    next captured input (or the network output); layers and segments together cover each network end to end;
  * conditioning vectors (UNet): every ResBlock's emb_out slices, every transformer's cond["sp"] / cond["tm"] and
    cond["pos"], against emb_layers.1(silu(emb)), the oracle's single-key cross-attention and time_pos_embed;
  * hand-offs: the tensor a layer wrote must be bit-identical when its consumer reads it.  The producer of every input
    column range comes from the oracle's structure (the hs stack of unet_forward, the layer order of the plans), never
    from the runtime's buffers, so that a wrong routing cannot make itself look consistent;
  * coverage: every layer of build_unet_plan / build_decoder_plan / build_encoder_plan and every segment of a network
    that ran must have been checked, or the run fails by name.

Bound (layers and segments): the output is partitioned per frame, per GroupNorm group of channels (C / 32 channels;
one channel per group below 32 channels) and into the border ring of every frame (outermost rows and columns) against
the interior.  Per partition, rel-L2(out, ref) <= C_KIND[kind] x rho, rho the rel-L2 of the fp64 reference rounded to
fp16 (the rounding floor of assert_conform; also for the fp32 outputs: net_out, the moments and the frames).
Conditioning vectors are fp32: they take the GEMM family's element rule, |out - ref| <= ulp32(ref) + eps x mag.

Gain check (tests/bias.py), per layer with a residual or an alpha blend (the UNet's ResBlocks and transformers, the
decoder's and encoder's ResBlocks and mid attention), per clip: e = out - RN16(ref) is fitted to the residual operands
the oracle records (``record=``), as they enter the output, and to d out / d alpha (the difference of the two blend
branches, with the blend's sign; for a transformer mapped through proj_out), with one intercept per (frame, channel) to
absorb constants rounded once per frame (emb_out, the cross-attention rows), standard errors clustered by frame (by
128-token tile for one frame).  A term fails above B + 4 sigma, B = U16 / 8: a gain of one rounding in every residual
add, or an alpha one fp16 ulp off, passes the partition rule and fails this one.  The decoder's ResBlocks accumulate the
fit band by band with their reference (the temporal residual and d out / d alpha; the spatial residual of their pieces
is not kept).

Failures are collected per key, one report() prints the census (per layer prefix: kind, output shape, worst partition
ratio), and assert_ok() raises with every failure."""
import contextlib
import inspect
import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

import bias
from oracle import vista_oracle as vo
from test_conformance_cpu import FAMILY, U24, rel_l2, ulp
from vista_b200 import unet as unet_mod
from vista_b200 import vae as vae_mod
from vista_b200.spec import ConvSpec, DecResBlockSpec, ResBlockSpec, SVTSpec, build_decoder_plan, build_encoder_plan

U16 = 2.0 ** -11           # unit roundoff of fp16


# ==================================================================================================================
# Bounds
# ==================================================================================================================
def c_of(n_round: int) -> float:
    """Layer bound factor from the number of fp16 rounding points on the layer's longest path.  Each one (a weight
    rounded at packing, an fp16 intermediate stored, the output stored, P rounded before P.V) perturbs what follows by
    about 2^-11 relative per element; the GroupNorms / LayerNorms, convolutions and projections after it carry a
    relative error through at about its size (they normalise, or mix many independent terms with random weights), so
    each contributes about rho (the store of the output contributes exactly rho) to the output's rel-L2.  Independent
    errors add in quadrature: sqrt(n) rho.  The factor 2 is the margin for correlated roundings and for the partitions
    where a residual cancels part of the branch."""
    return 2.0 * math.sqrt(n_round)


# kind -> (rounding points on the longest path, the path)
ROUNDINGS = {
    "unet.resblock": (14, "a1 = GN+SiLU store, conv1 weights, emb_out (fp16 silu(emb) and weights), h1 store, a2 store, "
                          "conv2 weights, xsp store, a3 store, tconv1 weights, embt, h2 store, a4 store, tconv2 weights, "
                          "out store"),
    "unet.svt": (36, "GN store, proj_in w, t0, LN1, qkv w, qkv, P, o, out w, sp constant, t1, LN3, ff1 w, g, ff2 w, t2, "
                     "pos, LN_in, ffin1 w, g, ffin2 w, u1, tLN1, tqkv w, qkv, P, o, tout w, tm constant, u2, tLN3, "
                     "tff1 w, g, tff2 w, x3, proj_out w + out store (counted once: the proj_out GEMM adds x exactly)"),
    "unet.down": (2, "im2col is exact; conv weights, out store"),
    "unet.up": (2, "the nearest upsample is exact; conv weights, out store"),
    "unet.conv_in": (2, "conv weights (tap-GEMM form) and out store"),
    "unet.head": (2, "GN+SiLU store, conv weights; net_out is fp32"),
    "dec.resblock": (12, "a1, conv1 w, h1, a2, conv2 w, xsp, a3, tconv1 w, h2, a4, tconv2 w, out store"),
    "dec.attn": (9, "GN store, q w, q store, S fp32 from fp16 q / k, P store, V^T w, V^T store, O store, proj w + out "
                    "store (counted as one: the residual is exact)"),
    "dec.upconv": (2, "weights, out store"),
    "dec.conv_in": (1, "fp32 weights (conv3x3_small_cin), out store"),
    "dec.head": (2, "GN+SiLU store, conv_out weights; y and the time mix are fp32"),
    "enc.resblock": (6, "a1, conv1 w, h1, a2, conv2 w, out store"),
    "enc.attn": (9, "as dec.attn"),
    "enc.down": (2, "im2col is exact; weights, out store"),
    "enc.conv_in": (1, "fp32 weights (conv3x3_small_cin), out store"),
    "enc.head": (2, "GN+SiLU store, conv_out o quant_conv weights (composed in fp32, rounded once); moments are fp32"),
}
C_KIND = {k: c_of(n) for k, (n, _) in ROUNDINGS.items()}

# Conditioning vectors (fp32 outputs) take the element rule |out - ref| <= ulp32(ref) + sum_i eps_i mag_i, every term
# first order: an fp16 rounding of an operand or an intermediate moves each product by at most U16 of its magnitude,
# so a chain of r roundings is bounded by r U16 times the fp64 magnitude chain |W2|.(1.1 (|W1|.|x| + |b1|)) + |b2|
# (1.1 = the largest slope of SiLU), plus the fp32 accumulation c_acc sqrt(K) U24 of each GEMM (FAMILY["gemm"]).
EMB_UP_ROUNDINGS = 4       # per MLP: temb store (fp16), W1, the hidden store (fp16), W2; blend_emb is fp32
EMB_ROUNDINGS = 2          # emb_layers.1: silu(emb) stored in fp16, its weight
ATTN2_ROUNDINGS = 5        # context store, to_v / v_adapter weights, v store, v2 store, to_out weight
POS_ROUNDINGS = 4          # timestep_embedding store, W0, the hidden store, W2


def _acc(K):
    return FAMILY["gemm"].c_acc * math.sqrt(K) * U24


# ==================================================================================================================
# Gain check of a layer
# ==================================================================================================================
GAIN_KINDS = {"unet.resblock", "unet.svt", "dec.resblock", "dec.attn", "enc.resblock", "enc.attn"}
GAIN_B = bias.base_bound(torch.float16)


def layer_labels(n, C, rows, W, row0, dev):
    """(cluster, n_clusters, group, n_groups) of an (n, C, rows, W) piece starting at image row ``row0``: clusters are
    frames (128-token tiles of the frame when n = 1), the nuisance groups (frame, channel).  ``W`` and the tile count
    assume rows of width W; n_clusters is an upper bound (unused labels cost nothing)."""
    group = (torch.arange(n, device=dev)[:, None, None, None] * C + torch.arange(C, device=dev)[None, :, None, None])
    if n >= 2:
        return torch.arange(n, device=dev)[:, None, None, None], n, group, n * C
    tok = (row0 + torch.arange(rows, device=dev))[:, None] * W + torch.arange(W, device=dev)[None, :]
    return (tok // 128)[None, None], None, group, C


def layer_directions(kind, rec, sd, prefix):
    """name -> fp64 (n, C, H, W) directions of a layer's output from the oracle's record: its residual operands and
    d out / d alpha = a - b of the blend out = alpha a + (1 - alpha) b (a transformer's through proj_out's weight)."""
    d = {k: rec[k] for k in ("res", "res2d", "res3d") if k in rec}
    if "blend" in rec:
        _, a, b = rec["blend"]
        diff = a - b
        if kind == "unet.svt":
            B_, C, H, W = rec["res"].shape
            diff = F.linear(diff, sd[f"{prefix}.proj_out.weight"]).reshape(B_, H, W, C).permute(0, 3, 1, 2)
        d["d_alpha"] = diff
    return d


class LayerGain:
    """The gain fit of one layer and clip, accumulated piece by piece."""

    def __init__(self, names, n, C, H, W, dev):
        self.names, self.n, self.C, self.W = list(names), n, C, W
        n_cl = n if n >= 2 else -(-H * W // 128)
        self.fit = bias.GainFit(self.names, {k: GAIN_B for k in self.names}, n_cl, n * C, device=dev)

    def add(self, out, ref, dirs, row0=0):
        cl, _, group, _ = layer_labels(self.n, self.C, ref.shape[2], self.W, row0, ref.device)
        e = out - bias.rn(ref, torch.float16)
        self.fit.add(e, [dirs[k] for k in self.names], cl, group, out=ref)

    def result(self):
        return self.fit.result()


# ==================================================================================================================
# The oracle at production size: spatial attention chunked per (frame, head)
# ==================================================================================================================
class _ChunkedSDPA:
    """Stands in for torch.nn.functional inside oracle/vista_oracle.py while a reference is evaluated: the same
    functions, except that scaled_dot_product_attention runs over the leading (batch, head) pairs in chunks whose
    score matrices fit in ``budget`` bytes.  The fp64 math backend would otherwise materialise every score matrix of
    the call at once (50 frames x 5 heads x 9216^2 at 576 x 1024)."""
    budget = 1 << 28

    def __getattr__(self, name):
        return getattr(F, name)

    def scaled_dot_product_attention(self, q, k, v, *a, **kw):
        lead, n, m = q.shape[:-2], q.shape[-2], k.shape[-2]
        qf, kf, vf = (t.reshape((-1,) + tuple(t.shape[-2:])) for t in (q, k, v))
        per = max(1, self.budget // max(1, n * m * q.element_size()))
        if per >= qf.shape[0]:
            return F.scaled_dot_product_attention(q, k, v, *a, **kw)
        out = torch.empty(qf.shape[0], n, vf.shape[-1], dtype=q.dtype, device=q.device)
        for i in range(0, qf.shape[0], per):
            out[i:i + per] = F.scaled_dot_product_attention(qf[i:i + per], kf[i:i + per], vf[i:i + per], *a, **kw)
        return out.reshape(tuple(lead) + (n, vf.shape[-1]))


@contextlib.contextmanager
def chunked_oracle(device):
    """The oracle's functional namespace with the chunked attention, and its timestep_embedding (fp32 on the host: the
    oracle's fp32 island; for the frame indices t < 25 of time_pos_embed its cos / sin are off by ~1e-6 absolute, far
    below the fp16 roundings of the bound) handed on in fp64 on ``device``, where the layer's reference runs."""
    saved, saved_te = vo.F, vo.timestep_embedding
    vo.F = _ChunkedSDPA()
    vo.timestep_embedding = lambda t, dim, max_period=10000.0: saved_te(t.cpu(), dim, max_period).to(device, torch.float64)
    try:
        yield
    finally:
        vo.F, vo.timestep_embedding = saved, saved_te


# ==================================================================================================================
# The decoder's oracle at production size, in pieces
# ==================================================================================================================
# At 576 x 1024 one fp64 tensor of a 14-frame decoder activation is 8.5 GiB (128 channels) to 17 GiB (256), and the
# oracle functions keep several alive at once.  The same maths runs in pieces: everything spatial (the per-frame
# GroupNorms, the 3x3 convolutions, the nearest upsample, the head's conv_out) works on one frame at a time, the clip's
# GroupNorm statistics of the temporal half are reduced over the whole clip in fp64, and the temporal half's (3,1,1)
# convolutions are pointwise in space, so they run on bands of rows with all frames.  test_block_conformance_cpu.py
# holds the pieces equal to the oracle functions (to fp64 re-association).
BAND_BYTES = 1 << 28       # fp64 bytes of one (C, T, rows, W) band of the temporal half


def group_stats(parts, groups):
    """(mean, biased var) per group [G] of a tensor given as pieces (C, ...) that together form it: Chan's merge of
    each piece's count, mean and sum of squared deviations, in fp64."""
    n, mean, m2 = 0, None, None
    for t in parts:
        C = t.shape[0]
        v = t.reshape(groups, -1)
        nb = v.shape[1]
        mb = v.mean(1)
        m2b = ((v - mb[:, None]) ** 2).sum(1)
        if mean is None:
            n, mean, m2 = nb, mb, m2b
        else:
            d = mb - mean
            tot = n + nb
            mean = mean + d * (nb / tot)
            m2 = m2 + m2b + d * d * (n * nb / tot)
            n = tot
    return mean, m2 / n


def _gn_apply(x, mean, var, gamma, beta, eps, groups):
    """F.group_norm of x (C, ...) with given group statistics."""
    C = x.shape[0]
    shape = (groups, C // groups) + tuple(x.shape[1:])
    bc = (-1,) + (1,) * (x.dim() - 1)
    y = (x.reshape(shape) - mean.reshape((groups,) + (1,) * x.dim())) * \
        torch.rsqrt(var + eps).reshape((groups,) + (1,) * x.dim())
    return y.reshape(x.shape) * gamma.reshape(bc) + beta.reshape(bc)


def dec_video_res_block_pieces(sd, p, frame, T, has_skip, sink, groups=32, band_bytes=BAND_BYTES, with_dirs=False):
    """vista_oracle.dec_video_res_block in pieces.  frame(f) -> fp64 (1, Cin, H, W) of input frame f; sink(ref, r0)
    receives the output rows r0 : r0 + ref.shape[2] of every frame, ref (T, C, rows, W); ``with_dirs``: sink(ref, r0,
    dirs) with the band's gain directions, "res3d" (the temporal residual operand) and "d_alpha" (temporal minus
    spatial branch: the blend is alpha temporal + (1 - alpha) spatial).
    Spatial half (per frame, its GroupNorms are per frame): the oracle's own enc_res_block, the first lines of
    dec_video_res_block.  Temporal half: res_block_3d (GroupNorm over (C/32, T, H, W), eps 1e-5, SiLU, (3,1,1)
    convolutions zero padded over frames) and the blend alpha * temporal + (1 - alpha) * spatial."""
    # the spatial half's output (C, T, H, W) in fp64 is kept in host memory (8.5 GiB for 14 frames of 128 channels at
    # 576 x 1024) and brought to the device one band at a time
    xs = None
    for f in range(T):
        o = vo.enc_res_block(sd, p, frame(f), has_skip)[0]
        if xs is None:
            dev = o.device
            xs = torch.empty((o.shape[0], T) + tuple(o.shape[1:]), dtype=torch.float64)
        xs[:, f] = o.cpu()
        del o
    C, _, H, W = xs.shape
    t = f"{p}.time_stack"
    rows = max(1, band_bytes // (C * T * W * 8))
    bands = [(r0, min(H, r0 + rows)) for r0 in range(0, H, rows)]
    band = lambda r0, r1: xs[:, :, r0:r1].to(dev)
    m1, v1 = group_stats((band(r0, r1) for r0, r1 in bands), groups)

    def h1(r0, r1):
        a = F.silu(_gn_apply(band(r0, r1), m1, v1, sd[f"{t}.in_layers.0.weight"], sd[f"{t}.in_layers.0.bias"], 1e-5,
                             groups))
        return F.conv3d(a[None], sd[f"{t}.in_layers.2.weight"], sd[f"{t}.in_layers.2.bias"], padding=(1, 0, 0))[0]
    m2, v2 = group_stats((h1(r0, r1) for r0, r1 in bands), groups)
    alpha = torch.sigmoid(sd[f"{p}.mix_factor"])
    for r0, r1 in bands:
        a = F.silu(_gn_apply(h1(r0, r1), m2, v2, sd[f"{t}.out_layers.0.weight"], sd[f"{t}.out_layers.0.bias"], 1e-5,
                             groups))
        h2 = F.conv3d(a[None], sd[f"{t}.out_layers.3.weight"], sd[f"{t}.out_layers.3.bias"], padding=(1, 0, 0))[0]
        x5 = band(r0, r1)
        ref = (alpha * (x5 + h2) + (1.0 - alpha) * x5).transpose(0, 1)
        if with_dirs:
            sink(ref, r0, {"res3d": x5.transpose(0, 1), "d_alpha": h2.transpose(0, 1)})
        else:
            sink(ref, r0)


def upconv_pieces(w, b, frame, T, sink):
    """The up-convolution (nearest x2, conv 3x3 pad 1) of decoder_forward, frame by frame: sink(ref (1, C, 2H, 2W), f)."""
    for f in range(T):
        sink(F.conv2d(F.interpolate(frame(f), scale_factor=2, mode="nearest"), w, b, padding=1), f)


def decoder_head_pieces(sd, frame, T):
    """The tail of decoder_forward: GroupNorm (per frame) + swish + conv_out frame by frame, then the 3-channel
    time_mix_conv over the clip.  Returns the frames (T, out_ch, H, W)."""
    y = torch.cat([F.conv2d(vo._swish(vo._gn(sd, "norm_out", frame(f), 1e-6)), sd["conv_out.weight"], sd["conv_out.bias"],
                            padding=1) for f in range(T)])
    y5 = F.conv3d(y.transpose(0, 1)[None], sd["conv_out.time_mix_conv.weight"], sd["conv_out.time_mix_conv.bias"],
                  padding=(1, 0, 0))
    return y5[0].transpose(0, 1)


# ==================================================================================================================
# Network structure: the producer of every input column range, from the oracle's structure
# ==================================================================================================================
class Node:
    def __init__(self, name, kind, spec, inputs, cout, hooked):
        self.name, self.kind, self.spec, self.inputs, self.cout, self.hooked = name, kind, spec, inputs, cout, hooked


def _cout(layer):
    return layer.ch if isinstance(layer, SVTSpec) else layer.cout


def unet_graph(plan) -> Dict[str, Node]:
    """unet_forward's dataflow: input blocks push their outputs on hs, output block j reads cat(h, hs.pop())."""
    nodes: Dict[str, Node] = {}
    kinds = {"conv_in": "unet.conv_in", "down": "unet.down", "up": "unet.up"}
    prev, pch = "net.in", plan.cfg.in_channels
    hs: List[Tuple[str, int]] = []

    def add(layer, inputs):
        kind = ("unet.resblock" if isinstance(layer, ResBlockSpec) else "unet.svt" if isinstance(layer, SVTSpec)
                else kinds[layer.kind])
        nodes[layer.prefix] = Node(layer.prefix, kind, layer, inputs, _cout(layer), kind != "unet.conv_in")
        return layer.prefix, _cout(layer)

    for blk in plan.input_blocks:
        for layer in blk.layers:
            prev, pch = add(layer, [(prev, 0, pch)])
        hs.append((prev, pch))
    for layer in plan.middle_block.layers:
        prev, pch = add(layer, [(prev, 0, pch)])
    for blk in plan.output_blocks:
        for li, layer in enumerate(blk.layers):
            if li == 0:
                skip, sch = hs.pop()
                prev, pch = add(layer, [(prev, 0, pch), (skip, pch, pch + sch)])
            else:
                prev, pch = add(layer, [(prev, 0, pch)])
    nodes["out"] = Node("out", "unet.head", None, [(prev, 0, pch)], plan.cfg.out_channels, False)
    return nodes


def decoder_graph(cfg) -> Dict[str, Node]:
    """decoder_forward's layer order: conv_in, mid (res, attn, res), per level the blocks and the up-convolution, head."""
    plan = build_decoder_plan(cfg)
    nodes: Dict[str, Node] = {}
    nodes["conv_in"] = Node("conv_in", "dec.conv_in", None, [("net.in", 0, cfg.z_channels)], plan.block_in, False)
    prev, pch = "conv_in", plan.block_in
    seq = [plan.mid[0], "mid.attn_1", plan.mid[1]]
    for blocks, up, ch in plan.levels:
        seq += list(blocks) + ([(up, ch)] if up is not None else [])
    for item in seq:
        if isinstance(item, DecResBlockSpec):
            nodes[item.prefix] = Node(item.prefix, "dec.resblock", item, [(prev, 0, pch)], item.cout, True)
            prev, pch = item.prefix, item.cout
        elif item == "mid.attn_1":
            nodes[item] = Node(item, "dec.attn", None, [(prev, 0, pch)], pch, True)
            prev = item
        else:
            up, ch = item
            nodes[up] = Node(up, "dec.upconv", None, [(prev, 0, pch)], ch, False)
            prev, pch = up, ch
    nodes["out"] = Node("out", "dec.head", None, [(prev, 0, pch)], cfg.out_ch, False)
    return nodes


def encoder_graph(cfg) -> Dict[str, Node]:
    """encoder_forward's layer order: conv_in, per level the blocks and the Downsample, mid (res, attn, res), head."""
    levels, mid_ch = build_encoder_plan(cfg)
    nodes: Dict[str, Node] = {}
    nodes["conv_in"] = Node("conv_in", "enc.conv_in", None, [("net.in", 0, cfg.in_channels)], cfg.ch, False)
    prev, pch = "conv_in", cfg.ch
    seq = []
    for blocks, down, ch in levels:
        seq += list(blocks) + ([(down, ch)] if down is not None else [])
    seq += [DecResBlockSpec("mid.block_1", mid_ch, mid_ch), "mid.attn_1", DecResBlockSpec("mid.block_2", mid_ch, mid_ch)]
    for item in seq:
        if isinstance(item, DecResBlockSpec):
            nodes[item.prefix] = Node(item.prefix, "enc.resblock", item, [(prev, 0, pch)], item.cout, True)
            prev, pch = item.prefix, item.cout
        elif item == "mid.attn_1":
            nodes[item] = Node(item, "enc.attn", None, [(prev, 0, pch)], pch, True)
            prev = item
        else:
            down, ch = item
            nodes[down] = Node(down, "enc.down", None, [(prev, 0, pch)], ch, False)
            prev, pch = down, ch
    nodes["out"] = Node("out", "enc.head", None, [(prev, 0, pch)], 2 * cfg.z_channels, False)
    return nodes


# ==================================================================================================================
# Partitions
# ==================================================================================================================
def nchw(t, n, h, w, C):
    """Token rows [(n h w), >= C] -> fp64 (n, C, h, w)."""
    return t[:, :C].double().reshape(n, h, w, C).permute(0, 3, 1, 2)


class Parts:
    """Squared error and squared fp16 rounding floor per partition: frame, GroupNorm group, border ring, interior."""

    def __init__(self):
        self.e2: Dict[tuple, float] = {}
        self.f2: Dict[tuple, float] = {}

    def _put(self, key, e, f):
        self.e2[key] = self.e2.get(key, 0.0) + float(e)
        self.f2[key] = self.f2.get(key, 0.0) + float(f)

    def add(self, out, ref, frame0=0, row0=0, height=None):
        """out / ref (frames, C, rows, W) fp64: rows row0 : row0 + rows of frames frame0 ... of a (height x W) image."""
        n, C, H, W = ref.shape
        height = H if height is None else height
        assert out.shape == ref.shape, (out.shape, ref.shape)
        err = (out - ref) ** 2
        flo = (ref.to(torch.float16).double() - ref) ** 2
        ef, ff = err.sum((1, 2, 3)), flo.sum((1, 2, 3))
        for i in range(n):
            self._put(("frame", frame0 + i), ef[i], ff[i])
        G = 32 if C % 32 == 0 else C
        eg, fg = err.reshape(n, G, C // G, H, W).sum((0, 2, 3, 4)), flo.reshape(n, G, C // G, H, W).sum((0, 2, 3, 4))
        for g in range(G):
            self._put(("group", g), eg[g], fg[g])
        ring = torch.zeros(H, W, dtype=torch.bool, device=ref.device)
        ring[:, 0], ring[:, -1] = True, True
        if row0 == 0:
            ring[0] = True
        if row0 + H == height:
            ring[-1] = True
        es, fs = err.sum((0, 1)), flo.sum((0, 1))
        self._put(("border",), es[ring].sum(), fs[ring].sum())
        if bool((~ring).any()):
            self._put(("interior",), es[~ring].sum(), fs[~ring].sum())

    def worst(self, c):
        """(worst ratio rel-L2 / (c rho), its partition)."""
        best = (0.0, None)
        for k, e in self.e2.items():
            f = self.f2[k]
            r = math.sqrt(e / f) / c if f > 0 else (0.0 if e == 0 else math.inf)
            if not math.isfinite(e):
                r = math.inf
            if r > best[0] or best[1] is None:
                best = (r, k)
        return best


# ==================================================================================================================
# The harness
# ==================================================================================================================
class Census:
    def __init__(self, kind):
        self.kind, self.shape, self.ratio, self.part, self.calls = kind, None, 0.0, None, 0
        self.gain, self.gain_term = 0.0, None         # worst |beta| / (B + 4 sigma) over its clips, and that term


class Run:
    """One forward of one runtime: the graph, the captured outputs still to be read, the network's inputs."""

    def __init__(self, net, rt, nodes, check_layers):
        self.net, self.rt, self.nodes, self.check_layers = net, rt, nodes, check_layers
        self.out: Dict[str, torch.Tensor] = {}
        self.geom: Dict[str, Tuple[int, int, int]] = {}
        self.readers = {n: 0 for n in nodes}
        self.readers["net.in"] = 0
        for nd in nodes.values():
            for p, _, _ in nd.inputs:
                self.readers[p] += 1
        self.done = set()


class BlockShadow:
    """``with BlockShadow(unet=(cfg, sd), decoder=(cfg, sd), encoder=(cfg, sd, post)) as bs: ...`` checks every layer,
    segment, conditioning vector and hand-off of the runs of the block; sd are the reference state dicts (fp32, any
    device); post = (W [o, 2 z], b [o]) the encoder's quant_conv or None.  ``decoder_layer_calls``: how many decoder
    forwards get layer checks (hand-offs are checked on every forward); None = all."""

    HOOKS = (
        (unet_mod.UNetRuntime, ("forward", "set_conditioning", "_resblock", "_svt", "_down", "_up")),
        (vae_mod.DecoderRuntime, ("forward", "_resblock", "_attn")),
        (vae_mod.EncoderRuntime, ("forward", "_enc_resblock")),
    )

    def __init__(self, unet=None, decoder=None, encoder=None, decoder_layer_calls=None, gain: bool = True):
        self.sd = {"unet": unet, "dec": decoder, "enc": encoder}
        self.gain = gain              # the gain check of the layers in GAIN_KINDS
        self.decoder_layer_calls = decoder_layer_calls
        self.census: Dict[str, Census] = {}
        self.failures: Dict[tuple, str] = {}
        self.handoffs = 0
        self.vectors: Dict[str, float] = {}
        self.ran = set()
        self.checked = {"unet": set(), "dec": set(), "enc": set()}
        self.n_forward = {"unet": 0, "dec": 0, "enc": 0}
        self._saved = []
        self._runs: Dict[int, Run] = {}
        self._cond_in: Dict[tuple, tuple] = {}

    # ------------------------------------------------------------------ install
    def __enter__(self):
        for cls, names in self.HOOKS:
            for name in names:
                real = cls.__dict__[name]
                self._saved.append((cls, name, real))
                setattr(cls, name, getattr(self, f"_hook_{'forward' if name == 'forward' else name.lstrip('_')}")(cls, real))
        return self

    def __exit__(self, *exc):
        for cls, name, real in reversed(self._saved):
            setattr(cls, name, real)
        self._saved = []
        return False

    # ------------------------------------------------------------------ helpers
    def _fail(self, key, msg):
        self.failures.setdefault(key, msg)

    def _sdl(self, net, prefix, dev):
        """The layer's reference weights in fp64 on the device (freed by the caller)."""
        sd = self.sd[net][1]
        pre = prefix + "."
        return {k: v.to(dev, torch.float64) for k, v in sd.items() if k.startswith(pre)}

    def _note(self, name, kind, shape, parts):
        c = C_KIND[kind]
        r, part = parts.worst(c)
        e = self.census.setdefault(name, Census(kind))
        e.shape, e.calls = tuple(shape), e.calls + 1
        if r >= e.ratio:
            e.ratio, e.part = r, part
        if r > 1.0:
            self._fail(("layer", name), f"{name} ({kind}): partition {part} rel-L2 is {r:.2f} x the bound "
                                        f"{c:.2f} rho")

    def _gain_note(self, name, kind, terms, clip):
        w = bias.worst(terms)
        e = self.census.setdefault(name, Census(kind))
        if w is not None and w.ratio >= e.gain:
            e.gain, e.gain_term = w.ratio, w
        bad = bias.failures(terms)
        if bad:
            self._fail(("gain", name), f"{name} ({kind}), clip {clip}: systematic gain on " +
                       "; ".join(repr(t) for t in bad))

    def _elements(self, name, out, ref, tol):
        err = (out.double() - ref).abs()
        r = float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0
        self.vectors[name] = max(self.vectors.get(name, 0.0), r)
        if not r <= 1.0:
            i = int(torch.argmax(err / tol.clamp_min(1e-300)))
            self._fail(("vector", name), f"{name}: {r:.2f} x the element bound; flat index {i}: out "
                                         f"{float(out.flatten()[i]):.7g} ref {float(ref.flatten()[i]):.7g}")

    @staticmethod
    def _sync(t):
        if t.is_cuda:
            torch.cuda.synchronize(t.device)

    # ------------------------------------------------------------------ runs
    def _begin(self, net, rt, nodes, net_in, geom):
        self.ran.add(net)
        self.n_forward[net] += 1
        check = True
        if net == "dec" and self.decoder_layer_calls is not None:
            check = self.n_forward[net] <= self.decoder_layer_calls
        run = Run(net, rt, nodes, check)
        run.out["net.in"], run.geom["net.in"] = net_in, geom
        self._runs[id(rt)] = run
        return run

    def _consume(self, run, node, x):
        """Hand-offs into ``node`` from the captured input x; a segment producer's output is x's column range (then
        that segment is checked)."""
        for p, c0, c1 in node.inputs:
            got = x[:, c0:c1]
            if p not in run.out:
                pn = run.nodes[p]
                assert not pn.hooked, f"{p} feeds {node.name} but never ran"
                run.out[p] = got.clone()
                run.geom[p] = run.geom[node.name + ".in"]
                self._segment(run, pn, got)
            else:
                want = run.out[p]
                self.handoffs += 1
                same = want.shape == got.shape and torch.equal(want, got)
                if not same:
                    n_bad = int((want != got).sum()) if want.shape == got.shape else -1
                    pl, cl = self.label(run.net, p), self.label(run.net, node.name)
                    self._fail(("handoff", pl, cl), f"hand-off {pl} -> {cl} (input columns {c0}:{c1}): "
                                                    f"not bit-identical, {n_bad} elements differ")
            run.readers[p] -= 1
            if run.readers[p] == 0:
                run.out.pop(p, None)

    def _produced(self, run, node, y, geom):
        if run.readers.get(node.name, 0) > 0:
            run.out[node.name] = y
        run.geom[node.name] = geom
        run.done.add(node.name)

    def _layer_call(self, rt, name, x, call, geom_in, geom_out, extra=None):
        """Clone x, run the layer, clone its output, synchronise; hand-offs, then the layer check."""
        run = self._runs.get(id(rt))
        x0 = x.clone()
        self._sync(x0)
        ret = call()
        y = ret[0] if isinstance(ret, tuple) else ret
        y0 = y.clone()
        self._sync(y0)
        if run is None:
            return ret
        node = run.nodes.get(name)
        if node is None:
            self._fail(("unknown", name), f"{name}: a layer call the {run.net} plan does not contain")
            return ret
        run.geom[name + ".in"] = geom_in
        self._consume(run, node, x0)
        if run.check_layers:
            self._check(run, node, x0, y0, geom_in, geom_out, extra)
        self._produced(run, node, y0, geom_out)
        return ret

    def _finish(self, run, out_ref_fn):
        """End of a forward: the head segment against the network output."""
        head = run.nodes["out"]
        p = head.inputs[0][0]
        x = run.out.get(p)
        if x is None:
            self._fail(("missing", run.net, p), f"{run.net}: {p} (the head's input) was never captured")
        elif run.check_layers:
            out_ref_fn(head, x)
        run.done.add("out")
        missing = [n for n, nd in run.nodes.items() if n not in run.done]
        if missing:
            self._fail(("missing", run.net, tuple(missing)), f"{run.net}: layers that never ran: {missing}")
        self._runs.pop(id(run.rt), None)

    # ------------------------------------------------------------------ layer checks
    def _check(self, run, node, x, y, gi, go, extra):
        net, kind = run.net, node.kind
        n, h, w = gi
        no, ho, wo = go
        C_in = node.inputs[-1][2]
        dev = x.device
        T = run.rt.T if net == "unet" else n
        parts = Parts()
        sdl = self._sdl(net, node.name if kind not in ("dec.attn", "enc.attn") else "mid.attn_1", dev)
        clips = n // T if net == "unet" else 1
        label = self.label(net, node.name)
        if kind in ("dec.resblock", "dec.upconv"):
            frame = lambda f: nchw(x[f * h * w:(f + 1) * h * w], 1, h, w, C_in)
            yt = y.reshape(T, ho, wo, -1)
            if kind == "dec.resblock" and not self.gain:
                sink = lambda ref, r0: parts.add(yt[:, r0:r0 + ref.shape[2], :, :node.cout].permute(0, 3, 1, 2).double(),
                                                 ref, 0, r0, ho)
                with torch.no_grad():
                    dec_video_res_block_pieces(sdl, node.name, frame, T, node.spec.has_skip, sink)
            elif kind == "dec.resblock":
                lg = LayerGain(("res3d", "d_alpha"), T, node.cout, ho, wo, dev)

                def sink(ref, r0, dirs):
                    yo = yt[:, r0:r0 + ref.shape[2], :, :node.cout].permute(0, 3, 1, 2).double()
                    parts.add(yo, ref, 0, r0, ho)
                    lg.add(yo, ref, dirs, r0)
                with torch.no_grad():
                    dec_video_res_block_pieces(sdl, node.name, frame, T, node.spec.has_skip, sink, with_dirs=True)
                self._gain_note(label, kind, lg.result(), 0)
            else:
                sink = lambda ref, f: parts.add(yt[f:f + 1, :, :, :node.cout].permute(0, 3, 1, 2).double(), ref, f)
                with torch.no_grad():
                    upconv_pieces(sdl[f"{node.name}.weight"], sdl[f"{node.name}.bias"], frame, T, sink)
            clips = 0
        with torch.no_grad(), chunked_oracle(dev):
            for c in range(clips):
                xr = x[c * T * h * w:(c + 1) * T * h * w]
                xi = nchw(xr, T, h, w, C_in)
                rec = {} if self.gain and kind in GAIN_KINDS else None
                if kind == "unet.resblock":
                    ref = vo.video_res_block(sdl, node.spec, xi, run.emb[c * T:(c + 1) * T], T, record=rec)
                elif kind == "unet.svt":
                    ref = vo.spatial_video_transformer(sdl, node.spec, xi, run.ctx[c * T:(c + 1) * T], T,
                                                       run.rt.cfg.context_dim, record=rec)
                elif kind == "unet.down":
                    ref = F.conv2d(xi, sdl[f"{node.name}.weight"], sdl[f"{node.name}.bias"], stride=2, padding=1)
                elif kind == "unet.up":
                    ref = F.conv2d(F.interpolate(xi, scale_factor=2, mode="nearest"), sdl[f"{node.name}.weight"],
                                   sdl[f"{node.name}.bias"], padding=1)
                elif kind in ("dec.attn", "enc.attn"):
                    ref = vo.dec_attn_block(sdl, "mid.attn_1", xi, record=rec)
                elif kind == "enc.resblock":
                    ref = vo.enc_res_block(sdl, node.name, xi, node.spec.has_skip, record=rec)
                elif kind == "enc.down":
                    ref = F.conv2d(F.pad(xi, (0, 1, 0, 1)), sdl[f"{node.name}.weight"], sdl[f"{node.name}.bias"],
                                   stride=2)
                elif kind in ("unet.conv_in", "dec.conv_in", "enc.conv_in"):
                    ref = F.conv2d(xi, sdl[f"{node.name}.weight"], sdl[f"{node.name}.bias"], padding=1)
                else:
                    raise AssertionError(kind)
                yo = nchw(y[c * T * ho * wo:(c + 1) * T * ho * wo], T, ho, wo, node.cout)
                parts.add(yo, ref, c * T)
                if rec is not None:
                    dirs = layer_directions(kind, rec, sdl, node.name)
                    lg = LayerGain(list(dirs), T, node.cout, ho, wo, dev)
                    lg.add(yo, ref, dirs)
                    self._gain_note(label, kind, lg.result(), c)
                    del dirs, lg
                del ref, xi, yo, rec
        del sdl
        self._note(label, kind, (no * ho * wo, node.cout), parts)
        self.checked[net].add(node.name)
        if extra is not None:
            extra()

    def _segment(self, run, node, y):
        """A segment without a method: its input is its producer's captured output, its output ``y``."""
        p = node.inputs[0][0]
        if not run.check_layers:
            run.done.add(node.name)
            run.readers[p] -= 1
            if run.readers[p] == 0:
                run.out.pop(p, None)
            return
        gi = run.geom[p]
        n, h, w = gi
        if node.kind in ("dec.upconv",):
            go = (n, 2 * h, 2 * w)
        elif node.kind == "enc.down":
            go = (n, (h - 2) // 2 + 1, (w - 2) // 2 + 1)
        else:
            go = gi
        self._check(run, node, run.out[p], y, gi, go, None)
        run.done.add(node.name)
        run.readers[p] -= 1
        if run.readers[p] == 0:
            run.out.pop(p, None)

    # ------------------------------------------------------------------ UNet hooks
    def _hook_forward(self, cls, real):
        sig = inspect.signature(real)
        bs = self

        if cls is unet_mod.UNetRuntime:
            def forward(rt, *a, **k):
                A = sig.bind(rt, *a, **k)
                A.apply_defaults()
                A = A.arguments
                x, c_noise, mask, h, w = A["x_tokens"], A["c_noise"], A["cond_mask"], A["h"], A["w"]
                B = c_noise.numel()
                run = bs._begin("unet", rt, unet_graph(rt.plan), x[:, :rt.cfg.in_channels].clone(), (B, h, w))
                run.c_noise = c_noise.clone()
                run.mask = None if mask is None else mask.clone()
                assert (id(rt), B) in bs._cond_in, f"block shadow: set_conditioning({B} rows) ran outside the harness"
                ctx, y = bs._cond_in[(id(rt), B)]
                dev = x.device
                run.ctx = ctx.to(dev, torch.float64)
                run.y = y.to(dev, torch.float64)
                run.emb, run.emb_mag = bs._emb(run)
                run.vec_done = False
                out = real(rt, *a, **k)
                net = out.clone()
                bs._sync(net)
                bs._finish(run, lambda head, xh: bs._unet_head(run, head, xh, net))
                return out
            return forward

        if cls is vae_mod.EncoderRuntime:
            def forward(rt, *a, **k):
                A = sig.bind(rt, *a, **k)
                A.apply_defaults()
                A = A.arguments
                x, n, h, w = A["x_tokens"], A["n"], A["h"], A["w"]
                run = bs._begin("enc", rt, encoder_graph(rt.cfg), x[:, :rt.cfg.in_channels].clone(), (n, h, w))
                out = real(rt, *a, **k)
                mom = out.clone()
                bs._sync(mom)
                bs._finish(run, lambda head, xh: bs._enc_head(run, head, xh, mom))
                return out
            return forward

        def forward(rt, *a, **k):           # DecoderRuntime
            A = sig.bind(rt, *a, **k)
            A.apply_defaults()
            A = A.arguments
            z, T, h, w = A["z_tokens"], A["T"], A["h"], A["w"]
            run = bs._begin("dec", rt, decoder_graph(rt.cfg), z[:, :rt.cfg.z_channels].clone(), (T, h, w))
            out = real(rt, *a, **k)
            frames = A["out"]
            bs._sync(frames)
            bs._finish(run, lambda head, xh: bs._dec_head(run, head, xh, A))
            return out
        return forward

    def _hook_set_conditioning(self, cls, real):
        bs = self

        def set_conditioning(rt, context, y):
            bs._cond_in[(id(rt), context.shape[0])] = (context.detach().clone(), y.detach().clone())
            return real(rt, context, y)
        return set_conditioning

    def _hook_resblock(self, cls, real):
        bs = self
        if cls is unet_mod.UNetRuntime:
            def resblock(rt, L, x, dst, B, h, w, xp=None, dp=None):
                return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, dst, B, h, w, xp=xp, dp=dp),
                                      (B, h, w), (B, h, w), extra=lambda: bs._emb_vectors(rt, L))
            return resblock

        def resblock(rt, L, x, T, h, w, name, xp=None):
            return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, T, h, w, name, xp), (T, h, w), (T, h, w))
        return resblock

    def _hook_enc_resblock(self, cls, real):
        bs = self

        def enc_resblock(rt, L, x, n, h, w, name):
            return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, n, h, w, name), (n, h, w), (n, h, w))
        return enc_resblock

    def _hook_attn(self, cls, real):
        bs = self

        def attn(rt, x, T, h, w, xp=None):
            return bs._layer_call(rt, "mid.attn_1", x, lambda: real(rt, x, T, h, w, xp), (T, h, w), (T, h, w))
        return attn

    def _hook_svt(self, cls, real):
        bs = self

        def svt(rt, L, x, dst, B, h, w, xp=None, dp=None):
            return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, dst, B, h, w, xp=xp, dp=dp),
                                  (B, h, w), (B, h, w), extra=lambda: bs._svt_vectors(rt, L))
        return svt

    def _hook_down(self, cls, real):
        bs = self

        def down(rt, L, x, dst, B, h, w, dp=None):
            return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, dst, B, h, w, dp=dp), (B, h, w),
                                  (B, (h - 1) // 2 + 1, (w - 1) // 2 + 1))
        return down

    def _hook_up(self, cls, real):
        bs = self

        def up(rt, L, x, dst, B, h, w, dp=None):
            return bs._layer_call(rt, L["spec"].prefix, x, lambda: real(rt, L, x, dst, B, h, w, dp=dp), (B, h, w),
                                  (B, 2 * h, 2 * w))
        return up

    # ------------------------------------------------------------------ UNet conditioning vectors
    def _mlp_mag(self, sd, p0, p2, x, xmag):
        """(fp64 Linear -> SiLU -> Linear of x, its magnitude chain |W2|.(1.1 (|W1|.xmag + |b1|)) + |b2|)."""
        w0, b0, w2, b2 = sd[f"{p0}.weight"], sd[f"{p0}.bias"], sd[f"{p2}.weight"], sd[f"{p2}.bias"]
        out = F.linear(F.silu(F.linear(x, w0, b0)), w2, b2)
        mag = (1.1 * (xmag @ w0.abs().t() + b0.abs())) @ w2.abs().t() + b2.abs()
        return out, mag

    def _emb(self, run):
        """emb of unet_forward (oracle lines 185-192) in fp64 from the c_noise, cond_mask and vector the forward
        received, and its magnitude chain.  timestep_embedding is the oracle's fp32 one: its cos / sin of arguments
        |c_noise| < 4 are off by ~1e-7, far below the fp16 roundings of the bound."""
        rt, dev = run.rt, run.c_noise.device
        sd = {k: v.to(dev, torch.float64) for k, v in self.sd["unet"][1].items()
              if k.split(".")[0] in ("time_embed", "cond_time_stack_embed", "label_emb")}
        t = vo.timestep_embedding(run.c_noise.double().cpu(), rt.cfg.model_channels).to(dev, torch.float64)
        plain, m_plain = self._mlp_mag(sd, "time_embed.0", "time_embed.2", t, t.abs())
        if run.mask is not None and bool(run.mask.any()):
            m = run.mask.double().reshape(-1, 1)
            cond, m_cond = self._mlp_mag(sd, "cond_time_stack_embed.0", "cond_time_stack_embed.2", t, t.abs())
            emb, mag = cond * m + plain * (1 - m), m_cond * m + m_plain * (1 - m)
        else:
            emb, mag = plain, m_plain
        lab, m_lab = self._mlp_mag(sd, "label_emb.0.0", "label_emb.0.2", run.y, run.y.abs())
        return emb + lab, mag + m_lab

    def _emb_vectors(self, rt, L):
        run = self._runs.get(id(rt))
        if run is None or not run.check_layers:
            return
        p, rb = L["spec"].prefix, L["spec"]
        dev = run.emb.device
        s = F.silu(run.emb)
        K = s.shape[1]
        sd = self.sd["unet"][1]
        up = EMB_UP_ROUNDINGS * U16 + 2 * _acc(K)
        for key, q in (("emb_off", f"{p}.emb_layers.1"), ("embt_off", f"{p}.time_stack.emb_layers.1")):
            wt, b = sd[f"{q}.weight"].to(dev, torch.float64), sd[f"{q}.bias"].to(dev, torch.float64)
            ref = F.linear(s, wt, b)
            got = rt.emb_out[:, L[key]:L[key] + rb.cout]
            tol = (ulp(ref, torch.float32) + (EMB_ROUNDINGS * U16 + _acc(K)) * (s.abs() @ wt.abs().t() + b.abs())
                   + 1.1 * up * (run.emb_mag @ wt.abs().t()))
            self._elements(f"{q} (emb_out)", got, ref, tol)

    def _attn2_ref(self, sd, a, ctx, C, heads, D):
        """The oracle's single-key cross-attention on ctx (B, 1, D + A) and its magnitude chain."""
        ref = vo.attention(sd, a, torch.zeros(ctx.shape[0], 1, C, dtype=torch.float64, device=ctx.device), heads, ctx, D)[:, 0]
        c, act = ctx[:, 0, :D].abs(), ctx[:, 0, D:].abs()
        v = c @ sd[f"{a}.to_v.weight"].abs().t()
        if f"{a}.v_adapter_action_control.weight" in sd:
            v = v + act @ sd[f"{a}.v_adapter_action_control.weight"].abs().t()
        mag = v @ sd[f"{a}.to_out.0.weight"].abs().t() + sd[f"{a}.to_out.0.bias"].abs()
        return ref, mag, ctx.shape[-1]

    def _svt_vectors(self, rt, L):
        run = self._runs.get(id(rt))
        if run is None or not run.check_layers or getattr(run, "vec_done_" + L["spec"].prefix, False):
            return
        t, T = L["spec"], rt.T
        p, dev, D = t.prefix, run.ctx.device, rt.cfg.context_dim
        sd = self._sdl("unet", p, dev)
        with torch.no_grad():
            for name, a, ctx in (("sp", f"{p}.transformer_blocks.0.attn2", run.ctx),
                                 ("tm", f"{p}.time_stack.0.attn2", run.ctx[::T])):
                ref, mag, K = self._attn2_ref(sd, a, ctx, t.ch, t.heads, D)
                tol = ulp(ref, torch.float32) + (ATTN2_ROUNDINGS * U16 + 3 * _acc(K)) * mag
                self._elements(f"{p} cond[{name!r}]", rt.cond[name][p][:ctx.shape[0], :t.ch], ref, tol)
            temb = vo.timestep_embedding(torch.arange(T, dtype=torch.float64), t.ch).to(dev, torch.float64)
            ref, mag = self._mlp_mag(sd, f"{p}.time_pos_embed.0", f"{p}.time_pos_embed.2", temb, temb.abs())
            tol = ulp(ref, torch.float32) + (POS_ROUNDINGS * U16 + 2 * _acc(4 * t.ch)) * mag
            self._elements(f"{p} cond['pos']", rt.cond["pos"][p][:T, :t.ch], ref, tol)
        setattr(run, "vec_done_" + p, True)

    # ------------------------------------------------------------------ heads
    def _unet_head(self, run, head, x, net):
        B, h, w = run.geom["net.in"]
        sd = {k: v.to(x.device, torch.float64) for k, v in self.sd["unet"][1].items() if k.startswith("out.")}
        T = run.rt.T
        parts = Parts()
        C = head.inputs[0][2]
        with torch.no_grad():
            for c in range(B // T):
                rows = slice(c * T * h * w, (c + 1) * T * h * w)
                hh = F.silu(vo._gn(sd, "out.0", nchw(x[rows], T, h, w, C), 1e-5))
                ref = F.conv2d(hh, sd["out.2.weight"], sd["out.2.bias"], padding=1)
                parts.add(nchw(net[rows], T, h, w, head.cout), ref, c * T)
        self._note("out", head.kind, (B * h * w, head.cout), parts)
        self.checked["unet"].add("out")

    def _dec_head(self, run, head, x, A):
        T, h, w = run.geom[head.inputs[0][0]]
        sd = {k: v.to(x.device, torch.float64) for k, v in self.sd["dec"][1].items()
              if k.startswith("norm_out.") or k.startswith("conv_out.")}
        blend, skip, out_u8, keep = A["blend"], A["skip_frames"], A["out_u8"], A["keep_f32_from"]
        frames = [t for t in range(skip, T) if (blend is None or int(blend[t]) == 0)
                  and (out_u8 is None or keep < 0 or t >= keep)]
        if not frames:
            return
        C = head.inputs[0][2]
        with torch.no_grad():
            ref = decoder_head_pieces(sd, lambda f: nchw(x[f * h * w:(f + 1) * h * w], 1, h, w, C), T)
            parts = Parts()
            for t in frames:
                parts.add(A["out"][A["out_frame0"] + t][None].double(), ref[t:t + 1], t)
        self._note("dec:out", head.kind, (len(frames),) + tuple(ref.shape[1:]), parts)
        self.checked["dec"].add("out")

    def _enc_head(self, run, head, x, mom):
        n, h, w = run.geom[head.inputs[0][0]]
        cfg, sd_all, post = self.sd["enc"][0], self.sd["enc"][1], self.sd["enc"][2]
        sd = {k: v.to(x.device, torch.float64) for k, v in sd_all.items()
              if k.startswith("norm_out.") or k.startswith("conv_out.")}
        with torch.no_grad():
            hh = vo._swish(vo._gn(sd, "norm_out", nchw(x, n, h, w, head.inputs[0][2]), 1e-6))
            ref = F.conv2d(hh, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)
            if post is not None:
                pw, pb = (t.to(x.device, torch.float64) for t in post)
                ref = F.conv2d(ref, pw.reshape(pw.shape[0], -1, 1, 1), pb)
            parts = Parts()
            parts.add(nchw(mom, n, h, w, ref.shape[1]), ref)
        self._note("enc:out", head.kind, (n * h * w, ref.shape[1]), parts)
        self.checked["enc"].add("out")

    # ------------------------------------------------------------------ results
    @staticmethod
    def label(net, name):
        """Census / failure name of a layer: the UNet's prefixes as they are, the VAE's under dec: / enc:."""
        return name if net == "unet" else f"{net}:{name}"

    def coverage(self):
        """Every layer and segment of every network that ran was checked; the names of the rest."""
        missing = []
        for net in sorted(self.ran):
            cfg = self.sd[net][0]
            nodes = (unet_graph(unet_mod.build_unet_plan(cfg)) if net == "unet" else
                     decoder_graph(cfg) if net == "dec" else encoder_graph(cfg))
            missing += [self.label(net, n) for n in nodes if n not in self.checked[net]]
        return missing

    def assert_ok(self):
        missing = self.coverage()
        if missing:
            self._fail(("coverage",), f"layers / segments never checked: {missing}")
        assert not self.failures, f"{len(self.failures)} block check(s) failed:\n" + "\n".join(self.failures.values())

    def worst_by_kind(self):
        out = {}
        for e in self.census.values():
            out[e.kind] = max(out.get(e.kind, 0.0), e.ratio)
        return out

    def worst_gain_by_kind(self):
        """kind -> (worst |beta| / (B + 4 sigma), its layer, its term) over the layers the gain check ran on."""
        out = {}
        for name, e in self.census.items():
            if e.gain_term is not None and e.gain >= out.get(e.kind, (-1.0,))[0]:
                out[e.kind] = (e.gain, name, e.gain_term)
        return out

    def report(self) -> str:
        lines = [f"{'layer':<44}{'kind':<15}{'shape':<18}{'worst ratio':>12}  partition / worst gain term"]
        for name, e in self.census.items():
            lines.append(f"{name:<44}{e.kind:<15}{str(e.shape):<18}{e.ratio:>12.3f}  {e.part}"
                         + ("" if e.gain_term is None else f" / {e.gain_term!r}"))
        lines.append("worst ratio per kind (rel-L2 / (c_kind rho)): " +
                     ", ".join(f"{k} {v:.3f} (c {C_KIND[k]:.2f})" for k, v in sorted(self.worst_by_kind().items())))
        lines.append("worst gain per kind (|beta| / (B + 4 sigma)): " +
                     ", ".join(f"{k} {g:.3f} ({n}: {t!r})" for k, (g, n, t) in sorted(self.worst_gain_by_kind().items())))
        if self.vectors:
            lines.append(f"conditioning vectors: {len(self.vectors)} checked, worst error / element bound "
                         f"{max(self.vectors.values()):.3f}")
        lines.append(f"{len(self.census)} layers / segments, {self.handoffs} hand-offs, {len(self.failures)} failing")
        return "\n".join(lines)
