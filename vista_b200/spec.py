"""Architecture plan + parameter inventory of the Vista denoising hot path.

This module is the single place that knows *what layers exist*, in which order, and
which ``state_dict`` keys / shapes they own.  It is pure Python (no torch) so that the
oracle, the synthetic-weight generator, the B200 executor and the tests all share it.

Reference behaviour followed (paths relative to the reference checkout):
  * UNet topology ............ vwm/modules/diffusionmodules/video_model.py:186-440
  * VideoResBlock ............ vwm/modules/diffusionmodules/video_model.py:9-75,
                               vwm/modules/diffusionmodules/openaimodel.py:146-284
  * SpatialVideoTransformer .. vwm/modules/video_attention.py:147-296,
                               vwm/modules/attention.py:246-324,424-490,527-609
  * VideoDecoder ............. vwm/modules/diffusionmodules/model.py:560-694,
                               vwm/modules/autoencoding/temporal_ae.py:11-151
Key naming follows SURVEY.md Appendix D (what ``load_state_dict`` must accept).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

ACTION_DIM = 128 * 19  # vwm/modules/attention.py:321


# --------------------------------------------------------------------------------------
# configs
# --------------------------------------------------------------------------------------
@dataclass
class UNetConfig:
    """Constructor arguments of the reference ``VideoUNet`` that matter at inference
    (configs/inference/vista.yaml:19-40)."""
    in_channels: int = 8
    out_channels: int = 4
    model_channels: int = 320
    attention_resolutions: Sequence[int] = (4, 2, 1)
    num_res_blocks: int = 2
    channel_mult: Sequence[int] = (1, 2, 4, 4)
    num_head_channels: int = 64
    context_dim: int = 1024
    adm_in_channels: int = 768
    transformer_depth: int = 1
    action_control: bool = True
    num_groups: int = 32

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4


@dataclass
class DecoderConfig:
    """``VideoDecoder`` arguments (configs/inference/vista.yaml:170-184)."""
    ch: int = 128
    out_ch: int = 3
    ch_mult: Sequence[int] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    num_groups: int = 32


@dataclass
class EncoderConfig:
    """``Encoder`` arguments (configs/inference/vista.yaml:155-168); SURVEY.md §8f rank 1 (next row)."""
    ch: int = 128
    in_channels: int = 3
    ch_mult: Sequence[int] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    double_z: bool = True
    num_groups: int = 32


VISTA_UNET = UNetConfig()
VISTA_DECODER = DecoderConfig()
VISTA_ENCODER = EncoderConfig()


# --------------------------------------------------------------------------------------
# layer descriptors (the "plan")
# --------------------------------------------------------------------------------------
@dataclass
class ResBlockSpec:
    prefix: str
    cin: int
    cout: int

    @property
    def has_skip(self) -> bool:
        return self.cin != self.cout


@dataclass
class SVTSpec:
    """SpatialVideoTransformer with depth 1 (one spatial + one temporal block)."""
    prefix: str
    ch: int
    heads: int
    d_head: int


@dataclass
class ConvSpec:
    prefix: str          # key prefix of the conv (".weight"/".bias" appended)
    cin: int
    cout: int
    kind: str            # "conv_in" | "down" | "up"


@dataclass
class UNetBlock:
    """One ``TimestepEmbedSequential`` entry."""
    name: str
    layers: List[object] = field(default_factory=list)


@dataclass
class UNetPlan:
    cfg: UNetConfig
    input_blocks: List[UNetBlock]
    middle_block: UNetBlock
    output_blocks: List[UNetBlock]
    skip_channels: List[int]      # channels pushed on `hs` by every input block

    def all_layers(self):
        for blk in self.input_blocks + [self.middle_block] + self.output_blocks:
            for layer in blk.layers:
                yield layer

    def res_blocks(self) -> List[ResBlockSpec]:
        return [l for l in self.all_layers() if isinstance(l, ResBlockSpec)]

    def transformers(self) -> List[SVTSpec]:
        return [l for l in self.all_layers() if isinstance(l, SVTSpec)]


def build_unet_plan(cfg: UNetConfig = VISTA_UNET) -> UNetPlan:
    """Walk the constructor logic of video_model.py:186-433 and record the layers."""
    mc = cfg.model_channels
    input_blocks = [UNetBlock("input_blocks.0",
                              [ConvSpec("input_blocks.0.0", cfg.in_channels, mc, "conv_in")])]
    chans = [mc]
    ch, ds = mc, 1
    idx = 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            name = f"input_blocks.{idx}"
            layers: List[object] = [ResBlockSpec(f"{name}.0", ch, mult * mc)]
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                layers.append(SVTSpec(f"{name}.1", ch, ch // cfg.num_head_channels, cfg.num_head_channels))
            input_blocks.append(UNetBlock(name, layers))
            chans.append(ch)
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            name = f"input_blocks.{idx}"
            input_blocks.append(UNetBlock(name, [ConvSpec(f"{name}.0.op", ch, ch, "down")]))
            chans.append(ch)
            ds *= 2
            idx += 1
    skip_channels = list(chans)

    heads = ch // cfg.num_head_channels
    middle = UNetBlock("middle_block", [
        ResBlockSpec("middle_block.0", ch, ch),
        SVTSpec("middle_block.1", ch, heads, cfg.num_head_channels),
        ResBlockSpec("middle_block.2", ch, ch),
    ])

    output_blocks = []
    oidx = 0
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks + 1):
            ich = chans.pop()
            name = f"output_blocks.{oidx}"
            layers = [ResBlockSpec(f"{name}.0", ch + ich, mc * mult)]
            ch = mc * mult
            if ds in cfg.attention_resolutions:
                layers.append(SVTSpec(f"{name}.{len(layers)}", ch, ch // cfg.num_head_channels,
                                      cfg.num_head_channels))
            if level and i == cfg.num_res_blocks:
                layers.append(ConvSpec(f"{name}.{len(layers)}.conv", ch, ch, "up"))
                ds //= 2
            output_blocks.append(UNetBlock(name, layers))
            oidx += 1
    return UNetPlan(cfg, input_blocks, middle, output_blocks, skip_channels)


# --------------------------------------------------------------------------------------
# parameter inventory
# --------------------------------------------------------------------------------------
# init kinds: "w" fan-in scaled weight, "wz" weight the reference zero-initialises,
# "b" bias, "g" norm gain (around 1), "mix" AlphaBlender logit
ParamSpec = Tuple[Tuple[int, ...], str]


def _lin(out: Dict[str, ParamSpec], p: str, cin: int, cout: int, bias: bool = True, zero: bool = False):
    out[f"{p}.weight"] = ((cout, cin), "wz" if zero else "w")
    if bias:
        out[f"{p}.bias"] = ((cout,), "b")


def _norm(out, p: str, c: int):
    out[f"{p}.weight"] = ((c,), "g")
    out[f"{p}.bias"] = ((c,), "b")


def _conv(out, p: str, cin: int, cout: int, k: Tuple[int, ...], zero: bool = False):
    out[f"{p}.weight"] = ((cout, cin) + tuple(k), "wz" if zero else "w")
    out[f"{p}.bias"] = ((cout,), "b")


def _resblock_params(out, rb: ResBlockSpec, emb_dim: int):
    p = rb.prefix
    _norm(out, f"{p}.in_layers.0", rb.cin)
    _conv(out, f"{p}.in_layers.2", rb.cin, rb.cout, (3, 3))
    _lin(out, f"{p}.emb_layers.1", emb_dim, rb.cout)
    _norm(out, f"{p}.out_layers.0", rb.cout)
    _conv(out, f"{p}.out_layers.3", rb.cout, rb.cout, (3, 3), zero=True)
    if rb.has_skip:
        _conv(out, f"{p}.skip_connection", rb.cin, rb.cout, (1, 1))
    t = f"{p}.time_stack"
    _norm(out, f"{t}.in_layers.0", rb.cout)
    _conv(out, f"{t}.in_layers.2", rb.cout, rb.cout, (3, 1, 1))
    _lin(out, f"{t}.emb_layers.1", emb_dim, rb.cout)
    _norm(out, f"{t}.out_layers.0", rb.cout)
    _conv(out, f"{t}.out_layers.3", rb.cout, rb.cout, (3, 1, 1), zero=True)
    out[f"{p}.time_mixer.mix_factor"] = ((1,), "mix")


def _attn_params(out, p: str, c: int, ctx: Optional[int], action: bool):
    kdim = c if ctx is None else ctx
    _lin(out, f"{p}.to_q", c, c, bias=False)
    _lin(out, f"{p}.to_k", kdim, c, bias=False)
    _lin(out, f"{p}.to_v", kdim, c, bias=False)
    _lin(out, f"{p}.to_out.0", c, c)
    if action:
        _lin(out, f"{p}.k_adapter_action_control", ACTION_DIM, c, bias=False, zero=True)
        _lin(out, f"{p}.v_adapter_action_control", ACTION_DIM, c, bias=False, zero=True)


def _ff_params(out, p: str, c: int):
    _lin(out, f"{p}.net.0.proj", c, 8 * c)
    _lin(out, f"{p}.net.2", 4 * c, c)


def _svt_params(out, t: SVTSpec, cfg: UNetConfig):
    p, c = t.prefix, t.ch
    _norm(out, f"{p}.norm", c)
    _lin(out, f"{p}.proj_in", c, c)
    s = f"{p}.transformer_blocks.0"
    _attn_params(out, f"{s}.attn1", c, None, False)
    _ff_params(out, f"{s}.ff", c)
    _attn_params(out, f"{s}.attn2", c, cfg.context_dim, cfg.action_control)
    for n in ("norm1", "norm2", "norm3"):
        _norm(out, f"{s}.{n}", c)
    m = f"{p}.time_stack.0"
    _norm(out, f"{m}.norm_in", c)
    _ff_params(out, f"{m}.ff_in", c)
    _attn_params(out, f"{m}.attn1", c, None, False)
    _ff_params(out, f"{m}.ff", c)
    _norm(out, f"{m}.norm2", c)
    _attn_params(out, f"{m}.attn2", c, cfg.context_dim, cfg.action_control)
    _norm(out, f"{m}.norm1", c)
    _norm(out, f"{m}.norm3", c)
    _lin(out, f"{p}.time_pos_embed.0", c, 4 * c)
    _lin(out, f"{p}.time_pos_embed.2", 4 * c, c)
    out[f"{p}.time_mixer.mix_factor"] = ((1,), "mix")
    _lin(out, f"{p}.proj_out", c, c, zero=True)


def unet_param_specs(cfg: UNetConfig = VISTA_UNET) -> Dict[str, ParamSpec]:
    """name -> (shape, init kind) for every tensor in ``VideoUNet.state_dict()``."""
    plan = build_unet_plan(cfg)
    out: Dict[str, ParamSpec] = {}
    mc, ed = cfg.model_channels, cfg.time_embed_dim
    for name in ("time_embed", "cond_time_stack_embed"):
        _lin(out, f"{name}.0", mc, ed)
        _lin(out, f"{name}.2", ed, ed)
    _lin(out, "label_emb.0.0", cfg.adm_in_channels, ed)
    _lin(out, "label_emb.0.2", ed, ed)
    for layer in plan.all_layers():
        if isinstance(layer, ResBlockSpec):
            _resblock_params(out, layer, ed)
        elif isinstance(layer, SVTSpec):
            _svt_params(out, layer, cfg)
        elif isinstance(layer, ConvSpec):
            _conv(out, layer.prefix, layer.cin, layer.cout, (3, 3))
    _norm(out, "out.0", mc)
    _conv(out, "out.2", mc, cfg.out_channels, (3, 3), zero=True)
    return out


# ---- VAE decoder ---------------------------------------------------------------------
@dataclass
class DecResBlockSpec:
    prefix: str
    cin: int
    cout: int

    @property
    def has_skip(self) -> bool:
        return self.cin != self.cout


@dataclass
class DecoderPlan:
    cfg: DecoderConfig
    block_in: int
    mid: List[DecResBlockSpec]
    # per level, highest index first (execution order): (resblocks, upsample-conv prefix or None, channels)
    levels: List[Tuple[List[DecResBlockSpec], Optional[str], int]]
    final_ch: int


def build_decoder_plan(cfg: DecoderConfig = VISTA_DECODER) -> DecoderPlan:
    """model.py:591-647: mid (res, attn, res) then levels from coarsest to finest."""
    nres = len(cfg.ch_mult)
    block_in = cfg.ch * cfg.ch_mult[nres - 1]
    mid = [DecResBlockSpec("mid.block_1", block_in, block_in),
           DecResBlockSpec("mid.block_2", block_in, block_in)]
    levels = []
    cur = block_in
    for i_level in reversed(range(nres)):
        block_out = cfg.ch * cfg.ch_mult[i_level]
        blocks = []
        for i_block in range(cfg.num_res_blocks + 1):
            blocks.append(DecResBlockSpec(f"up.{i_level}.block.{i_block}", cur, block_out))
            cur = block_out
        up = f"up.{i_level}.upsample.conv" if i_level != 0 else None
        levels.append((blocks, up, cur))
    return DecoderPlan(cfg, block_in, mid, levels, cur)


def _dec_resblock_params(out, rb: DecResBlockSpec):
    p = rb.prefix
    _norm(out, f"{p}.norm1", rb.cin)
    _conv(out, f"{p}.conv1", rb.cin, rb.cout, (3, 3))
    _norm(out, f"{p}.norm2", rb.cout)
    _conv(out, f"{p}.conv2", rb.cout, rb.cout, (3, 3))
    if rb.has_skip:
        _conv(out, f"{p}.nin_shortcut", rb.cin, rb.cout, (1, 1))
    t = f"{p}.time_stack"
    _norm(out, f"{t}.in_layers.0", rb.cout)
    _conv(out, f"{t}.in_layers.2", rb.cout, rb.cout, (3, 1, 1))
    _norm(out, f"{t}.out_layers.0", rb.cout)
    _conv(out, f"{t}.out_layers.3", rb.cout, rb.cout, (3, 1, 1), zero=True)
    out[f"{p}.mix_factor"] = ((1,), "mix0")


def decoder_param_specs(cfg: DecoderConfig = VISTA_DECODER) -> Dict[str, ParamSpec]:
    """name -> (shape, kind) for ``VideoDecoder.state_dict()`` (keys relative to the decoder)."""
    plan = build_decoder_plan(cfg)
    out: Dict[str, ParamSpec] = {}
    _conv(out, "conv_in", cfg.z_channels, plan.block_in, (3, 3))
    _dec_resblock_params(out, plan.mid[0])
    a = "mid.attn_1"
    _norm(out, f"{a}.norm", plan.block_in)
    for n in ("q", "k", "v", "proj_out"):
        _conv(out, f"{a}.{n}", plan.block_in, plan.block_in, (1, 1))
    _dec_resblock_params(out, plan.mid[1])
    for blocks, up, ch in plan.levels:
        for rb in blocks:
            _dec_resblock_params(out, rb)
        if up is not None:
            _conv(out, up, ch, ch, (3, 3))
    _norm(out, "norm_out", plan.final_ch)
    _conv(out, "conv_out", plan.final_ch, cfg.out_ch, (3, 3))
    _conv(out, "conv_out.time_mix_conv", cfg.out_ch, cfg.out_ch, (3, 1, 1))
    return out


# ---- VAE encoder (2-D, per frame) ----------------------------------------------------
def build_encoder_plan(cfg: EncoderConfig = VISTA_ENCODER):
    """model.py:476-523: per level the ResnetBlocks (prefix, cin, cout) and the Downsample conv prefix (or None);
    then the mid channel count."""
    levels = []
    in_ch_mult = (1,) + tuple(cfg.ch_mult)
    block_in = cfg.ch
    for i_level in range(len(cfg.ch_mult)):
        block_in = cfg.ch * in_ch_mult[i_level]
        block_out = cfg.ch * cfg.ch_mult[i_level]
        blocks = []
        for i_block in range(cfg.num_res_blocks):
            blocks.append(DecResBlockSpec(f"down.{i_level}.block.{i_block}", block_in, block_out))
            block_in = block_out
        down = f"down.{i_level}.downsample.conv" if i_level != len(cfg.ch_mult) - 1 else None
        levels.append((blocks, down, block_in))
    return levels, block_in


def _enc_resblock_params(out, rb: DecResBlockSpec):
    p = rb.prefix
    _norm(out, f"{p}.norm1", rb.cin)
    _conv(out, f"{p}.conv1", rb.cin, rb.cout, (3, 3))
    _norm(out, f"{p}.norm2", rb.cout)
    _conv(out, f"{p}.conv2", rb.cout, rb.cout, (3, 3))
    if rb.has_skip:
        _conv(out, f"{p}.nin_shortcut", rb.cin, rb.cout, (1, 1))


def encoder_param_specs(cfg: EncoderConfig = VISTA_ENCODER) -> Dict[str, ParamSpec]:
    """name -> (shape, kind) for ``Encoder.state_dict()`` (keys relative to the encoder)."""
    levels, mid_ch = build_encoder_plan(cfg)
    out: Dict[str, ParamSpec] = {}
    _conv(out, "conv_in", cfg.in_channels, cfg.ch, (3, 3))
    for blocks, down, ch in levels:
        for rb in blocks:
            _enc_resblock_params(out, rb)
        if down is not None:
            _conv(out, down, ch, ch, (3, 3))
    _enc_resblock_params(out, DecResBlockSpec("mid.block_1", mid_ch, mid_ch))
    a = "mid.attn_1"
    _norm(out, f"{a}.norm", mid_ch)
    for n in ("q", "k", "v", "proj_out"):
        _conv(out, f"{a}.{n}", mid_ch, mid_ch, (1, 1))
    _enc_resblock_params(out, DecResBlockSpec("mid.block_2", mid_ch, mid_ch))
    _norm(out, "norm_out", mid_ch)
    _conv(out, "conv_out", mid_ch, (2 if cfg.double_z else 1) * cfg.z_channels, (3, 3))
    return out


# --------------------------------------------------------------------------------------
# CLIP image tower of the conditioner (open_clip VisionTransformer under FrozenOpenCLIPImageEmbedder,
# vwm/modules/encoders/modules.py:251-399; configs/inference/vista.yaml:44-52)
# --------------------------------------------------------------------------------------
@dataclass
class ClipConfig:
    """open_clip ``VisionTransformer`` shape.  The native tower needs head width 80 (b200v_attention_d80), a LayerNorm
    width b200v_layernorm supports and widths that are multiples of 64 (the tap-GEMM's K granularity)."""
    width: int = 1280
    layers: int = 32
    head_width: int = 80
    patch_size: int = 14
    image_size: int = 224
    mlp_ratio: float = 4.0
    embed_dim: int = 1024
    ln_eps: float = 1e-5

    @property
    def heads(self) -> int:
        return self.width // self.head_width

    @property
    def mlp_width(self) -> int:
        return int(self.width * self.mlp_ratio)

    @property
    def grid(self) -> int:
        return self.image_size // self.patch_size

    @property
    def tokens(self) -> int:          # class token + patches
        return self.grid * self.grid + 1

    @property
    def patch_k(self) -> int:         # 3 * 14 * 14 = 588
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_k_pad(self) -> int:     # padded to the GEMM's 64-column K chunks
        return -(-self.patch_k // 64) * 64


VIT_H_14 = ClipConfig()

# what survives ``del model.transformer`` of the open_clip CLIP model besides ``visual`` (modules.py:277): the text
# tower's leftovers, accepted by load_state_dict and ignored
CLIP_TEXT_LEFTOVERS = ("token_embedding.weight", "positional_embedding", "ln_final.weight", "ln_final.bias",
                       "text_projection", "logit_scale")


def clip_param_specs(cfg: ClipConfig = VIT_H_14) -> Dict[str, ParamSpec]:
    """name -> (shape, kind) for open_clip's ``model.visual`` (keys relative to ``visual``)."""
    C, out = cfg.width, {}
    out["class_embedding"] = ((C,), "b")
    out["positional_embedding"] = ((cfg.tokens, C), "b")
    out["proj"] = ((C, cfg.embed_dim), "w")
    out["conv1.weight"] = ((C, 3, cfg.patch_size, cfg.patch_size), "w")
    _norm(out, "ln_pre", C)
    for i in range(cfg.layers):
        p = f"transformer.resblocks.{i}"
        _norm(out, f"{p}.ln_1", C)
        out[f"{p}.attn.in_proj_weight"] = ((3 * C, C), "w")
        out[f"{p}.attn.in_proj_bias"] = ((3 * C,), "b")
        _lin(out, f"{p}.attn.out_proj", C, C)
        _norm(out, f"{p}.ln_2", C)
        _lin(out, f"{p}.mlp.c_fc", C, cfg.mlp_width)
        _lin(out, f"{p}.mlp.c_proj", cfg.mlp_width, C)
    _norm(out, "ln_post", C)
    return out


def clip_preset(name: str) -> ClipConfig:
    if name == "vit_h_14":
        return ClipConfig()
    if name == "tiny":    # head width 80 kept (the attention kernel), 4 heads, 2 layers, same 1024-wide embedding
        return ClipConfig(width=320, layers=2)
    raise KeyError(name)


# --------------------------------------------------------------------------------------
# presets used by tests / oracle / bench
# --------------------------------------------------------------------------------------
def unet_preset(name: str) -> UNetConfig:
    if name == "vista":
        return UNetConfig()
    if name == "small":   # same topology, 64-wide: heads 1/2/4/4, ~66 M params
        return UNetConfig(model_channels=64)
    if name == "tiny":    # two levels, one res block per level: fast CPU oracle
        return UNetConfig(model_channels=64, channel_mult=(1, 2), num_res_blocks=1,
                          attention_resolutions=(1, 2))
    raise KeyError(name)


def decoder_preset(name: str) -> DecoderConfig:
    if name == "vista":
        return DecoderConfig()
    if name == "small":
        return DecoderConfig(ch=64)
    if name == "tiny":
        return DecoderConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1)
    raise KeyError(name)


def encoder_preset(name: str) -> EncoderConfig:
    if name == "vista":
        return EncoderConfig()
    if name == "small":
        return EncoderConfig(ch=64)
    if name == "tiny":
        return EncoderConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1)
    raise KeyError(name)
