"""TEST INFRASTRUCTURE — CPU restatement (fp32, plain torch functional ops) of the reference's
iterative-denoising hot path.  It is the checker for the CUDA path; it is never shipped, never
measured as the product and never used as a fallback.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s baseline legs (cpu_baseline, ``--impl reference``, and the eager-GPU
denominator ``gpu_eager_baseline``, where it runs on ``cuda`` as the stated port of the reference's eager path) import it.

Pinned: ``tests/test_oracle_golden.py`` compares every function below with outputs of the real
reference modules (generated in the build container by ``oracle/make_golden.py`` and committed
under ``tests/golden/``) and with the closed-form anchors of SURVEY.md §8c.

Each function cites the reference file:line it follows (paths relative to the reference root).
Weights come as a flat ``dict[str, Tensor]`` with the reference's state_dict key names.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from vista_b200.spec import (ConvSpec, DecoderConfig, ResBlockSpec, SVTSpec, UNetConfig,
                             build_decoder_plan, build_unet_plan)

SD = Dict[str, torch.Tensor]


# ---------------------------------------------------------------------------------------------
# small pieces
# ---------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """vwm/modules/diffusionmodules/util.py:141-165 — cos||sin, freqs = exp(-ln(P) k / half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat((torch.cos(args), torch.sin(args)), dim=-1)
    if dim % 2:
        emb = torch.cat((emb, torch.zeros_like(emb[:, :1])), dim=-1)
    return emb


def _lin(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, sd[f"{p}.weight"], sd.get(f"{p}.bias"))


def _mlp(sd: SD, p0: str, p2: str, x: torch.Tensor) -> torch.Tensor:
    """Linear -> SiLU -> Linear (video_model.py:148-157,176-182; video_attention.py:227-231)."""
    return _lin(sd, p2, F.silu(_lin(sd, p0, x)))


def _gn(sd: SD, p: str, x: torch.Tensor, eps: float, groups: int = 32) -> torch.Tensor:
    return F.group_norm(x, groups, sd[f"{p}.weight"], sd[f"{p}.bias"], eps)


def _ln(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[f"{p}.weight"], sd[f"{p}.bias"], 1e-5)


# ---------------------------------------------------------------------------------------------
# VideoResBlock
# ---------------------------------------------------------------------------------------------
def res_block_2d(sd: SD, p: str, x: torch.Tensor, emb: torch.Tensor, has_skip: bool, record: Optional[dict] = None
                 ) -> torch.Tensor:
    """openaimodel.py:258-284 with dims=2, no up/down, no scale-shift norm. GroupNorm32 eps 1e-5.  ``record``: receives
    the residual operand as "res2d" (test aid; the arithmetic is the same with or without it)."""
    h = F.conv2d(F.silu(_gn(sd, f"{p}.in_layers.0", x, 1e-5)),
                 sd[f"{p}.in_layers.2.weight"], sd[f"{p}.in_layers.2.bias"], padding=1)
    emb_out = _lin(sd, f"{p}.emb_layers.1", F.silu(emb))
    h = h + emb_out[:, :, None, None]
    h = F.conv2d(F.silu(_gn(sd, f"{p}.out_layers.0", h, 1e-5)),
                 sd[f"{p}.out_layers.3.weight"], sd[f"{p}.out_layers.3.bias"], padding=1)
    if has_skip:
        x = F.conv2d(x, sd[f"{p}.skip_connection.weight"], sd[f"{p}.skip_connection.bias"])
    if record is not None:
        record["res2d"] = x
    return x + h


def res_block_3d(sd: SD, p: str, x: torch.Tensor, emb: Optional[torch.Tensor]) -> torch.Tensor:
    """openaimodel.py:258-284 with dims=3, kernel (3,1,1), exchange_temb_dims (video_model.py:38-52)
    or skip_t_emb (temporal_ae.py:25-37).  x: (b, c, t, h, w); emb: (b, t, E) or None.
    GroupNorm statistics run over (C/32, T, H, W)."""
    h = F.conv3d(F.silu(_gn(sd, f"{p}.in_layers.0", x, 1e-5)),
                 sd[f"{p}.in_layers.2.weight"], sd[f"{p}.in_layers.2.bias"], padding=(1, 0, 0))
    if emb is not None:
        emb_out = _lin(sd, f"{p}.emb_layers.1", F.silu(emb))          # (b, t, c)
        h = h + emb_out.permute(0, 2, 1)[:, :, :, None, None]         # b c t 1 1
    h = F.conv3d(F.silu(_gn(sd, f"{p}.out_layers.0", h, 1e-5)),
                 sd[f"{p}.out_layers.3.weight"], sd[f"{p}.out_layers.3.bias"], padding=(1, 0, 0))
    return x + h


def video_res_block(sd: SD, rb: ResBlockSpec, x: torch.Tensor, emb: torch.Tensor, T: int,
                    record: Optional[dict] = None) -> torch.Tensor:
    """video_model.py:59-75; blend util.py:311-318: alpha*spatial + (1-alpha)*temporal.

    ``record`` (test aid, tests/block_shadow.py): receives every operand added as a residual ("res2d", the spatial
    block's; "res3d", the temporal block's) and the blend as "blend" = (alpha, a, b) with out = alpha a + (1 - alpha) b,
    all in the output's (bt, c, h, w) layout.  The arithmetic is the same with or without it."""
    x = res_block_2d(sd, rb.prefix, x, emb, rb.has_skip, record)
    bt, c, h, w = x.shape
    x5 = x.reshape(bt // T, T, c, h, w).permute(0, 2, 1, 3, 4)
    xt = res_block_3d(sd, f"{rb.prefix}.time_stack", x5, emb.reshape(bt // T, T, -1))
    alpha = torch.sigmoid(sd[f"{rb.prefix}.time_mixer.mix_factor"])
    out = alpha * x5 + (1.0 - alpha) * xt
    if record is not None:
        record["res3d"] = x
        record["blend"] = (alpha, x, xt.permute(0, 2, 1, 3, 4).reshape(bt, c, h, w))
    return out.permute(0, 2, 1, 3, 4).reshape(bt, c, h, w)


# ---------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------
def _heads(x: torch.Tensor, h: int) -> torch.Tensor:
    b, n, c = x.shape
    return x.reshape(b, n, h, c // h).permute(0, 2, 1, 3)


def attention(sd: SD, p: str, x: torch.Tensor, heads: int, context: Optional[torch.Tensor],
              ctx_dim: Optional[int]) -> torch.Tensor:
    """attention.py:326-421 (MemoryEfficientCrossAttention).  xformers' kernel == softmax(QK^T/sqrt d)V.
    With action_control the context splits at ctx_dim and the adapters add to k, v (:342-353)."""
    q = F.linear(x, sd[f"{p}.to_q.weight"])
    if context is None:
        k = F.linear(x, sd[f"{p}.to_k.weight"])
        v = F.linear(x, sd[f"{p}.to_v.weight"])
    else:
        ctx, act = context[..., :ctx_dim], context[..., ctx_dim:]
        k = F.linear(ctx, sd[f"{p}.to_k.weight"])
        v = F.linear(ctx, sd[f"{p}.to_v.weight"])
        if f"{p}.k_adapter_action_control.weight" in sd:
            k = k + F.linear(act, sd[f"{p}.k_adapter_action_control.weight"])
            v = v + F.linear(act, sd[f"{p}.v_adapter_action_control.weight"])
    o = F.scaled_dot_product_attention(_heads(q, heads), _heads(k, heads), _heads(v, heads))
    b, _, n, _ = o.shape
    o = o.permute(0, 2, 1, 3).reshape(b, n, -1)
    return _lin(sd, f"{p}.to_out.0", o)


def feed_forward(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """attention.py:85-128: GEGLU (value = first half, gate = second half, exact-erf GELU) then Linear."""
    val, gate = _lin(sd, f"{p}.net.0.proj", x).chunk(2, dim=-1)
    return _lin(sd, f"{p}.net.2", val * F.gelu(gate))


def basic_transformer_block(sd: SD, p: str, x, context, heads, ctx_dim):
    """attention.py:514-524."""
    x = attention(sd, f"{p}.attn1", _ln(sd, f"{p}.norm1", x), heads, None, None) + x
    x = attention(sd, f"{p}.attn2", _ln(sd, f"{p}.norm2", x), heads, context, ctx_dim) + x
    x = feed_forward(sd, f"{p}.ff", _ln(sd, f"{p}.norm3", x)) + x
    return x


def video_transformer_block(sd: SD, p: str, x, time_context, heads, ctx_dim, T: int):
    """video_attention.py:111-141. x: ((b t), s, c) -> ((b s), t, c) and back."""
    B, S, C = x.shape
    b = B // T
    x = x.reshape(b, T, S, C).permute(0, 2, 1, 3).reshape(b * S, T, C)
    x = feed_forward(sd, f"{p}.ff_in", _ln(sd, f"{p}.norm_in", x)) + x
    x = attention(sd, f"{p}.attn1", _ln(sd, f"{p}.norm1", x), heads, None, None) + x
    x = attention(sd, f"{p}.attn2", _ln(sd, f"{p}.norm2", x), heads, time_context, ctx_dim) + x
    x = feed_forward(sd, f"{p}.ff", _ln(sd, f"{p}.norm3", x)) + x
    return x.reshape(b, S, T, C).permute(0, 2, 1, 3).reshape(B, S, C)


def spatial_video_transformer(sd: SD, t: SVTSpec, x: torch.Tensor, context: torch.Tensor,
                              T: int, ctx_dim: int, record: Optional[dict] = None) -> torch.Tensor:
    """video_attention.py:239-296 (use_linear, use_spatial_context, depth 1); GroupNorm eps 1e-6
    (attention.py:141-142).  ``record`` (test aid): receives the residual operand x_in as "res" and the blend as
    "blend" = (alpha, x, x_mix) in the inner (B, H W, C) layout, before proj_out.  The arithmetic is unchanged."""
    B, C, H, W = x.shape
    p = t.prefix
    x_in = x
    time_context = context[::T]                                     # :256
    time_context = time_context.repeat_interleave(H * W, dim=0)      # :257  (b n) ...
    x = _gn(sd, f"{p}.norm", x, 1e-6)
    x = x.permute(0, 2, 3, 1).reshape(B, H * W, C)
    x = _lin(sd, f"{p}.proj_in", x)
    frames = torch.arange(T).repeat(B // T)
    emb = _mlp(sd, f"{p}.time_pos_embed.0", f"{p}.time_pos_embed.2", timestep_embedding(frames, C))[:, None]
    x = basic_transformer_block(sd, f"{p}.transformer_blocks.0", x, context, t.heads, ctx_dim)
    x_mix = video_transformer_block(sd, f"{p}.time_stack.0", x + emb, time_context, t.heads, ctx_dim, T)
    alpha = torch.sigmoid(sd[f"{p}.time_mixer.mix_factor"])
    if record is not None:
        record["res"], record["blend"] = x_in, (alpha, x, x_mix)
    x = alpha * x + (1.0 - alpha) * x_mix                            # util.py:317
    x = _lin(sd, f"{p}.proj_out", x)
    x = x.reshape(B, H, W, C).permute(0, 3, 1, 2)
    return x + x_in


# ---------------------------------------------------------------------------------------------
# VideoUNet
# ---------------------------------------------------------------------------------------------
def unet_forward(sd: SD, cfg: UNetConfig, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor,
                 y: torch.Tensor, cond_mask: Optional[torch.Tensor], num_frames: int) -> torch.Tensor:
    """video_model.py:442-503.  x: (B, in_channels, h, w) with B = cfg_rows * num_frames."""
    plan = build_unet_plan(cfg)
    t_emb = timestep_embedding(timesteps, cfg.model_channels)
    if cond_mask is not None and bool(cond_mask.any()):
        m = cond_mask[..., None].float()
        emb = _mlp(sd, "cond_time_stack_embed.0", "cond_time_stack_embed.2", t_emb) * m \
            + _mlp(sd, "time_embed.0", "time_embed.2", t_emb) * (1 - m)
    else:
        emb = _mlp(sd, "time_embed.0", "time_embed.2", t_emb)
    emb = emb + _mlp(sd, "label_emb.0.0", "label_emb.0.2", y)

    def run(block, h):
        for layer in block.layers:
            if isinstance(layer, ResBlockSpec):
                h = video_res_block(sd, layer, h, emb, num_frames)
            elif isinstance(layer, SVTSpec):
                h = spatial_video_transformer(sd, layer, h, context, num_frames, cfg.context_dim)
            elif isinstance(layer, ConvSpec):
                wgt, b = sd[f"{layer.prefix}.weight"], sd[f"{layer.prefix}.bias"]
                if layer.kind == "down":            # openaimodel.py:129-136: stride 2, pad 1
                    h = F.conv2d(h, wgt, b, stride=2, padding=1)
                elif layer.kind == "up":            # openaimodel.py:100-102: nearest x2 then conv
                    h = F.conv2d(F.interpolate(h, scale_factor=2, mode="nearest"), wgt, b, padding=1)
                else:
                    h = F.conv2d(h, wgt, b, padding=1)
        return h

    hs = []
    h = x
    for blk in plan.input_blocks:
        h = run(blk, h)
        hs.append(h)
    h = run(plan.middle_block, h)
    for blk in plan.output_blocks:
        h = run(blk, torch.cat((h, hs.pop()), dim=1))
    h = F.silu(_gn(sd, "out.0", h, 1e-5))
    return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)


def wrapper_forward(sd, cfg, x, t, c: dict, cond_mask, num_frames):
    """wrappers.py:25-40 (OpenAIWrapper): concat c['concat'] along channels, unpack c."""
    concat = c["concat"]
    if concat.shape[0] != x.shape[0]:
        concat = concat.repeat_interleave(num_frames, dim=0)
    return unet_forward(sd, cfg, torch.cat((x, concat), dim=1), t, c["crossattn"], c["vector"],
                        cond_mask, num_frames)


# ---------------------------------------------------------------------------------------------
# diffusion mechanics
# ---------------------------------------------------------------------------------------------
def edm_sigmas(n: int, sigma_min=0.002, sigma_max=700.0, rho=7.0) -> torch.Tensor:
    """discretizer.py:32-37 + append_zero (:16-19). fp32 like torch.linspace default."""
    ramp = torch.linspace(0, 1, n)
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    sig = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
    return torch.cat((sig, sig.new_zeros([1])))


def vscaling_edm_cnoise(sigma: torch.Tensor):
    """denoiser_scaling.py:51-59."""
    c_skip = 1.0 / (sigma ** 2 + 1.0)
    c_out = -sigma / (sigma ** 2 + 1.0) ** 0.5
    c_in = 1.0 / (sigma ** 2 + 1.0) ** 0.5
    c_noise = 0.25 * sigma.log()
    return c_skip, c_out, c_in, c_noise


def denoise(sd, cfg, x, sigma, c, cond_mask, num_frames):
    """denoiser.py:22-35."""
    s = sigma[:, None, None, None]
    c_skip, c_out, c_in, c_noise = vscaling_edm_cnoise(s)
    net = wrapper_forward(sd, cfg, x * c_in, c_noise.reshape(sigma.shape), c, cond_mask, num_frames)
    return net * c_out + x * c_skip


def triangle_scales(num_frames=25, max_scale=2.5, min_scale=1.0, period=1.0) -> torch.Tensor:
    """guiders.py:87-118 with period_fusing='max' and a single period."""
    v = torch.linspace(0, 1, num_frames)
    tri = 2 * (v / period - torch.floor(v / period + 0.5)).abs()
    return tri * (max_scale - min_scale) + min_scale


def guider_scales(guider: str, num_frames: int, scale: float) -> torch.Tensor:
    if guider == "VanillaCFG":
        return torch.full((num_frames,), float(scale))
    if guider == "TrianglePredictionGuider":
        return triangle_scales(num_frames, max_scale=scale)
    if guider == "LinearPredictionGuider":
        return torch.linspace(1.0, scale, num_frames)   # guiders.py:61
    raise KeyError(guider)


def euler_edm_sample(sd, cfg, noise, c, uc, cond_frame, cond_mask, num_steps, num_frames=25,
                     guider="VanillaCFG", scale=2.5, return_all=False, stop_after=None):
    """sampling.py:91-124 (s_churn = 0 -> gamma = 0) + guiders.py:19-36 (batch [uncond; cond]).
    stop_after = k (test aid): leave the num_steps-schedule after k steps and return the state the reference hands to
    its denoiser at call k (conditioning frames re-imposed, sampling.py:105-106)."""
    sigmas = edm_sigmas(num_steps)
    x = noise.clone() * torch.sqrt(1.0 + sigmas[0] ** 2)          # :36
    scales = guider_scales(guider, num_frames, scale)[:, None, None, None]
    keep = (1 - cond_mask)[:, None, None, None]
    put = cond_mask[:, None, None, None]
    replace = bool(cond_mask.any())
    cc = {k: torch.cat((uc[k], c[k]), 0) for k in ("vector", "crossattn", "concat")}
    traj = []
    for i in range(num_steps):
        if replace:
            x = x * keep + cond_frame * put                       # :105-106
        sig = x.new_ones([x.shape[0]]) * sigmas[i]
        nxt = x.new_ones([x.shape[0]]) * sigmas[i + 1]
        den = denoise(sd, cfg, torch.cat([x] * 2), torch.cat([sig] * 2), cc,
                      torch.cat([cond_mask] * 2), num_frames)
        x_u, x_c = den.chunk(2)
        den = x_u + scales * (x_c - x_u)                          # guiders.py:23-26 / 68-74
        d = (x - den) / sig[:, None, None, None]                  # sampling_utils.py:46
        x = x + d * (nxt - sig)[:, None, None, None]              # sampling.py:85-88
        if return_all:
            traj.append(x.clone())
        if stop_after is not None and i + 1 == stop_after:
            break
    if replace:
        x = x * keep + cond_frame * put                           # :122-123
    return (x, traj) if return_all else x


# ---------------------------------------------------------------------------------------------
# VAE decoder
# ---------------------------------------------------------------------------------------------
def _swish(x):
    return x * torch.sigmoid(x)


def dec_video_res_block(sd: SD, p: str, x: torch.Tensor, has_skip: bool, T: int,
                        record: Optional[dict] = None) -> torch.Tensor:
    """temporal_ae.py:55-72 on top of model.py:116-135 (temb=None).  VAE GroupNorm eps 1e-6 for the
    spatial norms, 1e-5 inside the temporal openaimodel.ResBlock; blend alpha*temporal + (1-alpha)*spatial.
    ``record`` (test aid): "res2d", "res3d" and "blend" = (alpha, a, b), out = alpha a + (1 - alpha) b, as in
    video_res_block.  The arithmetic is unchanged."""
    h = F.conv2d(_swish(_gn(sd, f"{p}.norm1", x, 1e-6)), sd[f"{p}.conv1.weight"], sd[f"{p}.conv1.bias"], padding=1)
    h = F.conv2d(_swish(_gn(sd, f"{p}.norm2", h, 1e-6)), sd[f"{p}.conv2.weight"], sd[f"{p}.conv2.bias"], padding=1)
    if has_skip:
        x = F.conv2d(x, sd[f"{p}.nin_shortcut.weight"], sd[f"{p}.nin_shortcut.bias"])
    if record is not None:
        record["res2d"] = x
    x = x + h
    bt, c, hh, ww = x.shape
    x5 = x.reshape(bt // T, T, c, hh, ww).permute(0, 2, 1, 3, 4)
    xt = res_block_3d(sd, f"{p}.time_stack", x5, None)
    alpha = torch.sigmoid(sd[f"{p}.mix_factor"])
    out = alpha * xt + (1.0 - alpha) * x5
    if record is not None:
        record["res3d"] = x
        record["blend"] = (alpha, xt.permute(0, 2, 1, 3, 4).reshape(bt, c, hh, ww), x)
    return out.permute(0, 2, 1, 3, 4).reshape(bt, c, hh, ww)


def dec_attn_block(sd: SD, p: str, x: torch.Tensor, record: Optional[dict] = None) -> torch.Tensor:
    """model.py:147-176: GN, 1x1 q/k/v, single-head SDPA with d = C, 1x1 proj_out, residual.  ``record`` (test aid):
    receives the residual operand as "res"."""
    b, c, h, w = x.shape
    hn = _gn(sd, f"{p}.norm", x, 1e-6)
    q, k, v = (F.conv2d(hn, sd[f"{p}.{n}.weight"], sd[f"{p}.{n}.bias"]) for n in ("q", "k", "v"))
    q, k, v = (t.reshape(b, 1, c, h * w).transpose(2, 3) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v)
    o = o.transpose(2, 3).reshape(b, c, h, w)
    if record is not None:
        record["res"] = x
    return x + F.conv2d(o, sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])


def decoder_forward(sd: SD, cfg: DecoderConfig, z: torch.Tensor, timesteps: int) -> torch.Tensor:
    """model.py:664-694 with VideoDecoder pieces (temporal_ae.py:105-151)."""
    plan = build_decoder_plan(cfg)
    h = F.conv2d(z, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    h = dec_video_res_block(sd, plan.mid[0].prefix, h, False, timesteps)
    h = dec_attn_block(sd, "mid.attn_1", h)
    h = dec_video_res_block(sd, plan.mid[1].prefix, h, False, timesteps)
    for blocks, up, _ in plan.levels:
        for rb in blocks:
            h = dec_video_res_block(sd, rb.prefix, h, rb.has_skip, timesteps)
        if up is not None:                                           # model.py:55-64
            h = F.conv2d(F.interpolate(h, scale_factor=2.0, mode="nearest"),
                         sd[f"{up}.weight"], sd[f"{up}.bias"], padding=1)
    h = _swish(_gn(sd, "norm_out", h, 1e-6))
    h = F.conv2d(h, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)       # AE3DConv: temporal_ae.py:90-97
    bt, c, hh, ww = h.shape
    h5 = h.reshape(bt // timesteps, timesteps, c, hh, ww).permute(0, 2, 1, 3, 4)
    h5 = F.conv3d(h5, sd["conv_out.time_mix_conv.weight"], sd["conv_out.time_mix_conv.bias"], padding=(1, 0, 0))
    return h5.permute(0, 2, 1, 3, 4).reshape(bt, c, hh, ww)


def decode_first_stage(sd: SD, cfg: DecoderConfig, z: torch.Tensor, scale_factor=0.18215,
                       n_samples=14, overlap=3) -> torch.Tensor:
    """models/diffusion.py:150-180: chunks of n_samples with `overlap` frames averaged."""
    z = z / scale_factor
    outs = []
    if overlap < n_samples:
        prev = z[:overlap]
        for cur in z[overlap:].split(n_samples - overlap, dim=0):
            ctx = torch.cat((prev, cur), dim=0)
            prev = cur[-overlap:]
            out = decoder_forward(sd, cfg, ctx, timesteps=cur.shape[0] + overlap)
            if not outs:
                outs.append(out)
            else:
                outs[-1][-overlap:] = (outs[-1][-overlap:] + out[:overlap]) / 2
                outs.append(out[overlap:])
    else:
        for cur in z.split(n_samples, dim=0):
            outs.append(decoder_forward(sd, cfg, cur, timesteps=cur.shape[0]))
    return torch.cat(outs, dim=0)


# ---------------------------------------------------------------------------------------------
# VAE encoder (SURVEY.md §8f rank 1: the next row; oracle first)
# ---------------------------------------------------------------------------------------------
def enc_res_block(sd: SD, p: str, x: torch.Tensor, has_skip: bool, record: Optional[dict] = None) -> torch.Tensor:
    """model.py:116-135 with temb = None (Encoder sets temb_ch = 0, model.py:467).  ``record`` (test aid): receives
    the residual operand as "res"."""
    h = F.conv2d(_swish(_gn(sd, f"{p}.norm1", x, 1e-6)), sd[f"{p}.conv1.weight"], sd[f"{p}.conv1.bias"], padding=1)
    h = F.conv2d(_swish(_gn(sd, f"{p}.norm2", h, 1e-6)), sd[f"{p}.conv2.weight"], sd[f"{p}.conv2.bias"], padding=1)
    if has_skip:
        x = F.conv2d(x, sd[f"{p}.nin_shortcut.weight"], sd[f"{p}.nin_shortcut.bias"])
    if record is not None:
        record["res"] = x
    return x + h


def encoder_forward(sd: SD, cfg, x: torch.Tensor) -> torch.Tensor:
    """Encoder.forward (model.py:527-557): conv_in, per level ResnetBlocks (+ Downsample: zero pad right / bottom by
    one, conv3x3 stride 2 without padding, model.py:69-83), mid (res, attn, res), GN, swish, conv_out ->
    (n, 2 z_channels, h/8, w/8) moments."""
    from vista_b200.spec import build_encoder_plan
    levels, mid_ch = build_encoder_plan(cfg)
    h = F.conv2d(x, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    for blocks, down, _ in levels:
        for rb in blocks:
            h = enc_res_block(sd, rb.prefix, h, rb.has_skip)
        if down is not None:
            h = F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[f"{down}.weight"], sd[f"{down}.bias"], stride=2)
    h = enc_res_block(sd, "mid.block_1", h, False)
    h = dec_attn_block(sd, "mid.attn_1", h)
    h = enc_res_block(sd, "mid.block_2", h, False)
    h = _swish(_gn(sd, "norm_out", h, 1e-6))
    return F.conv2d(h, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


def encode_first_stage(sd: SD, cfg, x: torch.Tensor, scale_factor=0.18215, n_samples: Optional[int] = None,
                       noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """DiffusionEngine.encode_first_stage (models/diffusion.py:183-195) over AutoencodingEngine.encode
    (autoencoder.py:190-203) with DiagonalGaussianRegularizer (regularizers/__init__.py:30-40): chunks of n_samples
    frames, z = mean + exp(0.5 clamp(logvar, -30, 20)) * noise (distributions.py:25-36; the reference draws the noise
    on the device: inject it), noise = None gives the mode; times scale_factor."""
    n_samples = x.shape[0] if n_samples is None else n_samples
    outs = []
    for i in range(0, x.shape[0], n_samples):
        mom = encoder_forward(sd, cfg, x[i:i + n_samples])
        mean, logvar = torch.chunk(mom, 2, dim=1)
        z = mean
        if noise is not None:
            z = mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * noise[i:i + n_samples]
        outs.append(z)
    return torch.cat(outs, dim=0) * scale_factor


def cond_frames_embed(sd: SD, quant_w: torch.Tensor, quant_b: torch.Tensor, cfg, vid: torch.Tensor, scale_factor: float = 1.0,
                      n_cond_frames: int = 1, n_copies: int = 1, n_samples: Optional[int] = None) -> torch.Tensor:
    """VideoPredictionEmbedderWithEncoder.forward without noise augmentation (encoders/modules.py:462-502) over
    AutoencoderKLModeOnly.encode (autoencoder.py:467-488,519-528): moments = quant_conv(Encoder(x)), the regulariser in
    mode (sample=False) keeps the mean half; chunks of n_samples; * scale_factor; "(b t) c h w -> b (t c) h w"; n_copies."""
    n_samples = vid.shape[0] if n_samples is None else n_samples
    outs = []
    for i in range(0, vid.shape[0], n_samples):
        mom = F.conv2d(encoder_forward(sd, cfg, vid[i:i + n_samples]), quant_w, quant_b)
        outs.append(torch.chunk(mom, 2, dim=1)[0])
    out = torch.cat(outs, dim=0) * scale_factor
    bt, c, h, w = out.shape
    out = out.reshape(bt // n_cond_frames, n_cond_frames * c, h, w)
    return out.repeat_interleave(n_copies, dim=0)
