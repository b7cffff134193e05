"""CPU fp32 restatement of the conditioner's CLIP image branch (the ``cond_frames_without_noise`` embedder of
configs/inference/vista.yaml:44-52).  Pure torch on the CPU; the fixtures in tests/golden/clip_*.npz come from the real
reference classes (oracle/make_golden_clip.py) and pin this file.

  FrozenOpenCLIPImagePredictionEmbedder.forward ... vwm/modules/encoders/modules.py:505-516
  FrozenOpenCLIPImageEmbedder.forward ............. modules.py:317-335 (output_tokens False, no crops, ucg_rate 0)
  encode_with_vision_transformer .................. modules.py:367-380
  preprocess ...................................... modules.py:293-305 (kornia resize, (x + 1) / 2, CLIP mean / std)
  the tower ....................................... open_clip VisionTransformer: conv1 (14 x 14, stride 14, no bias),
                                                    class token, positional embedding, ln_pre, pre-LN residual blocks
                                                    (nn.MultiheadAttention, GELU MLP), ln_post on the class token, @ proj
"""
from __future__ import annotations

import math
from typing import Dict, Sequence, Tuple

import torch
import torch.nn.functional as F

from vista_b200.spec import ClipConfig

SD = Dict[str, torch.Tensor]
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)    # modules.py:290
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)    # modules.py:291


def kornia_resize(x: torch.Tensor, size: Tuple[int, int], interpolation: str = "bicubic", align_corners: bool = True,
                  antialias: bool = False) -> torch.Tensor:
    """``kornia.geometry.resize`` as kornia 0.6.9 defines it, restated (kornia is not installed here): when ``antialias``
    and the image shrinks along some axis, a separable Gaussian blur (reflect border) with sigma = max((factor - 1) / 2,
    0.001) per axis and kernel size int(max(4 sigma, 3)) made odd; then ``F.interpolate``.  An input already of ``size``
    is returned unchanged.  This is the one piece of the CLIP path not pinned to executed upstream code."""
    h, w = x.shape[-2:]
    if (h, w) == tuple(size):
        return x
    factors = (h / size[0], w / size[1])
    if antialias and max(factors) > 1:
        sigmas = (max((factors[0] - 1.0) / 2.0, 0.001), max((factors[1] - 1.0) / 2.0, 0.001))
        ks = [int(max(2.0 * 2 * s, 3)) for s in sigmas]
        ks = [k + 1 if k % 2 == 0 else k for k in ks]
        n, c = x.shape[:2]
        y = x.reshape(n * c, 1, h, w)

        def gauss(k: int, s: float) -> torch.Tensor:
            t = torch.arange(k, dtype=x.dtype, device=x.device) - k // 2
            g = torch.exp(-t.pow(2.0) / float(2 * s ** 2))
            return g / g.sum()

        gy, gx = gauss(ks[0], sigmas[0]), gauss(ks[1], sigmas[1])
        y = F.conv2d(F.pad(y, (0, 0, ks[0] // 2, ks[0] // 2), mode="reflect"), gy.view(1, 1, -1, 1))
        y = F.conv2d(F.pad(y, (ks[1] // 2, ks[1] // 2, 0, 0), mode="reflect"), gx.view(1, 1, 1, -1))
        x = y.reshape(n, c, h, w)
    return F.interpolate(x, size=size, mode=interpolation, align_corners=align_corners)


def kornia_normalize(x: torch.Tensor, mean, std) -> torch.Tensor:
    """``kornia.enhance.normalize``: (x - mean) / std per channel."""
    mean = torch.as_tensor(mean, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    std = torch.as_tensor(std, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    return (x - mean) / std


def preprocess(x: torch.Tensor, antialias: bool = True, image_size: int = 224) -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.preprocess (modules.py:293-305): (n,3,H,W) in [-1, 1] -> (n,3,224,224)."""
    x = kornia_resize(x, (image_size, image_size), interpolation="bicubic", align_corners=True, antialias=antialias)
    x = (x + 1.0) / 2.0
    return kornia_normalize(x, CLIP_MEAN, CLIP_STD)


def vision_tower(sd: SD, cfg: ClipConfig, img: torch.Tensor, prefix: str = "") -> torch.Tensor:
    """open_clip VisionTransformer.forward (pooled output only): (n,3,224,224) -> (n, embed_dim)."""
    g = lambda k: sd[prefix + k].float()
    n, C, heads = img.shape[0], cfg.width, cfg.heads
    x = F.conv2d(img, g("conv1.weight"), stride=cfg.patch_size)                 # (n, C, 16, 16)
    x = x.flatten(2).transpose(1, 2)                                            # (n, 256, C)
    x = torch.cat([g("class_embedding").expand(n, 1, C), x], dim=1) + g("positional_embedding")
    ln = lambda p, t: F.layer_norm(t, (C,), g(f"{p}.weight"), g(f"{p}.bias"), cfg.ln_eps)
    x = ln("ln_pre", x)
    L = x.shape[1]
    for i in range(cfg.layers):
        p = f"transformer.resblocks.{i}"
        h = ln(f"{p}.ln_1", x)
        qkv = F.linear(h, g(f"{p}.attn.in_proj_weight"), g(f"{p}.attn.in_proj_bias"))
        q, k, v = (t.reshape(n, L, heads, cfg.head_width).transpose(1, 2) for t in qkv.split(C, dim=-1))
        a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(cfg.head_width), dim=-1) @ v
        a = a.transpose(1, 2).reshape(n, L, C)
        x = x + F.linear(a, g(f"{p}.attn.out_proj.weight"), g(f"{p}.attn.out_proj.bias"))
        h = ln(f"{p}.ln_2", x)
        h = F.gelu(F.linear(h, g(f"{p}.mlp.c_fc.weight"), g(f"{p}.mlp.c_fc.bias")))
        x = x + F.linear(h, g(f"{p}.mlp.c_proj.weight"), g(f"{p}.mlp.c_proj.bias"))
    pooled = ln("ln_post", x[:, 0])
    return pooled @ g("proj")


def image_embedder(sd: SD, cfg: ClipConfig, image: torch.Tensor, antialias: bool = True, prefix: str = "") -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.forward: (n,3,H,W) -> (n, embed_dim)."""
    return vision_tower(sd, cfg, preprocess(image.float(), antialias, cfg.image_size), prefix)


def prediction_embedder(sd: SD, cfg: ClipConfig, vid: torch.Tensor, n_cond_frames: int = 1, n_copies: int = 1,
                        antialias: bool = True, prefix: str = "") -> torch.Tensor:
    """FrozenOpenCLIPImagePredictionEmbedder.forward (modules.py:512-516): "(b t) d -> b t d", then n_copies repeats
    "b t d -> (b s) t d"."""
    z = image_embedder(sd, cfg, vid, antialias, prefix)
    z = z.reshape(-1, n_cond_frames, z.shape[-1])
    return z.repeat_interleave(n_copies, dim=0)


def recondition(c: dict, frames: torch.Tensor, sample: torch.Tensor, embed, scale_factor: float, n_cond: int = 3,
                clip_dim: int = 1024) -> dict:
    """The conditioning of the next rollout round (sample_utils.py:339-350) as the hot path sees it: frame [-3] of the
    decoded tail through CLIP (get_batch repeats it over the rows, sample_utils.py:243-244) into crossattn[..., :clip_dim],
    concat = sample[[-n_cond]] / scale_factor (skip_encode); the other crossattn slots and vector are kept."""
    c = dict(c)
    rows = c["crossattn"].shape[0]
    emb = embed(frames[[-3]].expand(rows, -1, -1, -1).contiguous())
    cross = c["crossattn"].clone()
    cross[..., :clip_dim] = emb.reshape(rows, 1, clip_dim).to(cross.dtype)
    c["crossattn"] = cross
    c["concat"] = (sample[[-n_cond]] / scale_factor).expand(c["concat"].shape[0], -1, -1, -1).contiguous()
    return c
