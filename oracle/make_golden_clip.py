"""Golden fixtures of the conditioner's CLIP image branch (tests/golden/clip_tiny.npz, clip_vith_14.npz).

Runs the REAL reference classes ``FrozenOpenCLIPImagePredictionEmbedder`` / ``FrozenOpenCLIPImageEmbedder``
(vwm/modules/encoders/modules.py:251-399,505-516) on the CPU in fp32 over stand-ins for the two packages that are not
installed here (the stubs of oracle/ref_loader.py leave them empty):
  open_clip.create_model_and_transforms -> a model whose ``.visual`` is transformers' CLIPVisionModelWithProjection
      (hidden_act "gelu") loaded from the open_clip-named synthetic weights: third-party arithmetic for the tower, in the
      role the SDPA shim plays for xformers.
  kornia.geometry.resize / kornia.enhance.normalize -> oracle.clip_oracle.kornia_resize / kornia_normalize, a restatement
      of kornia 0.6.9 (not executed upstream code; DESIGN.md §2).

    python -m oracle.make_golden_clip [--only clip_tiny]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import clip_oracle, ref_loader  # noqa: E402
from vista_b200 import spec, synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
PRE_STRIDE = 4          # the preprocessed 224 x 224 input is stored as x[:, :, ::4, ::4]

# fixture -> (preset, weight seed, [(frames name, n, H, W, antialias)])
CASES = {
    "clip_tiny": ("tiny", 11, [("a", 3, 64, 128, True), ("b", 2, 576, 1024, True), ("c", 2, 576, 1024, False)]),
    "clip_vith_14": ("vit_h_14", 12, [("a", 2, 576, 1024, True)]),
}


def clip_frames(seed: int, name: str, n: int, H: int, W: int) -> np.ndarray:
    """Synthetic frames in [-1, 1] with image-like spatial structure: a smooth field plus fine noise, clipped."""
    base = synth.normal(seed, f"clip.frames.{name}.base", (n, 3, H // 8 + 1, W // 8 + 1), std=0.6)
    t = torch.nn.functional.interpolate(torch.from_numpy(base), size=(H, W), mode="bilinear", align_corners=True)
    fine = torch.from_numpy(synth.normal(seed, f"clip.frames.{name}.fine", (n, 3, H, W), std=0.15))
    return torch.clamp(t + fine, -1.0, 1.0).numpy()


def clip_weights(preset: str, seed: int):
    cfg = spec.clip_preset(preset)
    return cfg, synth.synth_state_dict(spec.clip_param_specs(cfg), seed=seed)


def hf_vision_from_open_clip(cfg: spec.ClipConfig, sd) -> nn.Module:
    """transformers' CLIPVisionModelWithProjection holding the open_clip-named weights ``sd`` (keys relative to visual)."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    hc = CLIPVisionConfig(hidden_size=cfg.width, intermediate_size=cfg.mlp_width, num_hidden_layers=cfg.layers,
                          num_attention_heads=cfg.heads, image_size=cfg.image_size, patch_size=cfg.patch_size,
                          projection_dim=cfg.embed_dim, hidden_act="gelu", layer_norm_eps=cfg.ln_eps, num_channels=3)
    hc._attn_implementation = "eager"
    m = CLIPVisionModelWithProjection(hc).eval()
    t = lambda k: torch.from_numpy(np.ascontiguousarray(sd[k]))
    C = cfg.width
    w = {"vision_model.embeddings.patch_embedding.weight": t("conv1.weight"),
         "vision_model.embeddings.class_embedding": t("class_embedding"),
         "vision_model.embeddings.position_embedding.weight": t("positional_embedding"),
         "vision_model.pre_layrnorm.weight": t("ln_pre.weight"), "vision_model.pre_layrnorm.bias": t("ln_pre.bias"),
         "vision_model.post_layernorm.weight": t("ln_post.weight"), "vision_model.post_layernorm.bias": t("ln_post.bias"),
         "visual_projection.weight": t("proj").t().contiguous()}
    for i in range(cfg.layers):
        p, h = f"transformer.resblocks.{i}", f"vision_model.encoder.layers.{i}"
        iw, ib = t(f"{p}.attn.in_proj_weight"), t(f"{p}.attn.in_proj_bias")
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            w[f"{h}.self_attn.{n}.weight"] = iw[j * C:(j + 1) * C].contiguous()
            w[f"{h}.self_attn.{n}.bias"] = ib[j * C:(j + 1) * C].contiguous()
        for src, dst in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                         ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            w[f"{h}.{dst}.weight"], w[f"{h}.{dst}.bias"] = t(f"{p}.{src}.weight"), t(f"{p}.{src}.bias")
    missing, unexpected = m.load_state_dict(w, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


class _Visual(nn.Module):
    def __init__(self, hf):
        super().__init__()
        self.hf = hf
        self.output_tokens = False

    def forward(self, img):
        return self.hf(pixel_values=img).image_embeds


def install_stand_ins(cfg: spec.ClipConfig, sd):
    """open_clip / kornia modules with exactly what FrozenOpenCLIPImageEmbedder calls."""
    oc = types.ModuleType("open_clip")

    def create_model_and_transforms(arch, device=None, pretrained=None):
        model = nn.Module()
        model.visual = _Visual(hf_vision_from_open_clip(cfg, sd))
        model.transformer = nn.Identity()          # deleted by the reference (modules.py:277)
        return model, None, None

    oc.create_model_and_transforms = create_model_and_transforms
    ko = types.ModuleType("kornia")
    ko.geometry = types.SimpleNamespace(resize=clip_oracle.kornia_resize)
    ko.enhance = types.SimpleNamespace(normalize=clip_oracle.kornia_normalize)
    sys.modules["open_clip"], sys.modules["kornia"] = oc, ko
    sys.modules.pop("vwm.modules.encoders.modules", None)     # re-import against these modules
    ref_loader.load_reference()
    with contextlib.redirect_stdout(io.StringIO()):
        from vwm.modules.encoders import modules as enc
    return enc


def make(name: str):
    preset, seed, frames = CASES[name]
    cfg, sd = clip_weights(preset, seed)
    crc = synth.state_dict_checksum(sd)
    enc = install_stand_ins(cfg, sd)
    out = {"weights_crc": np.array(crc), "weight_seed": np.array(seed), "pre_stride": np.array(PRE_STRIDE)}
    for fname, n, H, W, aa in frames:
        x = clip_frames(seed, fname, n, H, W)
        emb = enc.FrozenOpenCLIPImagePredictionEmbedder(
            open_clip_embedding_config={"target": "vwm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder",
                                        "params": {"freeze": True, "antialias": aa, "device": "cpu"}},
            n_cond_frames=1, n_copies=1).eval()
        with torch.no_grad():
            xt = torch.from_numpy(x)
            z = emb(xt)
            pre = emb.open_clip.preprocess(xt)
        out[f"{fname}_shape"] = np.array([n, H, W, int(aa)], np.int64)
        out[f"{fname}_frames_crc"] = np.array(synth.checksum([x]))
        out[f"{fname}_emb"] = z.float().numpy()
        out[f"{fname}_pre"] = pre[:, :, ::PRE_STRIDE, ::PRE_STRIDE].float().numpy()
        print(f"{name}/{fname}: frames {x.shape} -> {tuple(z.shape)}, |z| = {float(z.norm()):.4f}")
    path = os.path.join(GOLDEN, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes), weights crc32 {crc}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    torch.set_num_threads(os.cpu_count() or 1)
    for n in CASES:
        if args.only in (None, n):
            make(n)
