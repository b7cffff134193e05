"""The conditioner's CLIP image branch on native sm_90a kernels.

``FrozenOpenCLIPImageEmbedder`` / ``FrozenOpenCLIPImagePredictionEmbedder`` mirror vwm/modules/encoders/modules.py:251-399
and :505-516 (same constructor keywords, same ``forward`` result) so that the first entry of ``conditioner_config``
(configs/inference/vista.yaml:44-52) can name them.  Weights load with ``load_state_dict`` under the module tree the
reference builds (``model.visual.*`` in open_clip's names); nothing is downloaded.  The tower runs on ``ClipRuntime``:

  preprocess + patchify ... b200v_clip_preprocess (kornia resize, (x + 1) / 2, CLIP mean / std, 14 x 14 patches)
  patch embedding ......... b200v_gemm; its row-vector epilogue (rv_mod 257) adds class embedding + positional embedding,
                            the class-token slot of every image being a zero patch row
  ln_pre / ln_1 / ln_2 .... b200v_layernorm
  attention ............... fused in-proj GEMM [3C, C] -> b200v_attention_d80 -> out_proj GEMM with the residual
  MLP ..................... c_fc GEMM with the erf-GELU epilogue (act 3) -> c_proj GEMM with the residual
  ln_post, proj ........... b200v_layernorm over the class rows -> b200v_gemm (no bias), fp32 out

The residual stream is fp16 with fp32 epilogue arithmetic; the reference runs the tower under autocast (modules.py:317).
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Union

import torch
import torch.nn as nn

from . import ops
from .diffusion import instantiate_from_config
from .modules import register_param_tree
from .spec import CLIP_TEXT_LEFTOVERS, ClipConfig, clip_param_specs, clip_preset
from .unet import Lin


class ClipRuntime:
    """Packed weights and persistent buffers of one tower on one device."""

    def __init__(self, cfg: ClipConfig, sd: Dict[str, torch.Tensor], device, prefix: str = "model.visual."):
        assert cfg.patch_size == 14 and cfg.image_size == 224 and cfg.head_width == 80, \
            "the native tower is the 224 px, patch 14, head width 80 ViT"
        self.cfg, self.dev, self.prefix = cfg, torch.device(device), prefix
        self._bufs = {}
        self._sd = sd
        self._pack()
        self._sd = None

    def _t(self, name, dtype=torch.float32):
        return self._sd[self.prefix + name].detach().to(self.dev, dtype).contiguous()

    def _lin(self, w: torch.Tensor, b: Optional[torch.Tensor]) -> Lin:
        return Lin(w.to(torch.float16).contiguous(), b, ops.pick_tile_n(w.shape[0]))

    def _norm(self, p):
        return self._t(f"{p}.weight"), self._t(f"{p}.bias")

    def _pack(self):
        cfg, C = self.cfg, self.cfg.width
        w = self._t("conv1.weight").reshape(C, cfg.patch_k)
        wp = torch.zeros(C, cfg.patch_k_pad, dtype=torch.float32, device=self.dev)
        wp[:, :cfg.patch_k] = w
        self.patch = self._lin(wp, None)
        tok = self._t("positional_embedding").clone()                 # [257, C]
        tok[0] += self._t("class_embedding")
        self.tok_rowvec = tok.contiguous()
        self.ln_pre = self._norm("ln_pre")
        self.blocks = []
        for i in range(cfg.layers):
            p = f"transformer.resblocks.{i}"
            self.blocks.append(dict(
                ln1=self._norm(f"{p}.ln_1"),
                qkv=self._lin(self._t(f"{p}.attn.in_proj_weight"), self._t(f"{p}.attn.in_proj_bias")),
                out=self._lin(self._t(f"{p}.attn.out_proj.weight"), self._t(f"{p}.attn.out_proj.bias")),
                ln2=self._norm(f"{p}.ln_2"),
                fc=self._lin(self._t(f"{p}.mlp.c_fc.weight"), self._t(f"{p}.mlp.c_fc.bias")),
                proj=self._lin(self._t(f"{p}.mlp.c_proj.weight"), self._t(f"{p}.mlp.c_proj.bias"))))
        self.ln_post = self._norm("ln_post")
        self.proj = self._lin(self._t("proj").t(), None)              # x @ proj == GEMM with proj^T [embed, C]

    def buf(self, name, rows, cols, dtype=torch.float16):
        key = (name, rows, cols, dtype)
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = torch.empty(rows, cols, dtype=dtype, device=self.dev)
        return t

    def gemm(self, a, lin: Lin, out, **kw):
        return ops.gemm(a, lin.w, out, bias=lin.b, tile_n=lin.tile_n, **kw)

    def forward(self, x: torch.Tensor, antialias: bool = True) -> torch.Tensor:
        """x (n,3,H,W) fp32 in [-1, 1] on this device -> (n, embed_dim) fp32 (a persistent buffer)."""
        cfg, C = self.cfg, self.cfg.width
        n, L = x.shape[0], cfg.tokens
        M = n * L
        rows = ops.clip_preprocess(x.float().contiguous(), self.buf("c.patch", M, cfg.patch_k_pad), antialias)
        x0 = self.gemm(rows, self.patch, self.buf("c.x1", M, C), rowvec=self.tok_rowvec, rv_mod=L)
        xa = ops.layernorm(x0, self.buf("c.x0", M, C), *self.ln_pre, eps=cfg.ln_eps)
        xb = self.buf("c.x1", M, C)
        h = self.buf("c.h", M, C)
        qkv = self.buf("c.qkv", M, 3 * C)
        o = self.buf("c.o", M, C)
        f = self.buf("c.f", M, cfg.mlp_width)
        for B in self.blocks:
            ops.layernorm(xa, h, *B["ln1"], eps=cfg.ln_eps)
            self.gemm(h, B["qkv"], qkv)
            ops.attention_d80(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o, n, L, cfg.heads)
            self.gemm(o, B["out"], xb, res1=xa)
            ops.layernorm(xb, h, *B["ln2"], eps=cfg.ln_eps)
            self.gemm(h, B["fc"], f, act=3)
            self.gemm(f, B["proj"], xa, res1=xb)
        cls = self.buf("c.cls", n, C)
        ops.layernorm(xa.view(n, L * C)[:, :C], cls, *self.ln_post, eps=cfg.ln_eps)
        return self.gemm(cls, self.proj, self.buf("c.emb", n, cfg.embed_dim, torch.float32))


class FrozenOpenCLIPImageEmbedder(nn.Module):
    """modules.py:251-399.  Supported: ``arch="ViT-H-14"`` (or a ``vista_b200.spec.ClipConfig`` for other towers with head
    width 80), ``output_tokens=False``, ``num_image_crops=0``, ``ucg_rate=0``, ``unsqueeze_dim=False``,
    ``repeat_to_max_len=False`` (the settings of vista.yaml:44-52), either ``antialias``; other values raise
    NotImplementedError.  ``version`` / ``init_device`` are accepted and unused: weights come from ``load_state_dict``
    (``load_open_clip_weights`` reads a local open_clip file)."""

    def __init__(self, arch: Union[str, ClipConfig] = "ViT-H-14", version: str = "laion2b_s32b_b79k", device: str = "cuda",
                 max_length: int = 77, freeze: bool = True, antialias: bool = True, ucg_rate: float = 0.0,
                 unsqueeze_dim: bool = False, repeat_to_max_len: bool = False, num_image_crops: int = 0,
                 output_tokens: bool = False, init_device=None):
        super().__init__()
        bad = [k for k, v in dict(arch=not (arch == "ViT-H-14" or isinstance(arch, ClipConfig)), ucg_rate=ucg_rate != 0.0,
                                  num_image_crops=num_image_crops != 0, output_tokens=bool(output_tokens),
                                  unsqueeze_dim=bool(unsqueeze_dim), repeat_to_max_len=bool(repeat_to_max_len)).items() if v]
        if bad:
            raise NotImplementedError(f"vista_b200.clip.FrozenOpenCLIPImageEmbedder: unsupported option(s) {bad}")
        self.b200_config = arch if isinstance(arch, ClipConfig) else clip_preset("vit_h_14")
        self.model = nn.Module()
        self.model.visual = nn.Module()
        register_param_tree(self.model.visual, clip_param_specs(self.b200_config))
        self.device, self.max_length = device, max_length
        self.antialias, self.ucg_rate = antialias, ucg_rate
        self.is_trainable, self.input_key = False, None      # AbstractEmbModel attributes the GeneralConditioner reads
        if freeze:
            self.requires_grad_(False)
        self._runtime = None
        self._register_load_state_dict_pre_hook(self._drop_text_leftovers)
        self.register_load_state_dict_post_hook(lambda module, keys: setattr(module, "_runtime", None))

    @staticmethod
    def _drop_text_leftovers(state_dict, prefix, *args):
        for k in CLIP_TEXT_LEFTOVERS:
            state_dict.pop(prefix + "model." + k, None)

    def _apply(self, fn, *args, **kwargs):     # keep the packed runtime unless a parameter moved / changed dtype
        before = tuple((p.device, p.dtype) for p in self.parameters())
        out = super()._apply(fn, *args, **kwargs)
        if tuple((p.device, p.dtype) for p in self.parameters()) != before:
            self._runtime = None
        return out

    def runtime(self, device) -> ClipRuntime:
        if torch.device(device).type != "cuda":
            raise RuntimeError("vista_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self._runtime is None or self._runtime.dev != torch.device(device):
            self._runtime = ClipRuntime(self.b200_config, self.state_dict(), device)
        return self._runtime

    @torch.no_grad()
    def forward(self, image: torch.Tensor, no_dropout: bool = False):
        if image.dim() == 5:
            raise NotImplementedError("multi-crop input (num_image_crops > 0) is not supported")
        return self.runtime(image.device).forward(image, self.antialias).to(image.dtype)

    def encode(self, image):
        return self(image)


class FrozenOpenCLIPImagePredictionEmbedder(nn.Module):
    """modules.py:505-516: the image embedder, then "(b t) d -> b t d" and ``n_copies`` repeats "b t d -> (b s) t d"."""

    def __init__(self, open_clip_embedding_config: Dict, n_cond_frames: int, n_copies: int):
        super().__init__()
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.open_clip = instantiate_from_config(open_clip_embedding_config)
        self.is_trainable, self.ucg_rate, self.input_key = False, 0.0, None

    def output_shape(self, vid: torch.Tensor):
        """Shape ``forward(vid)`` returns, without running the tower."""
        return (vid.shape[0] // self.n_cond_frames * self.n_copies, self.n_cond_frames, self.open_clip.b200_config.embed_dim)

    def forward(self, vid: torch.Tensor) -> torch.Tensor:
        z = self.open_clip(vid)
        z = z.reshape(-1, self.n_cond_frames, z.shape[-1])
        return z.repeat_interleave(self.n_copies, dim=0)


def load_open_clip_weights(path: str, prefix: str = "model.") -> Dict[str, torch.Tensor]:
    """State dict of ``FrozenOpenCLIPImageEmbedder`` from a local open_clip checkpoint (``open_clip_pytorch_model.bin`` or
    ``.safetensors``): the vision tower and the text leftovers under ``prefix``; the text transformer, which the reference
    deletes, is dropped.  Reads the file only; nothing is downloaded."""
    if not os.path.isfile(path):
        raise FileNotFoundError(path)
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
        sd = sd.get("state_dict", sd)
    return {prefix + k: v for k, v in sd.items() if not k.startswith("transformer.")}
