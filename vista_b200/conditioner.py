"""The conditioner: ``GeneralConditioner`` and the embedders of vista.yaml's ``conditioner_config`` that are not CLIP.

``GeneralConditioner`` mirrors vwm/modules/encoders/modules.py:70-180 (same ``emb_models`` list, same routing of the
embedder outputs into ``vector`` / ``crossattn`` / ``concat``, same ``get_unconditional_conditioning``) for inference:
  - every sinusoidal embedder of one output tensor is ONE ``b200v_sinusoid_embed`` launch that writes its column slices of
    the preallocated fp32 output, and the other embedders write theirs into it: no ``torch.cat``;
  - an embedder whose input key is forced to zero is not run, its slot is written with zeros;
  - an image input whose rows all equal row 0 (``get_batch`` repeats the one conditioning frame, sample_utils.py:243-244)
    is embedded once and the result broadcast; every embedder here computes each row on its own, so this is exact.
``ConcatTimestepEmbedderND`` mirrors modules.py:402-425 on the same kernel.

``VideoPredictionEmbedderWithEncoder`` mirrors vwm/modules/encoders/modules.py:428-502 (same constructor keywords, same
``forward`` / ``skip_encode`` behaviour) so that the ``cond_frames`` entry of ``conditioner_config`` (vista.yaml:68-96) can
name it; ``AutoencoderKLModeOnly`` mirrors vwm/models/autoencoder.py:432-528 for the one thing that embedder calls,
``encode(x)`` = mode of the posterior after ``quant_conv``.  Checkpoint keys are the reference's
(``...encoder.encoder.*``, ``...encoder.quant_conv.*``; the reference also carries an unused decoder + post_quant_conv
there, which ``load_state_dict(strict=False)`` — what sample_utils.py:72 uses — skips).  The encoder runs on
``vista_b200.vae.EncoderRuntime`` with ``quant_conv`` (1x1, 8 -> 8) folded into the 3x3 ``conv_out`` weights at packing
time: no extra pass, no torch compute on the path.  The CLIP branch lives in vista_b200/clip.py."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import ops
from .diffusion import instantiate_from_config
from .modules import register_param_tree
from .vae import Encoder, EncoderRuntime


class AutoencoderKLModeOnly(nn.Module):
    def __init__(self, embed_dim: int, ddconfig: Dict, **reference_only):
        super().__init__()
        known = {"monitor", "loss_config", "ckpt_path", "ckpt_engine", "max_batch_size", "lr_g_factor", "input_key",
                 "optimizer_config", "regularizer_config", "trainable_ae_params", "ae_optimizer_args", "ema_decay"}
        unknown = sorted(set(reference_only) - known)
        if unknown:
            raise TypeError(f"vista_b200.conditioner.AutoencoderKLModeOnly: unexpected keyword(s) {unknown}")
        dd = dict(ddconfig)
        if dd.get("attn_type") == "vanilla-xformers":      # same arithmetic (model.py:199-227 vs :158-170), our kernel either way
            dd["attn_type"] = "vanilla"
        if not dd.get("double_z", True):
            raise NotImplementedError("AutoencoderKLModeOnly needs double_z (mean | logvar moments)")
        self.encoder = Encoder(**dd)
        zc = self.encoder.b200_config.z_channels
        self.embed_dim = embed_dim
        register_param_tree(self, {"quant_conv.weight": ((2 * embed_dim, 2 * zc, 1, 1), "w"), "quant_conv.bias": ((2 * embed_dim,), "b")})
        self._runtime = None
        self.register_load_state_dict_post_hook(lambda module, keys: setattr(module, "_runtime", None))

    def _apply(self, fn, *args, **kwargs):
        before = tuple((p.device, p.dtype) for p in self.parameters())
        out = super()._apply(fn, *args, **kwargs)
        if tuple((p.device, p.dtype) for p in self.parameters()) != before:
            self._runtime = None
        return out

    def runtime(self, device) -> EncoderRuntime:
        if torch.device(device).type != "cuda":
            raise RuntimeError("vista_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self._runtime is None:
            qw = self.get_parameter("quant_conv.weight").detach().float().flatten(1)       # [2e, 2z]
            qb = self.get_parameter("quant_conv.bias").detach().float()
            self._runtime = EncoderRuntime(self.encoder.b200_config, self.encoder.state_dict(), device, post=(qw, qb))
        return self._runtime

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_reg_log: bool = False):
        """autoencoder.py:467-488 with the DiagonalGaussianRegularizer in mode (sample=False): (n,3,H,W) -> (n,embed_dim,H/8,W/8).
        One frame per pass: the GroupNorm statistics' work split follows the frame count of a call, so this keeps a frame's
        latent independent of how many frames share the call (GeneralConditioner's one-row shortcut relies on it)."""
        rt = self.runtime(x.device)
        n, cin, H, W = x.shape
        down = 2 ** (len(rt.cfg.ch_mult) - 1)
        x = x.float().contiguous()
        mom = torch.empty(n, 8, H // down, W // down, dtype=torch.float32, device=x.device)
        tok = rt.buf("e.x", H * W, 8)
        for i in range(n):
            tok.zero_()
            ops.nchw_to_tokens(x[i:i + 1], tok, 1, cin, H, W)
            mom_tok = rt.forward(tok, 1, H, W)
            ops.tokens_to_nchw(mom_tok, mom[i:i + 1], 1, 8, H // down, W // down)
        z = mom[:, : self.embed_dim]
        return (z, {}) if return_reg_log else z


class VideoPredictionEmbedderWithEncoder(nn.Module):
    """encoders/modules.py:428-502.  ``forward(vid)``: latents pass through when ``skip_encode`` is set (the rollout's
    re-conditioning, sample_utils.py:345-350); otherwise optional noise augmentation, the encoder in chunks of
    ``en_and_decode_n_samples_a_time``, ``* scale_factor``, "(b t) c h w -> b () (t c) h w" and ``n_copies`` repeats."""

    def __init__(self, n_cond_frames: int, n_copies: int, encoder_config: dict, sigma_sampler_config: Optional[dict] = None,
                 sigma_cond_config: Optional[dict] = None, is_ae: bool = False, scale_factor: float = 1.0,
                 disable_encoder_autocast: bool = False, en_and_decode_n_samples_a_time: Optional[int] = None):
        super().__init__()
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.encoder = instantiate_from_config(encoder_config)
        self.sigma_sampler = instantiate_from_config(sigma_sampler_config) if sigma_sampler_config is not None else None
        self.sigma_cond = instantiate_from_config(sigma_cond_config) if sigma_cond_config is not None else None
        self.is_ae, self.scale_factor = is_ae, scale_factor
        self.disable_encoder_autocast = disable_encoder_autocast
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time
        self.skip_encode = False
        # AbstractEmbModel attributes the GeneralConditioner sets / reads (encoders/modules.py:31-74)
        self.is_trainable, self.ucg_rate, self.input_key = False, 0.0, None

    def output_shape(self, vid: torch.Tensor):
        """Shape ``forward(vid)`` returns, without running the encoder (None where it cannot be known up front)."""
        if self.skip_encode:
            return tuple(vid.shape)
        if self.sigma_cond is not None or not (self.is_ae and isinstance(self.encoder, AutoencoderKLModeOnly)):
            return None
        n, _, H, W = vid.shape
        down = 2 ** (len(self.encoder.encoder.b200_config.ch_mult) - 1)
        return (n // self.n_cond_frames * self.n_copies, self.n_cond_frames * self.encoder.embed_dim, H // down, W // down)

    def forward(self, vid: torch.Tensor, noise: Optional[torch.Tensor] = None):
        if self.skip_encode:
            return vid
        sigma_cond = None
        if self.sigma_sampler is not None:
            bs = vid.shape[0] // self.n_cond_frames
            sigmas = self.sigma_sampler(bs).to(vid.device)
            if self.sigma_cond is not None:
                sigma_cond = self.sigma_cond(sigmas).repeat_interleave(self.n_copies, dim=0)
            sigmas = sigmas.repeat_interleave(self.n_cond_frames, dim=0)
            noise = torch.randn_like(vid) if noise is None else noise
            vid = vid + noise * sigmas.reshape(-1, *([1] * (vid.ndim - 1)))
        n_samples = self.en_and_decode_n_samples_a_time or vid.shape[0]
        outs = []
        for i in range(math.ceil(vid.shape[0] / n_samples)):
            chunk = vid[i * n_samples:(i + 1) * n_samples]
            outs.append(self.encoder.encode(chunk) if self.is_ae else self.encoder(chunk))
        out = torch.cat(outs, dim=0) * self.scale_factor
        bt, c, h, w = out.shape
        out = out.reshape(bt // self.n_cond_frames, self.n_cond_frames * c, h, w)          # "(b t) c h w -> b () (t c) h w"
        out = out.repeat_interleave(self.n_copies, dim=0)                                 # "b 1 c h w -> (b t) c h w"
        return (out, sigma_cond) if sigma_cond is not None else out


# ---------------------------------------------------------------------------------------------------------------------
# Sinusoidal scalar embedders and the GeneralConditioner
# ---------------------------------------------------------------------------------------------------------------------
_FREQS: Dict = {}


def _freq_table(outdims, device):
    """(device fp32 table, {outdim: offset}) of timestep_embedding's frequencies for every width in ``outdims``, computed
    on the host with the reference's own expression (util.py:155-160), so the kernel's arguments are the reference's."""
    outdims = tuple(sorted(set(int(d) for d in outdims)))
    key = (outdims, str(torch.device(device)))
    hit = _FREQS.get(key)
    if hit is None:
        parts, offs, off = [], {}, 0
        for d in outdims:
            half = d // 2
            parts.append(torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half))
            offs[d] = off
            off += half
        table = torch.cat(parts) if off else torch.zeros(1)
        hit = _FREQS[key] = (table.to(device).contiguous(), offs)
    return hit


class ConcatTimestepEmbedderND(nn.Module):
    """modules.py:402-425: each of the ``num_features`` values of a row gets its own ``outdim``-wide cos | sin embedding,
    "(b d) d2 -> b (d d2)", and ``add_sequence_dim`` adds a middle axis of 1.  Inputs are cast with ``.float()`` as
    util.py:161 does (``command`` arrives as int64).  Runs on ``b200v_sinusoid_embed``."""

    def __init__(self, outdim: int, num_features: Optional[int] = None, add_sequence_dim: bool = False):
        super().__init__()
        self.outdim, self.num_features, self.add_sequence_dim = outdim, num_features, add_sequence_dim
        self.is_trainable, self.ucg_rate, self.input_key = False, 0.0, None

    def values(self, x: torch.Tensor) -> torch.Tensor:
        """The (b, d) fp32 values one call embeds."""
        if x.ndim == 1:
            x = x[:, None]
        assert x.ndim == 2
        assert x.shape[1] == self.num_features or self.num_features is None
        return x.float()

    def width(self, dims: int) -> int:
        return dims * self.outdim

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        v = self.values(x).contiguous()
        b, dims = v.shape
        out = torch.empty(b, self.width(dims), dtype=torch.float32, device=v.device)
        freqs, offs = _freq_table([self.outdim], v.device)
        ops.sinusoid_embed(v, [(0, dims, self.outdim, 0, False, offs[self.outdim])], freqs, out)
        return out[:, None] if self.add_sequence_dim else out


def _image_embedder(emb) -> bool:
    from .clip import FrozenOpenCLIPImagePredictionEmbedder
    return isinstance(emb, (FrozenOpenCLIPImagePredictionEmbedder, VideoPredictionEmbedderWithEncoder))


class GeneralConditioner(nn.Module):
    """modules.py:70-180 for inference.  ``embedders`` is an nn.ModuleList of the embedder modules themselves (do_sample
    toggles ``skip_encode`` on them, sample_utils.py:345-351).  Training-time settings (``ucg_rate`` > 0,
    ``legacy_ucg_value``, ``is_trainable: True``, ``input_keys``) raise NotImplementedError.

    ``rows_embedded`` counts, per input key, the image rows the CLIP / cond-frame embedders actually ran on."""
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}

    def __init__(self, emb_models: List[Dict]):
        super().__init__()
        embedders = []
        for n, cfg in enumerate(emb_models):
            bad = [k for k, v in dict(is_trainable=bool(cfg.get("is_trainable", False)), ucg_rate=cfg.get("ucg_rate", 0.0) > 0.0,
                                      legacy_ucg_value=cfg.get("legacy_ucg_value") is not None,
                                      input_keys="input_keys" in cfg).items() if v]
            if bad:
                raise NotImplementedError(f"vista_b200.conditioner.GeneralConditioner: embedder #{n}: training-time "
                                          f"option(s) {bad} are not supported")
            if "input_key" not in cfg:
                raise KeyError(f"Need either `input_key` or `input_keys` for embedder #{n} ({cfg.get('target')})")
            emb = instantiate_from_config(cfg)
            emb.is_trainable, emb.ucg_rate, emb.input_key = False, 0.0, cfg["input_key"]
            emb.legacy_ucg_val = None
            emb.requires_grad_(False)
            emb.eval()
            embedders.append(emb)
        self.embedders = nn.ModuleList(embedders)
        self.rows_embedded: Dict[str, int] = {}

    # -- one embedder output -----------------------------------------------------------------------------------------
    def _embed(self, emb, x: torch.Tensor, zero: bool):
        """-> a tensor (the embedder's output), or ("zeros", shape) when nothing needs computing."""
        if zero and hasattr(emb, "output_shape"):
            shape = emb.output_shape(x)
            if shape is not None:
                return ("zeros", shape)
        if _image_embedder(emb) and not getattr(emb, "skip_encode", False):
            one_row = (x.shape[0] > 1 and emb.n_cond_frames == 1 and getattr(emb, "sigma_sampler", None) is None
                       and bool((x == x[:1]).all()))
            rows = 1 if one_row else x.shape[0]
            self.rows_embedded[emb.input_key] = self.rows_embedded.get(emb.input_key, 0) + rows
            if one_row:
                one = emb(x[:1])
                return one[:1].expand((x.shape[0] * emb.n_copies,) + tuple(one.shape[1:]))
        out = emb(x)
        assert isinstance(out, torch.Tensor), f"{type(emb).__name__} returned {type(out)}; only tensor outputs are supported"
        return ("zeros", tuple(out.shape)) if zero else out

    # -- GeneralConditioner.forward ----------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, batch: Dict, force_zero_embeddings: Optional[List] = None) -> Dict:
        force_zero_embeddings = force_zero_embeddings or []
        # 1) what every embedder contributes, in embedder order: (out_key, kind, payload, shape, added)
        plan, shapes = [], {}
        for emb in self.embedders:
            if emb.ucg_rate > 0.0:
                raise NotImplementedError("ucg_rate > 0 (training-time dropout) is not supported")
            key = emb.input_key
            zero = key in force_zero_embeddings
            if isinstance(emb, ConcatTimestepEmbedderND):
                if key in batch:
                    v = emb.values(batch[key])
                    rows, dims = v.shape
                elif emb.add_sequence_dim:              # modules.py:128-130: zeros of (B, 1, num_features * outdim)
                    v, rows, dims, zero = None, batch["cond_aug"].shape[0], emb.num_features, True
                else:                                   # modules.py:131-132: an added embedding is left out
                    continue
                shape = (rows, 1, emb.width(dims)) if emb.add_sequence_dim else (rows, emb.width(dims))
                item = ("sin", (None if zero else v, dims, emb.outdim, zero), shape)
            else:
                if key not in batch:                    # the reference fails here too (no add_sequence_dim attribute)
                    raise KeyError(f"the batch has no {key!r} for {type(emb).__name__}")
                r = self._embed(emb, batch[key], zero)
                if isinstance(r, tuple):
                    item = ("zeros", None, tuple(r[1]))
                else:
                    item = ("tensor", r, tuple(r.shape))
            out_key = self.OUTPUT_DIM2KEYS[len(item[2])]
            added = out_key in shapes and item[2][-1] == 768 and out_key == "vector"
            if out_key not in shapes:
                shapes[out_key] = list(item[2])
            elif not added:
                cd = self.KEY2CATDIM[out_key]
                prev = shapes[out_key]
                if len(prev) != len(item[2]) or any(a != b for i, (a, b) in enumerate(zip(prev, item[2])) if i != cd):
                    raise ValueError(f"{out_key}: cannot concatenate {tuple(item[2])} to {tuple(prev)} along dim {cd}")
                prev[cd] += item[2][cd]
            plan.append((out_key, item, added))
        # 2) the outputs: one fp32 buffer per key, every slot written into its column slice
        out = {k: torch.empty(s, dtype=torch.float32, device=self._device(batch)) for k, s in shapes.items()}
        offsets = {k: 0 for k in out}
        sin_slots, adds = {}, []
        for out_key, (kind, payload, shape), added in plan:
            buf = out[out_key]
            if added:
                adds.append((out_key, kind, payload, shape))
                continue
            cd = self.KEY2CATDIM[out_key]
            dst = buf.narrow(cd, offsets[out_key], shape[cd])
            if kind == "sin":
                sin_slots.setdefault(out_key, []).append((payload, offsets[out_key]))
            elif kind == "zeros":
                dst.zero_()
            else:
                dst.copy_(payload)
            offsets[out_key] += shape[cd]
        for out_key, slots in sin_slots.items():
            self._sinusoids(out[out_key], slots)
        for out_key, kind, payload, shape in adds:         # modules.py:155-156, in embedder order, onto the first 768 columns
            dst = out[out_key][..., :shape[-1]]
            if kind == "sin":
                t = torch.empty(shape, dtype=torch.float32, device=dst.device)
                self._sinusoids(t, [(payload, 0)])
                dst += t
            elif kind == "tensor":
                dst += payload
        return out

    @staticmethod
    def _device(batch: Dict):
        for v in batch.values():
            if isinstance(v, torch.Tensor):
                return v.device
        return torch.device("cpu")

    @staticmethod
    def _sinusoids(buf: torch.Tensor, slots):
        """One b200v_sinusoid_embed launch for all sinusoid slots of one output: ((values | None, dims, outdim, zero), col)."""
        rows = buf.shape[0]
        flat = buf.view(rows, -1)
        freqs, offs = _freq_table([s[0][2] for s in slots], buf.device)
        vals = [s[0][0] for s in slots if s[0][0] is not None]
        packed = torch.cat([v.to(buf.device) for v in vals], dim=1).contiguous() if vals else None
        table, vc = [], 0
        for (v, dims, outdim, zero), col in slots:
            if v is not None and v.shape[0] != rows:
                raise ValueError(f"a sinusoid embedder has {v.shape[0]} rows, its output {rows}")
            table.append((vc if v is not None else 0, dims, outdim, col, v is None, offs[outdim]))
            vc += dims if v is not None else 0
        for i in range(0, len(table), 16):                 # B200V_SINUSOID_MAX_SLOTS per launch
            ops.sinusoid_embed(packed, table[i:i + 16], freqs, flat)

    def get_unconditional_conditioning(self, batch_c: Dict, batch_uc: Optional[Dict] = None,
                                       force_cond_zero_embeddings: Optional[List[str]] = None,
                                       force_uc_zero_embeddings: Optional[List[str]] = None):
        """modules.py:163-180: (c, uc) with dropout off."""
        rates = [e.ucg_rate for e in self.embedders]
        for e in self.embedders:
            e.ucg_rate = 0.0
        try:
            c = self(batch_c, force_cond_zero_embeddings)
            uc = self(batch_c if batch_uc is None else batch_uc, force_uc_zero_embeddings)
        finally:
            for e, r in zip(self.embedders, rates):
                e.ucg_rate = r
        return c, uc
