"""Drop-in ``nn.Module`` surface for the reference's plug-in seams (SURVEY.md §8b).

  * ``VideoUNet``   — usable as ``network_config.target`` (same constructor keywords and the same
                     ``state_dict`` key names/shapes as vwm.modules.diffusionmodules.video_model.VideoUNet,
                     so ``load_state_dict`` of a Vista checkpoint fills it; video_model.py:78-503).
  * ``B200Wrapper`` — usable as ``DiffusionEngine(network_wrapper=...)``: called as
                     ``Cls(model, compile_model=bool)`` (models/diffusion.py:54-58) and as
                     ``forward(x, t, c, cond_mask, num_frames)`` (wrappers.py:25-40).  It accepts either
                     our ``VideoUNet`` or the *reference* ``VideoUNet`` instance (it only reads its
                     hyper-parameters and ``state_dict``) and runs the B200 executor.

Both fail loudly without the CUDA library or a CUDA device: there is no CPU / eager fallback.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Union

import torch
import torch.nn as nn

from . import ops
from .spec import UNetConfig, unet_param_specs
from .unet import UNetRuntime, padded_input_rows


class _Node(nn.Module):
    """Anonymous container so that parameters can be registered under dotted reference names."""


def register_param_tree(root: nn.Module, specs: Dict[str, tuple], dtype=torch.float32) -> None:
    """Creates nested sub-modules / parameters so that ``root.state_dict()`` has exactly the keys of
    ``specs``.  Initial values: zeros for tensors the reference zero-initialises, N(0, fan_in^-1/2)
    otherwise, ones for norm gains, the reference's blend logits (0.5 / 0.0)."""
    for name, (shape, kind) in specs.items():
        parts = name.split(".")
        mod = root
        for p in parts[:-1]:
            if not hasattr(mod, p):
                mod.add_module(p, _Node())
            mod = getattr(mod, p)
        t = torch.empty(shape, dtype=dtype)
        if kind == "w":
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t.normal_(0.0, (1.0 / max(fan_in, 1)) ** 0.5 * 0.577)
        elif kind in ("wz", "b"):
            t.zero_()
        elif kind == "g":
            t.fill_(1.0)
        elif kind == "mix":
            t.fill_(0.5)
        elif kind == "mix0":
            t.fill_(0.0)
        else:
            raise KeyError(kind)
        mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))


def _infer_config(model: nn.Module) -> UNetConfig:
    """UNetConfig of a reference ``VideoUNet`` instance from its attributes (video_model.py:127-145) and
    weight shapes."""
    if hasattr(model, "b200_config"):
        return model.b200_config
    sd = model.state_dict()
    ctx_key = next(k for k in sd if k.endswith("transformer_blocks.0.attn2.to_k.weight"))
    cfg = UNetConfig(
        in_channels=int(model.in_channels), out_channels=int(model.out_channels),
        model_channels=int(model.model_channels), attention_resolutions=tuple(model.attention_resolutions),
        num_res_blocks=int(model.num_res_blocks), channel_mult=tuple(model.channel_mult),
        num_head_channels=int(model.num_head_channels), context_dim=int(sd[ctx_key].shape[1]),
        adm_in_channels=int(sd["label_emb.0.0.weight"].shape[1]),
        action_control=any(k.endswith("k_adapter_action_control.weight") for k in sd))
    mine = {k: tuple(v[0]) for k, v in unet_param_specs(cfg).items()}
    theirs = {k: tuple(v.shape) for k, v in sd.items()}
    if mine != theirs:
        diff = [k for k in set(mine) | set(theirs) if mine.get(k) != theirs.get(k)][:5]
        raise NotImplementedError(f"network architecture not supported by the B200 executor (e.g. {diff})")
    return cfg


class _RuntimeOwner:
    """Lazily (re)builds the device-side executor from the module's current parameters."""

    def _rt_init(self):
        self._runtime: Optional[UNetRuntime] = None
        self._runtime_key = None
        self._cond_cache = None
        self._shard_group = None
        self.frame_sharded = False
        self._frame_world = 1
        self.cfg_half = None          # 0: this rank runs the unconditional half of the CFG batch, 1: the conditional
        self.pair_group = None        # the two ranks that own the same frames of the two halves

    def enable_frame_sharding(self, group=None, cfg_split: Optional[bool] = None):
        """Spread ONE clip over the ranks of `group` (BASELINE config 5); see vista_b200/sharded.py.
        With an even world size the two halves of the classifier-free-guidance batch go to the two halves of
        the ranks (no collective between them inside the UNet; the 4-channel network outputs of a frame's two
        halves are exchanged once per step for the guidance), and the frames of each half are sharded over
        world/2 ranks.  With an odd world size (or cfg_split=False) only the frames are sharded.
        Only the fused sampler drives this mode (every rank passes the same full-clip inputs)."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        if cfg_split is None:
            cfg_split = world % 2 == 0
        self.frame_sharded = True
        self.world_group = group          # the group the clip is spread over (engine.decode_first_stage deals chunks over it)
        self.cfg_half, self.pair_group = None, None
        if cfg_split:
            assert world % 2 == 0, "cfg_split needs an even number of ranks"
            ranks = list(range(world)) if group is None else dist.get_process_group_ranks(group)
            wf = world // 2
            # every rank creates every group, in the same order
            fgroups = [dist.new_group([ranks[hh * wf + i] for i in range(wf)]) for hh in range(2)]
            pgroups = [dist.new_group([ranks[i], ranks[i + wf]]) for i in range(wf)]
            self.cfg_half = rank // wf
            self.pair_group = pgroups[rank % wf]
            self._shard_group = fgroups[self.cfg_half]
            self._frame_world = wf
        else:
            self._shard_group = group
            self._frame_world = world
        self._rt_invalidate()

    def peer_window(self, T: int, h: int, w: int, model_channels: int, device):
        """The NVLink peer window of this rank (vista_b200/peer.py), created on first use — collectively: every rank of the
        group the clip is spread over calls this at the same point (the sharded sampler does).  None when the peer-memory
        collectives are off (VISTA_B200_PEER=0) or the layout is not the one they serve (one clip per rank)."""
        if not self.frame_sharded or os.environ.get("VISTA_B200_PEER", "1") == "0" or self.cfg_half is None \
                or torch.device(device).type != "cuda":     # (the emulated-operator tests run the host logic on CPU tensors)
            return None
        if getattr(self, "_peer", None) is None:
            from .peer import PeerWindow
            fw = self._frame_world
            tp = -(-T // fw)                                                # frames of the largest shard
            ext = (tp + 2) * h * w * model_channels * 2                     # one halo-extended L0 activation
            kv = fw * tp * h * w * 2 * model_channels * 2                   # gathered K|V of an L0 transformer
            net = 2 * 2 * tp * h * w * 8 * 4                                # CFG pair exchange (double the rows for slack)
            nbytes = (4 * ext + kv + net + (16 << 20)) if fw > 1 else (net + (4 << 20))
            self._peer = PeerWindow(self.world_group, nbytes, device)
        return self._peer

    def _rt_invalidate(self):
        self._runtime, self._runtime_key, self._cond_cache = None, None, None

    @staticmethod
    def _placement(module: nn.Module):
        """(device, dtype) of every parameter: what `.cuda()` / `.half()` / `.to()` can change."""
        return tuple((p.device, p.dtype) for p in module.parameters())

    def _apply_keep_runtime(self, fn, *args, **kwargs):
        """nn.Module._apply that drops the packed runtime only when a parameter really moved or changed dtype: the
        reference's do_sample calls `load_model(model.model)` (= an unconditional `.cuda()`, sample_utils.py:34-47)
        once per call, which must not cost a re-pack of 1.6 B parameters and a graph re-capture."""
        before = self._placement(self)
        out = nn.Module._apply(self, fn, *args, **kwargs)
        if self._placement(self) != before:
            self._rt_invalidate()
        return out

    @staticmethod
    def _weights_version(model: nn.Module) -> int:
        """Changes whenever a parameter is written in place (load_state_dict copies in place) or replaced."""
        return hash(tuple((id(p), p._version) for p in model.parameters()))

    @staticmethod
    def _require_cuda(device):
        if not torch.cuda.is_available() or torch.device(device).type != "cuda":
            raise RuntimeError("vista_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")

    def _rt_get(self, model: nn.Module, num_frames: int, device) -> UNetRuntime:
        self._require_cuda(device)
        key = (num_frames, str(device), id(model), self.frame_sharded, self._weights_version(model))
        if self._runtime is None or self._runtime_key != key:
            cfg = _infer_config(model)
            if self.frame_sharded and self._frame_world > 1:
                from .sharded import ShardedUNetRuntime
                self._runtime = ShardedUNetRuntime(cfg, model.state_dict(), device, num_frames, group=self._shard_group)
            else:
                self._runtime = UNetRuntime(cfg, model.state_dict(), device, num_frames)
                self._runtime.t0, self._runtime.t1, self._runtime.group = 0, num_frames, None
            self._runtime.cfg_half, self._runtime.pair_group = self.cfg_half, self.pair_group
            self._runtime_key = key
            self._cond_cache = None
        return self._runtime

    def _rt_forward(self, model, x, timesteps, context, y, cond_mask, num_frames):
        if self.frame_sharded:
            raise RuntimeError("frame-sharded mode is driven by the fused sampler (EulerEDMSampler with a B200Denoiser)")
        rt = self._rt_get(model, num_frames, x.device)
        B, Cin, h, w = x.shape
        if context.shape[0] != B:                                   # video_model.py:463-465
            assert context.shape[0] == B // num_frames
            context = context.repeat_interleave(num_frames, dim=0)
        if y.shape[0] != B:                                         # video_model.py:468-470
            assert y.shape[0] == B // num_frames
            y = y.repeat_interleave(num_frames, dim=0)
        cc = self._cond_cache
        if cc is None or cc[0].shape != context.shape or cc[1].shape != y.shape \
                or not (torch.equal(cc[0], context) and torch.equal(cc[1], y)):
            rt.set_conditioning(context, y)
            self._cond_cache = (context.detach().clone(), y.detach().clone())
        key = ("io.x", B * h * w)
        tok = rt._bufs.get(key)
        if tok is None:
            tok = rt._bufs[key] = padded_input_rows(B * h * w, x.device)
        if Cin < 8:
            tok.zero_()
        ops.nchw_to_tokens(x.float().contiguous(), tok, B, Cin, h, w)
        mask = None if cond_mask is None else cond_mask.to(x.device, torch.float32).contiguous()
        out_tok = rt.forward(tok, timesteps.to(x.device, torch.float32).contiguous(), mask, h, w)
        out = torch.empty(B, rt.cfg.out_channels, h, w, dtype=torch.float32, device=x.device)
        ops.tokens_to_nchw(out_tok, out, B, rt.cfg.out_channels, h, w)
        return out


class VideoUNet(nn.Module, _RuntimeOwner):
    """B200-native stand-in for the reference ``VideoUNet`` (same keywords; unsupported variants of the
    reference's option space raise ``NotImplementedError`` instead of silently computing something else)."""

    def __init__(self, in_channels: int, model_channels: int, out_channels: int, num_res_blocks: int,
                 attention_resolutions: Sequence[int], dropout: float = 0.0,
                 channel_mult: Sequence[int] = (1, 2, 4, 8), conv_resample: bool = True, dims: int = 2,
                 num_classes: Optional[Union[int, str]] = None, use_checkpoint: bool = False, num_heads: int = -1,
                 num_head_channels: int = -1, num_heads_upsample: int = -1, use_scale_shift_norm: bool = False,
                 resblock_updown: bool = False, transformer_depth: Union[List[int], int] = 1,
                 transformer_depth_middle: Optional[int] = None, context_dim: Optional[int] = None,
                 time_downup: bool = False, time_context_dim: Optional[int] = None, extra_ff_mix_layer: bool = False,
                 use_spatial_context: bool = False, merge_strategy: str = "learned_with_images",
                 merge_factor: float = 0.5, spatial_transformer_attn_type: str = "softmax",
                 video_kernel_size: Union[int, List[int]] = 3, use_linear_in_transformer: bool = False,
                 adm_in_channels: Optional[int] = None, disable_temporal_crossattention: bool = False,
                 max_ddpm_temb_period: int = 10000, add_lora: bool = False, action_control: bool = False):
        super().__init__()
        depth = transformer_depth if isinstance(transformer_depth, int) else None
        if not isinstance(transformer_depth, int) and len(set(transformer_depth)) == 1:
            depth = transformer_depth[0]
        unsupported = {
            "dims": dims != 2, "num_classes": num_classes != "sequential", "num_head_channels": num_head_channels != 64,
            "use_scale_shift_norm": use_scale_shift_norm, "resblock_updown": resblock_updown,
            "transformer_depth": depth != 1 or transformer_depth_middle not in (None, 1), "time_downup": time_downup,
            "extra_ff_mix_layer": not extra_ff_mix_layer, "use_spatial_context": not use_spatial_context,
            "merge_strategy": merge_strategy != "learned_with_images",
            "video_kernel_size": list(video_kernel_size) != [3, 1, 1] if not isinstance(video_kernel_size, int) else True,
            "use_linear_in_transformer": not use_linear_in_transformer, "conv_resample": not conv_resample,
            "disable_temporal_crossattention": disable_temporal_crossattention, "add_lora": add_lora,
            "max_ddpm_temb_period": max_ddpm_temb_period != 10000, "dropout": dropout != 0.0,
            "context_dim": context_dim is None, "adm_in_channels": adm_in_channels is None,
        }
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError(f"vista_b200.VideoUNet supports the Vista inference configuration only; "
                                      f"unsupported option(s): {bad}")
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        self.num_res_blocks, self.attention_resolutions = num_res_blocks, list(attention_resolutions)
        self.channel_mult, self.num_head_channels, self.num_classes = list(channel_mult), num_head_channels, num_classes
        self.b200_config = UNetConfig(in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
                                      attention_resolutions=tuple(attention_resolutions), num_res_blocks=num_res_blocks,
                                      channel_mult=tuple(channel_mult), num_head_channels=num_head_channels,
                                      context_dim=context_dim, adm_in_channels=adm_in_channels,
                                      action_control=action_control)
        register_param_tree(self, unet_param_specs(self.b200_config))
        self._rt_init()
        self.register_load_state_dict_post_hook(lambda module, keys: module._rt_invalidate())

    def _apply(self, fn, *args, **kwargs):       # .cuda() / .half() / .to(): re-pack on next forward if anything moved
        return self._apply_keep_runtime(fn, *args, **kwargs)

    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, context: Optional[torch.Tensor] = None,
                y: Optional[torch.Tensor] = None, time_context: Optional[torch.Tensor] = None,
                cond_mask: Optional[torch.Tensor] = None, num_frames: Optional[int] = None) -> torch.Tensor:
        assert y is not None, "Must specify y if and only if the model is class-conditional"   # video_model.py:452
        assert context is not None and num_frames is not None
        return self._rt_forward(self, x, timesteps, context, y, cond_mask, num_frames)


class B200Wrapper(nn.Module, _RuntimeOwner):
    """``network_wrapper`` drop-in for vwm.modules.diffusionmodules.wrappers.OpenAIWrapper."""

    def __init__(self, diffusion_model: nn.Module, compile_model: bool = False):
        super().__init__()
        self.diffusion_model = diffusion_model      # keeps `model.diffusion_model.*` checkpoint keys (sample_utils.py:72)
        self._rt_init()

    def _apply(self, fn, *args, **kwargs):
        return self._apply_keep_runtime(fn, *args, **kwargs)

    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, cond_mask: torch.Tensor, num_frames: int,
                **kwargs) -> torch.Tensor:
        concat = c.get("concat", None)
        if concat is not None:
            if num_frames > 1 and concat.shape[0] != x.shape[0]:                 # wrappers.py:28-30
                assert concat.shape[0] == x.shape[0] // num_frames, f"{concat.shape} {x.shape}"
                concat = concat.repeat_interleave(num_frames, dim=0)
                c["concat"] = concat
            x = torch.cat((x, concat.to(x.dtype)), dim=1)
        model = self.diffusion_model
        if isinstance(model, VideoUNet):
            return model(x, timesteps=t, context=c.get("crossattn", None), y=c.get("vector", None),
                         cond_mask=cond_mask, num_frames=num_frames, **kwargs)
        return self._rt_forward(model, x, t, c.get("crossattn", None), c.get("vector", None), cond_mask, num_frames)
