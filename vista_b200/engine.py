"""``DiffusionEngine`` surface (vwm/models/diffusion.py:20-131,150-180,306-329) for the hot path: the attributes
and methods ``sample_utils`` uses (.model, .denoiser, .first_stage_model, .scale_factor, .decode_first_stage,
.sample, .ema_scope) on top of the B200 executors, plus the SURVEY §8f rows as engine calls (``encode_first_stage`` with
``encoder_config: vista_b200.vae.Encoder``, ``rollout``, ``sample_ensemble``, ``decode_first_stage_u8``).  Training is out of
scope and raises; a conditioner is built when a ``conditioner_config`` is given (``vista_b200.conditioner.GeneralConditioner``
runs every embedder natively, configs/inference/vista_b200_native.yaml), not otherwise; ``condition`` turns a user's
inputs into ``c`` / ``uc`` with it."""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from .diffusion import B200Denoiser, get_obj_from_str, instantiate_from_config
from .modules import B200Wrapper
from .vae import VideoDecoder, decode_first_stage as _decode_first_stage


class FirstStage(nn.Module):
    """Holds the decoder under the reference's key prefix ``first_stage_model.decoder.*``
    (AutoencodingEngine.decode, vwm/models/autoencoder.py:206-208)."""

    def __init__(self, decoder_config: Dict, encoder_config: Optional[Dict] = None, **reference_only):
        super().__init__()
        # AutoencodingEngine keywords (vwm/models/autoencoder.py:106-125) without a meaning at inference are accepted
        known = {"loss_config", "regularizer_config", "optimizer_config", "lr_g_factor", "trainable_ae_params",
                 "ae_optimizer_args", "trainable_disc_params", "disc_optimizer_args", "disc_start_iter", "diff_boost_factor",
                 "ckpt_engine", "ckpt_path", "additional_decode_keys", "ema_decay", "monitor", "input_key"}
        unknown = sorted(set(reference_only) - known)
        if unknown:
            raise TypeError(f"vista_b200.engine.FirstStage: unexpected keyword(s) {unknown}")
        self.decoder = instantiate_from_config(decoder_config)
        # optional: the B200 encoder (SURVEY.md §8f rank 1, vista_b200.vae.Encoder), keys
        # ``first_stage_model.encoder.*`` as in the reference checkpoint
        if encoder_config is not None:
            self.encoder = instantiate_from_config(encoder_config)

    def decode(self, z: torch.Tensor, **kwargs) -> torch.Tensor:
        return self.decoder(z, **kwargs)

    def encode(self, x, **kwargs):
        if not hasattr(self, "encoder"):
            raise NotImplementedError("no encoder_config given: the VAE encoder is the next row after the hot path "
                                      "(SURVEY.md §8f); pass latents, or add encoder_config: vista_b200.vae.Encoder")
        return self.encoder(x)                 # moments (mean | logvar); sampling lives in encode_first_stage


class DiffusionEngine(nn.Module):
    def __init__(self, network_config: Dict, denoiser_config: Dict, first_stage_config: Optional[Dict] = None,
                 conditioner_config=None, sampler_config: Optional[Dict] = None, scale_factor: float = 1.0,
                 disable_first_stage_autocast: bool = False, en_and_decode_n_samples_a_time: Optional[int] = None,
                 num_frames: int = 25, network_wrapper: Optional[str] = None, replace_cond_frames: bool = False,
                 fixed_cond_frames: Optional[List[int]] = None, input_key: str = "img_seq", **reference_only):
        super().__init__()
        # keywords of the reference constructor (vwm/models/diffusion.py:20-46) that only matter for training / logging
        # are accepted and ignored; anything else is a mistyped YAML key and must not be dropped silently
        known = {"optimizer_config", "scheduler_config", "loss_fn_config", "ckpt_path", "use_ema", "ema_decay_rate",
                 "log_keys", "no_cond_log", "compile_model", "slow_spatial_layers", "train_peft_adapters"}
        unknown = sorted(set(reference_only) - known)
        if unknown:
            raise TypeError(f"vista_b200.engine.DiffusionEngine: unexpected keyword(s) {unknown}")
        if reference_only.get("use_ema") or reference_only.get("ckpt_path"):
            raise NotImplementedError("use_ema / ckpt_path are training-side options; load weights with load_state_dict")
        model = instantiate_from_config(network_config)
        wrapper = get_obj_from_str(network_wrapper) if network_wrapper else B200Wrapper
        self.model = wrapper(model, compile_model=False)
        self.denoiser = instantiate_from_config(denoiser_config)
        self.sampler = instantiate_from_config(sampler_config) if sampler_config is not None else None
        # The conditioner (CLIP / VAE-encoder / sinusoids, encoders/modules.py): built from conditioner_config when given
        # (vista_b200.conditioner.GeneralConditioner is the native one; do_sample calls
        # model.conditioner.get_unconditional_conditioning), none otherwise.  Checkpoint keys `conditioner.*` load into it.
        self._conditioner = instantiate_from_config(conditioner_config) if conditioner_config is not None else None
        self._register_load_state_dict_pre_hook(self._conditioner_keys)
        if first_stage_config is not None:
            params = first_stage_config.get("params", first_stage_config)
            self.first_stage_model = FirstStage(params["decoder_config"], params.get("encoder_config")
                                                if str(params.get("encoder_config", {}).get("target", "")).startswith("vista_b200.") else None)
        else:
            self.first_stage_model = None
        self.scale_factor = scale_factor
        self.disable_first_stage_autocast = disable_first_stage_autocast
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time
        self.num_frames = num_frames
        self.replace_cond_frames = replace_cond_frames
        self.fixed_cond_frames = fixed_cond_frames
        self.input_key = input_key
        self.use_ema = False

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def conditioner(self):
        if self._conditioner is None:
            raise NotImplementedError("no conditioner_config given: the conditioner (CLIP / VAE-encoder / sinusoids) is "
                                      "outside the hot path; pass c / uc dicts, or give a conditioner_config to host")
        return self._conditioner

    @staticmethod
    def _conditioner_keys(state_dict, prefix, *args):
        """The reference checkpoint holds the conditioner under `conditioner.*`; this engine keeps it as `_conditioner`."""
        src, dst = prefix + "conditioner.", prefix + "_conditioner."
        for k in [k for k in state_dict if k.startswith(src)]:
            state_dict[dst + k[len(src):]] = state_dict.pop(k)

    @torch.no_grad()
    def condition(self, value_dict: Dict, num_frames: int, force_uc_zero_embeddings: Optional[List[str]] = None):
        """(c, uc) from a user's inputs: get_batch + get_condition (sample_utils.py:232-276) on the hosted conditioner —
        every input repeated over ``num_frames`` rows, the unconditional batch a copy with ``force_uc_zero_embeddings``
        zeroed, the results trimmed to ``num_frames`` rows (a result with fewer keeps its first row)."""
        dev = self.device
        batch = {}
        for key in {e.input_key for e in self.conditioner.embedders}:
            if key not in value_dict:
                continue
            v = value_dict[key]
            if key in ("fps", "fps_id", "motion_bucket_id", "cond_aug"):
                batch[key] = torch.tensor([v]).to(dev).repeat(num_frames)
            elif key in ("command", "trajectory", "speed", "angle", "goal", "cond_frames", "cond_frames_without_noise"):
                v = torch.as_tensor(v).to(dev)
                v = v[None] if key in ("command", "trajectory", "speed", "angle", "goal") else v
                batch[key] = v.expand((num_frames,) + tuple(v.shape[1:])).contiguous()
            else:
                raise NotImplementedError(f"condition: no batch rule for input {key!r} (sample_utils.py:237-247)")
        batch_uc = {k: v.clone() for k, v in batch.items()}
        c, uc = self.conditioner.get_unconditional_conditioning(batch, batch_uc=batch_uc,
                                                                force_uc_zero_embeddings=list(force_uc_zero_embeddings or []))
        for k in c:
            if isinstance(c[k], torch.Tensor):
                c[k], uc[k] = c[k][:num_frames], uc[k][:num_frames]
                if c[k].shape[0] < num_frames:
                    c[k] = c[k][[0]]
                if uc[k].shape[0] < num_frames:
                    uc[k] = uc[k][[0]]
        return c, uc

    @contextlib.contextmanager
    def ema_scope(self, context=None):          # no-op at inference (diffusion.py:241-255, use_ema False)
        yield None

    @torch.no_grad()
    def decode_first_stage(self, z: torch.Tensor, overlap: int = 3) -> torch.Tensor:
        dec = self.first_stage_model.decoder
        if not isinstance(dec, VideoDecoder):
            raise NotImplementedError("decode_first_stage needs vista_b200.vae.VideoDecoder as decoder_config.target")
        if getattr(self.model, "frame_sharded", False):     # one clip on several ranks: spread the decode as well
            import torch.distributed as dist
            from .vae import _decode_chunks, decode_first_stage_parallel
            group = getattr(self.model, "world_group", None)
            n_chunks = len(_decode_chunks(z.shape[0], self.en_and_decode_n_samples_a_time or z.shape[0], overlap))
            # frame-shard the chunks when there are more ranks than chunks — up to 4 ranks, where that path is validated
            # on hardware; an 8-rank frame chain over NCCL point-to-point timed out in its first hardware run, so larger
            # worlds deal whole chunks out instead
            if n_chunks < dist.get_world_size(group) <= 4:
                # more ranks than chunks: shard the FRAMES of every chunk (sharded.ShardedDecoderRuntime)
                from .sharded import ShardedDecoderRuntime, decode_first_stage_sharded
                srt = getattr(dec, "_sharded_rt", None)
                if srt is None or srt.dev != torch.device(z.device) or srt.group is not group:
                    srt = dec._sharded_rt = ShardedDecoderRuntime(dec.b200_config, dec.state_dict(), z.device, group=group)
                return decode_first_stage_sharded(srt, z, self.scale_factor, self.en_and_decode_n_samples_a_time, overlap)
            # as many chunks as ranks (or fewer ranks): deal whole chunks out, bit-identical to the serial decode
            return decode_first_stage_parallel(dec.runtime(z.device), z, self.scale_factor,
                                               self.en_and_decode_n_samples_a_time, overlap, group=group)
        return _decode_first_stage(dec.runtime(z.device), z, self.scale_factor, self.en_and_decode_n_samples_a_time, overlap)

    @torch.no_grad()
    def decode_first_stage_u8(self, z: torch.Tensor, overlap: int = 3) -> torch.Tensor:
        """Extension (SURVEY.md 8f rank 4): the decoded frames as (F, H, W, 3) uint8 — bit for bit what the reference's
        output path (sample_utils.py:374 clamp, :96-126 scaling / truncation / "t h w c") makes of decode_first_stage's
        result, produced by the decoder's last kernel instead of three full-resolution fp32 passes on the host."""
        dec = self.first_stage_model.decoder
        if not isinstance(dec, VideoDecoder):
            raise NotImplementedError("decode_first_stage_u8 needs vista_b200.vae.VideoDecoder as decoder_config.target")
        return _decode_first_stage(dec.runtime(z.device), z, self.scale_factor, self.en_and_decode_n_samples_a_time, overlap,
                                   u8=True)

    @torch.no_grad()
    def encode_first_stage(self, x, noise: Optional[torch.Tensor] = None, sample: bool = True):
        """diffusion.py:183-195.  Needs ``encoder_config`` (the B200 encoder).  The reference samples the
        posterior with device RNG (DiagonalGaussianRegularizer, sample=True): pass ``noise`` for a reproducible draw,
        ``sample=False`` for the mode."""
        enc = getattr(self.first_stage_model, "encoder", None)
        if enc is None:
            raise NotImplementedError("the VAE encoder is outside the B200 hot path (SURVEY.md §8f); add encoder_config")
        from .vae import Encoder, encode_first_stage as _encode_first_stage
        if not isinstance(enc, Encoder):
            raise NotImplementedError("encode_first_stage needs vista_b200.vae.Encoder as encoder_config.target")
        rt = enc.runtime(x.device)
        if sample and noise is None:
            d = 2 ** (len(rt.cfg.ch_mult) - 1)
            noise = torch.randn(x.shape[0], rt.cfg.z_channels, x.shape[2] // d, x.shape[3] // d, device=x.device)
        return _encode_first_stage(rt, x, self.scale_factor, self.en_and_decode_n_samples_a_time, noise if sample else None)

    @torch.no_grad()
    def sample(self, cond: Dict, cond_frame=None, uc: Union[Dict, None] = None, N: int = 25,
               shape: Union[None, Tuple, List] = None, noise: Optional[torch.Tensor] = None, **kwargs):
        """diffusion.py:306-329; ``noise`` may be injected (device RNG is not reproducible across devices)."""
        randn = torch.randn(N, *shape).to(self.device) if noise is None else noise.to(self.device).clone()
        cond_mask = torch.zeros(N).to(self.device)
        if self.replace_cond_frames:
            assert self.fixed_cond_frames
            cond_mask = cond_mask.reshape(-1, self.num_frames)
            cond_mask[:, self.fixed_cond_frames] = 1
            cond_mask = cond_mask.reshape(-1)
        denoiser = B200Denoiser(self.denoiser, self.model)
        return self.sampler(denoiser, randn, cond, uc=uc, cond_frame=cond_frame, cond_mask=cond_mask)

    # ---- the callers' loops as engine operations (SURVEY.md 8f rows 2 / 3; vista_b200/rollout.py) ----
    def rollout(self, cond: Dict, uc: Dict, z: torch.Tensor, num_rounds: int, **kwargs):
        """Long-horizon rollout, the body of sample_utils.do_sample (sample_utils.py:318-373) -> (frames, samples_z)."""
        from .rollout import rollout
        return rollout(self, cond, uc, z, num_rounds, **kwargs)

    def rollout_session(self, value_dict: Dict, z: torch.Tensor, **kwargs):
        """The same rollout in closed loop (vista_b200/session.py): ``step(action)`` samples one round conditioned on that
        action and returns its final uint8 frames; ``close()`` returns the last round's final three; ``score(candidates)``
        rates actions for the next round with the ensemble reward, and ``fork()`` copies the session."""
        from .session import RolloutSession
        return RolloutSession(self, value_dict, z, **kwargs)

    @torch.no_grad()
    def frames_from_u8(self, frames: torch.Tensor, height: int = 576, width: int = 1024) -> torch.Tensor:
        """sample.py's load_img (sample.py:174-201) on decoded RGB frames: uint8 (T, Hs, Ws, 3), on the host or a device,
        -> (T, 3, height, width) fp32 in [-1, 1] on the engine's device, ``torch.equal`` to load_img's tensors for the
        same pixels (centre crop, PIL LANCZOS resize, ToTensor, ``* 2 - 1``; vista_b200/ingest.py).  A host tensor is
        copied to the device as uint8."""
        from . import ingest
        ingest.check_frames(frames, height, width)
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("frames_from_u8 runs on the CUDA kernels of csrc/ingest/ingest.cu; move the engine to a GPU")
        return ingest.frames_u8_resize(frames.to(dev), height, width)

    @torch.no_grad()
    def rollout_session_from_frames(self, frames: torch.Tensor, n_conds: int = 1, cond_aug: float = 0.0,
                                    action: Optional[Dict] = None, force_uc_zero_embeddings: Optional[List[str]] = None,
                                    height: int = 576, width: int = 1024, cond_aug_noise: Optional[torch.Tensor] = None,
                                    encode_noise: Optional[torch.Tensor] = None):
        """A rollout session started from camera frames, as sample.py does it (sample.py:222-253 and the head of
        sample_utils.do_sample): frames [0, n_conds) through ``frames_from_u8``; a value dict of
        sample_utils.init_embedder_options, the first frame as ``cond_frames_without_noise``, that frame plus
        ``cond_aug * cond_aug_noise`` as ``cond_frames``, ``cond_aug`` and the action keys of ``action``; the frames encoded
        with ``encode_first_stage``; ``initial_cond_indices = range(n_conds)``.

        Only the conditioning frames [0, n_conds) reach a session: the sampler reads ``z`` under the initial mask,
        ``rollout_advance`` and ``score`` read z[0].  So only those frames are resized and encoded, and ``z`` is zero on
        the other frames.  ``frames``: uint8 (>= n_conds, Hs, Ws, 3).  ``cond_aug_noise``: (1, 3, height, width), by
        default drawn with ``torch.randn_like``.  ``encode_noise``: the posterior noise, (>= n_conds, 4, h, w) of which
        frames [0, n_conds) are used; by default drawn by ``encode_first_stage``."""
        from . import ingest
        from .session import ACTION_KEYS
        if not isinstance(n_conds, int) or not 1 <= n_conds <= self.num_frames:
            raise ValueError(f"n_conds must be in [1, {self.num_frames}], got {n_conds}")
        ingest.check_frames(frames, height, width, min_frames=n_conds)
        action = dict(action or {})
        unknown = sorted(set(action) - set(ACTION_KEYS))
        if unknown:
            raise ValueError(f"rollout_session_from_frames: {unknown} are not action keys {ACTION_KEYS}")
        img = self.frames_from_u8(frames[:n_conds], height, width)
        value_dict = ingest.embedder_options({e.input_key for e in self.conditioner.embedders})
        cond_img = img[0:1]
        noise = torch.randn_like(cond_img) if cond_aug_noise is None else cond_aug_noise.to(img.device, torch.float32)
        value_dict["cond_frames_without_noise"] = cond_img
        value_dict["cond_aug"] = cond_aug
        value_dict["cond_frames"] = cond_img + cond_aug * noise
        value_dict.update(action)
        if encode_noise is not None:
            encode_noise = encode_noise[:n_conds].to(img.device, torch.float32).contiguous()
        zc = self.encode_first_stage(img, noise=encode_noise)
        z = zc.new_zeros((self.num_frames,) + tuple(zc.shape[1:]))
        z[:n_conds] = zc
        return self.rollout_session(value_dict, z, force_uc_zero_embeddings=force_uc_zero_embeddings,
                                    initial_cond_indices=list(range(n_conds)))

    def sample_ensemble(self, cond: Dict, uc: Dict, z: torch.Tensor, ensemble_size: int = 5, **kwargs):
        """The reward path (reward_utils.py:318-337) -> (reward, members)."""
        from .rollout import sample_ensemble
        return sample_ensemble(self, cond, uc, z, ensemble_size, **kwargs)
