"""Closed-loop rollout: ``engine.rollout`` one round at a time, with a new action every round and that round's final uint8
frames as soon as it is sampled — Vista driven as a simulator by a planner that looks at the frames so far.

At T = 25, n_cond = 3 and the engine's 14-frame decode chunks with a 3-frame overlap, the batch decode of ``samples_z``
(22 N + 3 frames) uses chunks [11 k, 11 k + 14) for k = 0 .. 2 N - 1 (``vae._decode_chunks``).  Round n owns latents
[22 n, 22 n + 25): exactly chunks 2 n and 2 n + 1.  Once round n is sampled its frames [22 n, 22 n + 22) are therefore
final; frames 22 n + 22 .. 22 n + 24 are averaged with chunk 2 n + 2, so their raw fp32 is carried to the next round; and
the first of them is the decoded frame ``do_sample`` re-embeds with CLIP between rounds (sample_utils.py:340-343), the
raw output of chunk 2 n + 1.  N rounds cost 2 N chunk decodes, against 3 N - 1 for ``engine.rollout`` (N - 1 decodes of
the tail for the re-conditioning, then the whole clip).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from . import ops
from .diffusion import B200Denoiser
from .rollout import _masks, conditioner_recondition
from .vae import VideoDecoder, _decode_chunks, decode_chunk_u8

ACTION_KEYS = ("command", "trajectory", "speed", "angle", "goal")
# the geometry whose decode chunks line up with the rounds (sample.py's defaults): T = 25, n_cond = 3, 14-frame chunks
# overlapping by 3 (the overlap of decode_first_stage)
_T, _N_COND, _CHUNK, _OVERLAP = 25, 3, 14, 3


class RolloutSession:
    """``engine.rollout(c, uc, z, N, recondition=conditioner_recondition(engine, value_dict, uc_keys), u8=True)`` stepped
    one round per ``step``.  ``step(action)`` x N followed by ``close()``, concatenated, are the bytes of that call's frames,
    and ``samples_z`` its latents, when the action is the same every round.

    ``value_dict``: what ``engine.condition`` takes.  ``z``: the encoded clip (T, 4, h, w), as ``engine.rollout`` takes it.
    ``action`` of ``step``: a dict of ``ACTION_KEYS`` merged into ``value_dict`` for that round only, or None to keep the
    previous round's action."""

    def __init__(self, engine, value_dict: Dict, z: torch.Tensor, force_uc_zero_embeddings: Optional[Sequence[str]] = None,
                 initial_cond_indices: Sequence[int] = (0,), n_cond: int = 3):
        engine.conditioner                                          # raises when the engine hosts no conditioner
        if getattr(engine.model, "frame_sharded", False):
            raise NotImplementedError("rollout_session: a frame-sharded engine is not supported; use engine.rollout")
        if (engine.num_frames, z.shape[0], n_cond, engine.en_and_decode_n_samples_a_time) != (_T, _T, _N_COND, _CHUNK):
            raise NotImplementedError(
                f"rollout_session: the decode chunks must line up with the rounds, which needs num_frames = {_T}, "
                f"n_cond = {_N_COND} and en_and_decode_n_samples_a_time = {_CHUNK} (got num_frames = {engine.num_frames}, "
                f"z frames = {z.shape[0]}, n_cond = {n_cond}, en_and_decode_n_samples_a_time = "
                f"{engine.en_and_decode_n_samples_a_time})")
        dec = engine.first_stage_model.decoder
        if not isinstance(dec, VideoDecoder):
            raise NotImplementedError("rollout_session needs vista_b200.vae.VideoDecoder as decoder_config.target")
        self.engine, self.value_dict, self.n_cond = engine, dict(value_dict), n_cond
        self.uc_keys = list(force_uc_zero_embeddings or [])
        self.z = z.float().contiguous()
        self.rounds = 0
        self._den = B200Denoiser(engine.denoiser, engine.model)
        self._init_mask, self._pred_mask = _masks(_T, initial_cond_indices, n_cond, z.device)
        self._samples_z = self.z.new_zeros((0,) + tuple(z.shape[1:]))
        self._filled = torch.zeros_like(self.z)
        self._action: Dict = {}
        self._sample = None             # the last round's sample
        self._carry = None              # raw fp32 of the last round's final n_cond frames, before their averaging
        self._tail = None               # uint8 of those frames, final once no round follows
        self._closed = False

    @property
    def samples_z(self) -> torch.Tensor:
        """The latents of the rounds so far, laid out as ``engine.rollout``'s ``samples_z``."""
        return self._samples_z

    @torch.no_grad()
    def step(self, action: Optional[Dict] = None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Sample the next round -> its (T - n_cond, H, W, 3) uint8 frames, final.  ``noise``: the round's sampler noise
        (T, 4, h, w); by default ``torch.randn_like(z)``, drawn in the order ``engine.rollout`` draws it."""
        if self._closed:
            raise RuntimeError("rollout_session: step() after close()")
        if action is not None:
            unknown = sorted(set(action) - set(ACTION_KEYS))
            if unknown:
                raise ValueError(f"rollout_session: {unknown} are not action keys {ACTION_KEYS}")
            self._action = dict(action)
        eng, z, n, r = self.engine, self.z, self.n_cond, self.rounds
        vd = dict(self.value_dict)
        vd.update(self._action)
        if r == 0:
            cond, uc = eng.condition(vd, _T, self.uc_keys)
        else:
            # the decoded frame do_sample re-embeds is the first carried frame: decode_tail()[[-n_cond]]
            cond, uc = conditioner_recondition(eng, vd, self.uc_keys, n)(r, self._sample, lambda: self._carry)
        x = torch.randn_like(z) if noise is None else noise.to(z.device, torch.float32).clone().contiguous()
        self._samples_z = torch.cat([self._samples_z, z.new_zeros((_T if r == 0 else _T - n,) + tuple(z.shape[1:]))])
        if r == 0:
            sample = eng.sampler(self._den, x, cond, uc=uc, cond_frame=z, cond_mask=self._init_mask)
            ops.rollout_advance(sample, z, self._samples_z, self._filled, 0, 0, n)
        else:
            sample = eng.sampler(self._den, x, cond, uc=uc, cond_frame=self._filled.clone(), cond_mask=self._pred_mask)
            ops.rollout_advance(sample, None, self._samples_z, self._filled, r * (_T - n), n, n)
        self._sample = sample
        self.rounds += 1
        return self._decode(r)

    def _decode(self, r: int) -> torch.Tensor:
        """Chunks 2 r and 2 r + 1 of the batch decode, with the arguments decode_first_stage(..., u8=True) gives them."""
        eng, n = self.engine, self.n_cond
        rt = eng.first_stage_model.decoder.runtime(self.z.device)
        zs = (self._samples_z[r * (_T - n):r * (_T - n) + _T] / eng.scale_factor).contiguous()
        _, _, h, w = zs.shape
        up = 2 ** (len(rt.cfg.ch_mult) - 1)
        out8 = torch.empty(_T, h * up, w * up, rt.cfg.out_ch, dtype=torch.uint8, device=zs.device)
        # one chunk's fp32 frames: its first _OVERLAP are read for the averaging, its last _OVERLAP kept for the next chunk
        f32 = torch.empty(_CHUNK, rt.cfg.out_ch, h * up, w * up, dtype=torch.float32, device=zs.device)
        for f0, cn, o0, nov in _decode_chunks(_T, _CHUNK, _OVERLAP):
            if self._carry is not None:          # every chunk after the clip's first averages with its predecessor
                nov = _OVERLAP
                f32[:nov].copy_(self._carry)
            decode_chunk_u8(rt, zs[f0:f0 + cn], f32, out8[o0:], 0, nov, cn - _OVERLAP)
            self._carry = f32[cn - _OVERLAP:].clone()
        self._tail = out8[_T - n:]
        return out8[:_T - n]

    def close(self) -> torch.Tensor:
        """End the rollout -> the last round's final n_cond frames, (n_cond, H, W, 3) uint8."""
        if self._tail is None:
            raise RuntimeError("rollout_session: close() before the first step()")
        self._closed = True
        return self._tail
