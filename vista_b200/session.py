"""Closed-loop rollout: ``engine.rollout`` one round at a time, with a new action every round and that round's final uint8
frames as soon as it is sampled — Vista driven as a simulator by a planner that looks at the frames so far.

At T = 25, n_cond = 3 and the engine's 14-frame decode chunks with a 3-frame overlap, the batch decode of ``samples_z``
(22 N + 3 frames) uses chunks [11 k, 11 k + 14) for k = 0 .. 2 N - 1 (``vae._decode_chunks``).  Round n owns latents
[22 n, 22 n + 25): exactly chunks 2 n and 2 n + 1.  Once round n is sampled its frames [22 n, 22 n + 22) are therefore
final; frames 22 n + 22 .. 22 n + 24 are averaged with chunk 2 n + 2, so their raw fp32 is carried to the next round; and
the first of them is the decoded frame ``do_sample`` re-embeds with CLIP between rounds (sample_utils.py:340-343), the
raw output of chunk 2 n + 1.  N rounds cost 2 N chunk decodes, against 3 N - 1 for ``engine.rollout`` (N - 1 decodes of
the tail for the re-conditioning, then the whole clip).

Because that frame is carried, ``score`` samples the next round from the session's state without a decode: it conditions
each candidate action as ``step`` would, samples an ensemble and rates it with ``reward_utils.do_sample``'s reward.
"""
from __future__ import annotations

import copy
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
    previous round's action.

    For a planner: ``score(candidates)`` rates actions for the next round with the ensemble reward without advancing the
    session, and ``fork()`` copies the session for a look-ahead over several rounds."""

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

    @staticmethod
    def _check_action(action: Dict):
        unknown = sorted(set(action) - set(ACTION_KEYS))
        if unknown:
            raise ValueError(f"rollout_session: {unknown} are not action keys {ACTION_KEYS}")

    def _round_inputs(self, action: Dict):
        """-> (cond, uc, cond_frame, cond_mask): the sampler's inputs for the next round under ``action``.  Round 0 is
        conditioned on the clip under the initial mask; a later round re-runs the conditioner on the last sample and the
        carried frames, and is conditioned on the filled latents under the prediction mask.  Reads the session's state and
        changes none of it."""
        eng, r = self.engine, self.rounds
        vd = dict(self.value_dict)
        vd.update(action)
        if r == 0:
            cond, uc = eng.condition(vd, _T, self.uc_keys)
            return cond, uc, self.z, self._init_mask
        # the decoded frame do_sample re-embeds is the first carried frame: decode_tail()[[-n_cond]]
        cond, uc = conditioner_recondition(eng, vd, self.uc_keys, self.n_cond)(r, self._sample, lambda: self._carry)
        return cond, uc, self._filled.clone(), self._pred_mask

    @torch.no_grad()
    def step(self, action: Optional[Dict] = None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Sample the next round -> its (T - n_cond, H, W, 3) uint8 frames, final.  ``noise``: the round's sampler noise
        (T, 4, h, w); by default ``torch.randn_like(z)``, drawn in the order ``engine.rollout`` draws it."""
        if self._closed:
            raise RuntimeError("rollout_session: step() after close()")
        if action is not None:
            self._check_action(action)
            self._action = dict(action)
        eng, z, n, r = self.engine, self.z, self.n_cond, self.rounds
        cond, uc, cond_frame, cond_mask = self._round_inputs(self._action)
        x = torch.randn_like(z) if noise is None else noise.to(z.device, torch.float32).clone().contiguous()
        self._samples_z = torch.cat([self._samples_z, z.new_zeros((_T if r == 0 else _T - n,) + tuple(z.shape[1:]))])
        sample = eng.sampler(self._den, x, cond, uc=uc, cond_frame=cond_frame, cond_mask=cond_mask)
        if r == 0:
            ops.rollout_advance(sample, z, self._samples_z, self._filled, 0, 0, n)
        else:
            ops.rollout_advance(sample, None, self._samples_z, self._filled, r * (_T - n), n, n)
        self._sample = sample
        self.rounds += 1
        return self._decode(r)

    @torch.no_grad()
    def score(self, candidates: Sequence[Optional[Dict]], ensemble_size: int = 5, num_steps: int = 10,
              noises: Optional[Sequence[torch.Tensor]] = None, seed: int = 0, sampler=None):
        """Score candidate actions for the next round with the ensemble reward of ``reward_utils.do_sample``
        (reward_utils.py:318-337) -> (rewards (K,) fp32, members (K, E, T, 4, h, w) fp32), E = ``ensemble_size``.

        Candidate k is sampled E times as the next ``step(candidates[k])`` would sample its round — same conditioning,
        conditioning frames and mask — but with ``num_steps`` steps, ``sampler`` (default ``engine.sampler``) and member
        e's noise.  In round 0, member frame 0 is then set to z[0], so round 0 is ``engine.sample_ensemble`` on the same
        conditioning.  The reward is exp(-mean unbiased variance) over the members, on all T frames (``ops.ensemble_reward``);
        the re-imposed conditioning frames add no variance.

        ``candidates``: action dicts of ``ACTION_KEYS``, None for the session's current action.  ``noises``: E tensors
        (T, 4, h, w), member e's noise for every candidate; by default drawn from a generator seeded with ``seed`` on z's
        device, so the rewards of two candidates differ by their actions only and the global RNG is not drawn from.  The
        session is not changed: a session that scores samples the same rounds as one that does not."""
        if self._closed:
            raise RuntimeError("rollout_session: score() after close()")
        if isinstance(candidates, dict) or len(candidates) == 0:
            raise ValueError("rollout_session: score() takes a non-empty list of candidate actions")
        if not 2 <= ensemble_size <= 64:
            raise ValueError(f"rollout_session: ensemble_size must be in [2, 64] (the reward kernel's limit), "
                             f"got {ensemble_size}")
        for a in candidates:
            if a is not None:
                self._check_action(a)
        z = self.z
        if noises is None:
            g = torch.Generator(device=z.device).manual_seed(seed)
            noises = [torch.randn(z.shape, generator=g, dtype=torch.float32, device=z.device) for _ in range(ensemble_size)]
        elif len(noises) != ensemble_size or any(tuple(nz.shape) != tuple(z.shape) for nz in noises):
            raise ValueError(f"rollout_session: noises must be {ensemble_size} tensors of shape {tuple(z.shape)}, got "
                             f"{[tuple(nz.shape) for nz in noises]}")
        smp = self.engine.sampler if sampler is None else sampler
        members = z.new_empty((len(candidates), ensemble_size) + tuple(z.shape))
        for k, a in enumerate(candidates):
            cond, uc, cond_frame, cond_mask = self._round_inputs(self._action if a is None else a)
            for e in range(ensemble_size):
                x = noises[e].to(z.device, torch.float32).clone().contiguous()
                members[k, e] = smp(self._den, x, cond, uc=uc, cond_frame=cond_frame, cond_mask=cond_mask,
                                    num_steps=num_steps)
            if self.rounds == 0:
                members[k, :, 0] = z[0]                     # reward_utils.py:324
        rewards = torch.stack([ops.ensemble_reward(list(members[k]))[1] for k in range(len(candidates))])
        return rewards, members

    def fork(self) -> "RolloutSession":
        """A copy of the session that shares the engine: stepping either one afterwards leaves the other as it was."""
        new = copy.copy(self)
        new.value_dict, new._action, new.uc_keys = dict(self.value_dict), dict(self._action), list(self.uc_keys)
        new._samples_z, new._filled = self._samples_z.clone(), self._filled.clone()
        new._sample, new._carry, new._tail = (None if t is None else t.clone() for t in (self._sample, self._carry, self._tail))
        return new

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
