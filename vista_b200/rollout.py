"""The callers' loops around the sampler as engine-level operations (SURVEY.md §8f rows 2 and 3).

``rollout``         long-horizon autoregressive sampling, the body of ``sample_utils.do_sample``
                    (sample_utils.py:318-373; BASELINE config 4): round 1 conditioned on ``initial_cond_indices``, every
                    later round on the last three latents of the previous one, results stitched into ``samples_z``.
                    The latent bookkeeping between rounds (sample[0] = z[0], samples_z slices, fill_latent) is ONE kernel
                    (``b200v_rollout_advance``) on persistent device buffers, so nothing between two rounds waits for the
                    host; the reference's decode -> CLIP -> re-encode round trip between rounds is an optional callback
                    (``clip_recondition`` builds it on the native CLIP embedder, ``conditioner_recondition`` re-runs the
                    engine's whole conditioner as do_sample does).
``sample_ensemble`` the "reward" path (reward_utils.py:318-337): K samples of the same conditioning with different
                    noise, reward = exp(-mean variance); members are independent, so with a process group they are
                    dealt out over the ranks (replicas, no data-path collective except the final exchange).

Both call the engine's own sampler / denoiser / decoder — the fused B200 loop — and take injected noise (the reference
draws it with the device RNG, which is not reproducible across devices).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import torch

from . import ops
from .diffusion import B200Denoiser


def _masks(T: int, initial_cond_indices: Sequence[int], n_cond: int, device):
    init_mask = torch.zeros(T, device=device)
    pred_mask = torch.zeros(T, device=device)
    init_mask[list(initial_cond_indices)] = 1          # sample_utils.py:320-323
    pred_mask[list(range(n_cond))] = 1
    return init_mask, pred_mask


@torch.no_grad()
def rollout(engine, cond: Dict, uc: Dict, z: torch.Tensor, num_rounds: int, noises: Optional[List[torch.Tensor]] = None,
            recondition: Optional[Callable] = None, initial_cond_indices: Sequence[int] = (0,), n_cond: int = 3,
            decode: bool = True, u8: bool = False):
    """-> (frames or None, samples_z).  z: (T,4,h,w) scaled latents of the conditioning clip (encode_first_stage output);
    ``recondition(round, sample, decode_tail) -> (cond, uc)`` stands for sample_utils.py:340-348 (decode_tail() =
    decode_first_stage(sample[-14:]) for a CLIP re-encode; called lazily); without it ``cond["concat"]`` follows the
    reference's skip_encode rule, sample[[-n_cond]] / scale_factor (:343, encoders/modules.py:470-471), and the rest of the
    conditioning is kept.  frames: decode_first_stage(samples_z) clamped to [0,1] like :374 (fp32 NCHW), or uint8 NHWC."""
    T = z.shape[0]
    dev = z.device
    assert T == engine.num_frames and num_rounds >= 1 and 0 < n_cond < T
    den = B200Denoiser(engine.denoiser, engine.model)
    init_mask, pred_mask = _masks(T, initial_cond_indices, n_cond, dev)
    z = z.float().contiguous()
    samples_z = torch.zeros((num_rounds * (T - n_cond) + n_cond,) + tuple(z.shape[1:]), dtype=torch.float32, device=dev)
    filled = torch.zeros_like(z)
    draw = (lambda i: torch.randn_like(z)) if noises is None else (lambda i: noises[i].to(dev, torch.float32).clone().contiguous())

    sample = engine.sampler(den, draw(0), cond, uc=uc, cond_frame=z, cond_mask=init_mask)
    ops.rollout_advance(sample, z, samples_z, filled if num_rounds > 1 else None, 0, 0, n_cond)
    for n in range(num_rounds - 1):
        if recondition is not None:
            cond, uc = recondition(n + 1, sample, lambda s=sample: engine.decode_first_stage(s[-14:]))
        else:
            cond = dict(cond)
            rows = cond["concat"].shape[0]                      # get_batch repeats the frame (sample_utils.py:240-241)
            cond["concat"] = (sample[[-n_cond]] / engine.scale_factor).expand(rows, -1, -1, -1).contiguous()
        last = n + 2 == num_rounds
        sample = engine.sampler(den, draw(n + 1), cond, uc=uc, cond_frame=filled.clone(), cond_mask=pred_mask)
        ops.rollout_advance(sample, None, samples_z, None if last else filled, (n + 1) * (T - n_cond), n_cond, n_cond)
    if not decode:
        return None, samples_z
    if u8:
        return engine.decode_first_stage_u8(samples_z), samples_z
    x = engine.decode_first_stage(samples_z)
    return torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0), samples_z


def clip_recondition(embedder, cond: Dict, uc: Dict, scale_factor: float, n_cond: int = 3, clip_dim: int = 1024) -> Callable:
    """Opt-in ``recondition=`` callback for ``rollout`` that follows the reference between rounds (sample_utils.py:339-350):
    decode the tail, embed frame [-3] with ``embedder`` (a vista_b200.clip.FrozenOpenCLIPImagePredictionEmbedder; the frame
    is repeated over the conditioning rows as get_batch does, :243-244) into ``crossattn[..., :clip_dim]``, and set
    ``concat`` = sample[[-n_cond]] / scale_factor (the skip_encode rule).  The other crossattn slots and ``vector`` come
    from ``cond``; ``uc`` is returned as given (its CLIP and concat entries are zero per force_uc_zero_embeddings)."""
    def recondition(round_idx: int, sample: torch.Tensor, decode_tail: Callable):
        frames = decode_tail()
        c = dict(cond)
        rows = c["crossattn"].shape[0]
        emb = embedder(frames[[-3]].expand(rows, -1, -1, -1).contiguous())
        cross = c["crossattn"].clone()
        cross[..., :clip_dim] = emb.reshape(rows, 1, clip_dim).to(cross.dtype)
        c["crossattn"] = cross
        c["concat"] = (sample[[-n_cond]] / scale_factor).expand(c["concat"].shape[0], -1, -1, -1).contiguous()
        return c, uc
    return recondition


def conditioner_recondition(engine, value_dict: Dict, force_uc_zero_embeddings: Optional[Sequence[str]] = None,
                            n_cond: int = 3) -> Callable:
    """Opt-in ``recondition=`` callback for ``rollout`` that re-runs the engine's conditioner between rounds the way
    sample_utils.py:338-351 does: decoded frame [-n_cond] of the tail -> ``cond_frames_without_noise``,
    sample[[-n_cond]] / scale_factor -> ``cond_frames``, and ``engine.condition`` with ``skip_encode`` set on the embedders
    that have it (the latents pass through the cond-frame embedder).  ``value_dict`` is not modified."""
    def recondition(round_idx: int, sample: torch.Tensor, decode_tail: Callable):
        vd = dict(value_dict)
        vd["cond_frames_without_noise"] = decode_tail()[[-n_cond]]
        vd["cond_frames"] = sample[[-n_cond]] / engine.scale_factor
        toggled = [e for e in engine.conditioner.embedders if hasattr(e, "skip_encode")]
        for e in toggled:
            e.skip_encode = True
        try:
            return engine.condition(vd, engine.num_frames, force_uc_zero_embeddings)
        finally:
            for e in toggled:
                e.skip_encode = False
    return recondition


@torch.no_grad()
def sample_ensemble(engine, cond: Dict, uc: Dict, z: torch.Tensor, ensemble_size: int = 5,
                    noises: Optional[List[torch.Tensor]] = None, initial_cond_indices: Sequence[int] = (0,), group=None,
                    distributed: bool = False):
    """-> (reward 0-dim fp32 tensor, [members]).  reward_utils.py:318-337.  ``distributed``: member k is sampled by rank
    k % world of ``group`` and broadcast (every rank ends with all members and the same reward)."""
    T = z.shape[0]
    dev = z.device
    den = B200Denoiser(engine.denoiser, engine.model)
    init_mask, _ = _masks(T, initial_cond_indices, 1, dev)
    z = z.float().contiguous()
    world, rank = 1, 0
    if distributed:
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        to_global = (lambda r: r) if group is None else (lambda r: dist.get_global_rank(group, r))
    members = []
    for k in range(ensemble_size):
        if k % world == rank:
            noise = torch.randn_like(z) if noises is None else noises[k].to(dev, torch.float32).clone().contiguous()
            s = engine.sampler(den, noise, cond, uc=uc, cond_frame=z, cond_mask=init_mask)
            s[0] = z[0]                                       # reward_utils.py:324
            members.append(s.contiguous())
        else:
            members.append(torch.empty_like(z))
    if world > 1:
        for k in range(ensemble_size):
            dist.broadcast(members[k], src=to_global(k % world), group=group)
    out = ops.ensemble_reward(members)
    return out[1], members
