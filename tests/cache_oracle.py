"""Feature caching over the fp32 oracle (oracle/vista_oracle.py).

``unet_forward`` is ``vo.unet_forward`` (video_model.py:442-503) with a cache: built from the oracle's own layer
functions, it records the tensor entering output block n-1-b on a full call and starts the up-path from it on a cached
one; without a cache it is ``vo.unet_forward`` operation for operation (tests/test_feature_cache_cpu.py holds it
``torch.equal`` to it).  ``oracle_sample`` runs the samplers' own torch loop, Euler or 2M under any guider, around
``denoise`` whose network calls follow ``diffusion.cache_schedule``.  Every per-clip operation of the UNet is row-block
independent, so one 3T-row oracle call of ActionCFG caches what the fused loop's 2T- and T-row calls cache."""
import copy
from typing import Optional

import torch
import torch.nn.functional as F

from oracle import vista_oracle as vo
from vista_b200.spec import ConvSpec, ResBlockSpec, SVTSpec, build_unet_plan


def unet_forward(sd, cfg, x, timesteps, context, y, cond_mask, num_frames: int, cache: Optional[dict] = None):
    """``vo.unet_forward`` with ``cache`` (feature caching, Ma et al. 2024, DeepCache): a dict with the branch b as
    "branch".  With no "h" in it the forward runs whole and stores the tensor entering output block n-1-b (the h before
    its torch.cat) as "h"; with "h" it runs input blocks 0..b, starts output block n-1-b from that tensor and skips every
    deeper block."""
    plan = build_unet_plan(cfg)
    t_emb = vo.timestep_embedding(timesteps, cfg.model_channels)
    if cond_mask is not None and bool(cond_mask.any()):
        m = cond_mask[..., None].float()
        emb = vo._mlp(sd, "cond_time_stack_embed.0", "cond_time_stack_embed.2", t_emb) * m \
            + vo._mlp(sd, "time_embed.0", "time_embed.2", t_emb) * (1 - m)
    else:
        emb = vo._mlp(sd, "time_embed.0", "time_embed.2", t_emb)
    emb = emb + vo._mlp(sd, "label_emb.0.0", "label_emb.0.2", y)

    def run(block, h):
        for layer in block.layers:
            if isinstance(layer, ResBlockSpec):
                h = vo.video_res_block(sd, layer, h, emb, num_frames)
            elif isinstance(layer, SVTSpec):
                h = vo.spatial_video_transformer(sd, layer, h, context, num_frames, cfg.context_dim)
            elif isinstance(layer, ConvSpec):
                wgt, b = sd[f"{layer.prefix}.weight"], sd[f"{layer.prefix}.bias"]
                if layer.kind == "down":
                    h = F.conv2d(h, wgt, b, stride=2, padding=1)
                elif layer.kind == "up":
                    h = F.conv2d(F.interpolate(h, scale_factor=2, mode="nearest"), wgt, b, padding=1)
                else:
                    h = F.conv2d(h, wgt, b, padding=1)
        return h

    n = len(plan.output_blocks)
    j0 = n - 1 - cache["branch"] if cache is not None else 0
    reuse = cache is not None and cache.get("h") is not None
    hs = []
    h = x
    for i, blk in enumerate(plan.input_blocks):
        if reuse and i > cache["branch"]:
            break
        h = run(blk, h)
        hs.append(h)
    h = cache["h"] if reuse else run(plan.middle_block, h)
    for j, blk in enumerate(plan.output_blocks):
        if reuse and j < j0:
            continue
        if j == j0 and cache is not None and not reuse:
            cache["h"] = h
        h = run(blk, torch.cat((h, hs.pop()), dim=1))
    h = F.silu(vo._gn(sd, "out.0", h, 1e-5))
    return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)


def wrapper_forward(sd, cfg, x, t, c: dict, cond_mask, num_frames: int, cache: Optional[dict] = None):
    """``vo.wrapper_forward`` (wrappers.py:25-40) over ``unet_forward`` with ``cache``."""
    concat = c["concat"]
    if concat.shape[0] != x.shape[0]:
        concat = concat.repeat_interleave(num_frames, dim=0)
    return unet_forward(sd, cfg, torch.cat((x, concat), dim=1), t, c["crossattn"], c["vector"], cond_mask, num_frames,
                        cache)


def denoise(sd, cfg, x, sigma, c, cond_mask, num_frames: int, cache: Optional[dict] = None):
    """``vo.denoise`` (denoiser.py:22-35) over ``wrapper_forward`` with ``cache``."""
    s = sigma[:, None, None, None]
    c_skip, c_out, c_in, c_noise = vo.vscaling_edm_cnoise(s)
    net = wrapper_forward(sd, cfg, x * c_in, c_noise.reshape(sigma.shape), c, cond_mask, num_frames, cache)
    return net * c_out + x * c_skip


class CachedOracleDenoiser:
    """``(x, sigma, c, cond_mask)`` denoiser of the torch loop: call i is step i, full where ``full[i]``."""

    def __init__(self, sd, cfg, full, branch: int, num_frames: int = 25):
        self.sd, self.cfg, self.full, self.branch, self.T = sd, cfg, list(full), branch, num_frames
        self.calls, self.cache = 0, None

    def __call__(self, x, sigma, c, cond_mask):
        if self.full[self.calls]:
            self.cache = {"branch": self.branch}
        else:
            assert self.cache["h"].shape[0] == x.shape[0], "a cached step follows a full step of other rows"
        self.calls += 1
        with torch.device(x.device):           # the oracle's timestep embedding builds its tables on the default device
            return denoise(self.sd, self.cfg, x, sigma, c, cond_mask, self.T, self.cache)


def step_kinds(sampler, n: int):
    """Whether each of the n steps is guided, from the fp32 sigma table the loops read (fused.fused_sample's rule)."""
    from vista_b200.diffusion import IdentityGuider, IntervalCFG
    g = sampler.guider
    if isinstance(g, IdentityGuider):
        return [False] * n
    if isinstance(g, IntervalCFG):
        sig = sampler.discretization(n, device="cpu").to(torch.float32)
        return [g.guided(sig[i]) for i in range(n)]
    return [True] * n


def oracle_sample(sampler, sd, cfg, noise, c, uc, cond_frame, cond_mask, num_frames: int = 25):
    """``sampler`` (cache_interval k, cache_branch b) restated: its torch loop with caching off, over the oracle cached
    on the schedule cache_schedule(kinds, k) -> (sample, the schedule)."""
    from vista_b200.diffusion import cache_schedule
    n = sampler.num_steps
    full = cache_schedule(step_kinds(sampler, n), sampler.cache_interval)
    plain = copy.copy(sampler)
    plain.cache_interval = 1
    den = CachedOracleDenoiser(sd, cfg, full, sampler.cache_branch, num_frames)
    with torch.no_grad():
        out = plain(den, noise.clone(), c, uc=uc, cond_frame=cond_frame, cond_mask=cond_mask)
    assert den.calls == n
    return out, full
