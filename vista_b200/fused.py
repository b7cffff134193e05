"""Fused EDM sampling loop on the B200 executor, for the Euler and the DPM-Solver++(2M) samplers.

Per step: ``sampler_prepare`` (cond-frame re-imposition, c_in scaling, CFG batch doubling, concat,
c_noise) -> UNet executor -> ``sampler_update`` (preconditioning, guidance, Euler step) or
``sampler_update_2m`` (the same denoised value, then the 2M step from the host's coefficient table).  Under action
guidance (``diffusion.ActionCFG``) a second, T-row forward runs the conditional half of the prepared batch under the
action-free conditioning, and ``sampler_update_action`` combines the three denoised values.  A step that is not guided
(``diffusion.IntervalCFG`` outside its interval, ``IdentityGuider``) runs only the conditional half of the prepared batch
through a T-row forward, then ``sampler_update_cond``; the host knows the schedule and replays each step's kind of graph.
Under feature caching (``cache_interval`` > 1, ``diffusion.cache_schedule``) a cached step is the same step with its
network calls cut to the outermost blocks (``UNetRuntime.forward(..., cached=True)``); it has a graph of its own.
All state
lives in persistent device buffers, the step index and sigma table are read on the device, so one
step is a fixed launch sequence that is captured once in a CUDA graph and replayed (no host
synchronisation inside the loop; the reference has two per step: sampling.py:102,109).

Semantics follow vwm/modules/diffusionmodules/sampling.py:91-124 with s_churn = 0 and
guiders.py:19-36,68-74; checked against the oracle in tests/test_sampler_gpu.py.
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Tuple

import torch

from . import lib as _lib
from . import ops
from .unet import padded_input_rows

USE_GRAPH = os.environ.get("VISTA_B200_GRAPH", "1") != "0"
USE_TAPE = os.environ.get("VISTA_B200_TAPE", "1") != "0"     # launch-tape replay of steps that hold collectives
COND_SLOT = "cond"     # the runtime's conditioning slot of the unguided steps' N rows (UNetRuntime.set_conditioning)


class _LoopState:
    """Persistent buffers + captured graph for one (N, h, w, num_steps) problem."""

    def __init__(self, rt, N: int, h: int, w: int):
        dev = rt.dev
        f32 = dict(dtype=torch.float32, device=dev)
        self.N, self.h, self.w = N, h, w
        self.x = torch.empty(N, 4, h, w, **f32)
        self.cond_frame = torch.zeros(N, 4, h, w, **f32)
        self.concat_u = torch.zeros(N, 4, h, w, **f32)
        self.concat_c = torch.zeros(N, 4, h, w, **f32)
        self.mask = torch.zeros(N, **f32)
        self.mask2 = torch.zeros(2 * N, **f32)
        self.scales = torch.ones(N, **f32)
        self.sigmas = torch.zeros(1024, **f32)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.c_noise = torch.empty(2 * N, **f32)
        self.unet_in = padded_input_rows(2 * N * h * w, dev)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.graph_steps = None
        # one captured step per (schedule length, 2M), and per (schedule length, 2M, True) under action guidance:
        # num_steps is a kernel argument, and the steps differ
        self.graphs: Dict[Tuple, torch.cuda.CUDAGraph] = {}
        self.coefs: Optional[torch.Tensor] = None     # 2M only: [1024, 4] fp32 {a, b, c, e} per step
        self.d_prev: Optional[torch.Tensor] = None    # 2M only: the previous step's denoised latent
        # action guidance only: per-frame s_act on the device (a captured graph replays the values set per sample), the
        # action-free conditioning of the conditional rows, and the output of the T-row forward that reads it
        self.action_scales: Optional[torch.Tensor] = None
        self.img_cond = None          # (crossattn, vector) of the N image rows, as last handed to the runtime
        self.net_img: Optional[torch.Tensor] = None
        self.tape, self.tape_steps = None, None      # launch tape of one step (frame-sharded runtimes)
        # CFG-split mode (modules.enable_frame_sharding): this rank runs one half of the doubled batch
        self.split = None            # (half, pair process group)
        self.net_full = None         # [2 N h w, 8] fp32: both halves' network outputs after the pair exchange
        self._fwd_out = None
        self.pair_peer = None        # peer-memory pair exchange (configure_split with a PeerWindow): dict of device arrays

    def configure_split(self, half: int, pair_group, win=None, partner: Optional[int] = None, rows_pad: Optional[int] = None):
        """win / partner: the rank's PeerWindow and the WINDOW rank of the other CFG half's owner of the same frames: the
        pair exchange then is two kernels over NVLink (put my half into the partner's net_full + flag, wait for its half)
        instead of an NCCL all-gather, and the whole step is graph-capturable."""
        self.split = (half, pair_group)
        rows = self.N * self.h * self.w
        if win is None:
            if self.net_full is None:
                self.net_full = torch.empty(2 * rows, 8, dtype=torch.float32, device=self.x.device)
            return
        dev = self.x.device
        # regions are sized by the LARGEST shard (rows_pad) so that every rank's window has the same layout
        rp = rows if rows_pad is None else rows_pad
        off = win.region(f"cfg.net_full.{rp}", 2 * rp * 8 * 4)
        foff = win.region(f"cfg.flags.{rp}", 1024)      # +0: partner's half has landed; +256: partner has consumed mine
        doff = win.region(f"cfg.ack_dummy.{rp}", 1024)
        self.net_full = win.tensor(off, (2 * rows, 8), torch.float32)
        half_bytes = rows * 8 * 4
        z = lambda name: win.counter(f"cfg.{rp}.{name}")     # counters live with the window (its flags outlive this state)
        self.pair_peer = dict(
            src=win.local(off + half * half_bytes), bytes=half_bytes,
            dst=win.ptr_array([win.remote(partner, off + half * half_bytes)]), dst_flag=win.ptr_array([win.remote(partner, foff)]),
            my_flag=win.ptr_array([win.local(foff)]),
            ack_src=win.local(doff), ack_dst=win.ptr_array([win.remote(partner, doff + 512)]),
            ack_flag_remote=win.ptr_array([win.remote(partner, foff + 256)]), ack_flag_mine=win.ptr_array([win.local(foff + 256)]),
            c_put=z("put"), t_put=z("ticket"), c_wait=z("wait"), c_ack_put=z("ack_put"), t_ack=z("ack_ticket"), c_ack_wait=z("ack_wait"))
        # prime the acknowledgement once per window: every step WAITS for "the partner has consumed my previous half" before
        # it stores, the very first step has nothing to wait for
        pp = self.pair_peer
        if win.once(f"cfg.{rp}.ack_primed"):
            ops.peer_put(pp["ack_src"], 16, 1, 16, pp["ack_dst"], 16, pp["ack_flag_remote"], 1, pp["c_ack_put"], pp["t_ack"], "cfg ack (prime)")

    def _prepare(self):
        ops.sampler_prepare(self.x, self.cond_frame, self.mask, self.concat_u, self.concat_c, self.sigmas, self.step,
                            self.unet_in, self.c_noise, self.N, self.h, self.w)

    def _forward(self, rt, cache=None):
        """``cache``: the keywords of a cached forward (``_cache_kw``), or None for a full one."""
        N, h, w = self.N, self.h, self.w
        if self.split is None:
            return rt.forward(self.unet_in, self.c_noise, self.mask2, h, w, **(cache or {}))
        half, rows = self.split[0], N * h * w
        out = self.net_full[half * rows:(half + 1) * rows] if self.pair_peer is not None else None   # straight into the exchange buffer
        return rt.forward(self.unet_in[half * rows:(half + 1) * rows], self.c_noise[half * N:(half + 1) * N],
                          self.mask2[half * N:(half + 1) * N], h, w, net_out=out)

    def _forward_img(self, rt, cache=None):
        """The action-free image branch: the conditional half of the prepared batch (rows bit for bit what the branch
        needs) through an N-row forward under the runtime's N-row conditioning."""
        N, h, w = self.N, self.h, self.w
        self.net_img = rt.forward(self.unet_in[N * h * w:], self.c_noise[N:], self.mask2[N:], h, w, **(cache or {}))
        return self.net_img

    def _forward_cond(self, rt, cache=None):
        """An unguided step's network call: the conditional half of the prepared batch through an N-row forward under
        the runtime's conditioning of the full ``c`` (its own slot, beside action guidance's action-free N rows)."""
        N, h, w = self.N, self.h, self.w
        return rt.forward(self.unet_in[N * h * w:], self.c_noise[N:], self.mask2[N:], h, w, slot=COND_SLOT,
                          **(cache or {}))

    @staticmethod
    def _cache_kw(cached: bool, cache_branch: int):
        """The forward keywords of a step: none for a full step (the launches of an uncached loop), the branch for a
        cached one.  The N-row forwards of ActionCFG's image branch and of unguided steps share their buffers; the cache
        schedule never lets a cached step follow a full step of the other kind."""
        return dict(cache_branch=cache_branch, cached=True) if cached else None

    def enable_action(self):
        """Allocates the per-frame action scale (once per state)."""
        if self.action_scales is None:
            self.action_scales = torch.zeros_like(self.scales)

    def enable_multistep(self):
        """Allocates the 2M sampler's coefficient table and D_prev buffer (once per state)."""
        if self.d_prev is None:
            self.coefs = torch.zeros(self.sigmas.numel(), 4, dtype=torch.float32, device=self.x.device)
            self.d_prev = torch.empty_like(self.x)

    def _finish(self, net_out, num_steps: int, multistep: bool = False, net_img=None):
        if self.split is not None and self.pair_peer is not None:
            # my half sits in net_full already (the output convolution wrote it there): store it into the partner's
            # net_full once the partner has consumed the previous step's (ack), raise its flag, wait for its half
            pp = self.pair_peer
            ops.peer_wait(pp["ack_flag_mine"], 1, pp["c_ack_wait"], "cfg ack")
            ops.peer_put(pp["src"], pp["bytes"], 1, pp["bytes"], pp["dst"], pp["bytes"], pp["dst_flag"], 1, pp["c_put"], pp["t_put"], "cfg half")
            ops.peer_wait(pp["my_flag"], 1, pp["c_wait"], "cfg half")
            net_out = self.net_full
        elif self.split is not None:                # guidance needs both halves of the frames this rank owns
            import torch.distributed as dist
            full, pg = self.net_full, self.split[1]
            _lib.tape_host(lambda src=net_out: dist.all_gather_into_tensor(full, src, group=pg), "cfg pair all_gather")   # bind now: net_out is rebound below
            net_out = full
        if net_img is not None:
            ops.sampler_update_action(self.x, net_out, net_img, self.cond_frame, self.mask, self.scales, self.action_scales,
                                      self.coefs if multistep else None, self.d_prev if multistep else None, self.sigmas,
                                      self.step, num_steps, self.N, self.h, self.w)
        elif multistep:
            ops.sampler_update_2m(self.x, net_out, self.cond_frame, self.mask, self.scales, self.coefs, self.d_prev,
                                  self.sigmas, self.step, num_steps, self.N, self.h, self.w)
        else:
            ops.sampler_update(self.x, net_out, self.cond_frame, self.mask, self.scales, self.sigmas, self.step,
                               num_steps, self.N, self.h, self.w)
        if self.split is not None and self.pair_peer is not None:      # the partner may overwrite my copy of its half now
            pp = self.pair_peer
            ops.peer_put(pp["ack_src"], 16, 1, 16, pp["ack_dst"], 16, pp["ack_flag_remote"], 1, pp["c_ack_put"], pp["t_ack"], "cfg ack")

    def one_step(self, rt, num_steps: int, multistep: bool = False, action: bool = False, guided: bool = True,
                 cached: bool = False, cache_branch: int = 0):
        """``cached``: run the step's network calls as cached forwards of branch ``cache_branch``; the update is the same."""
        cache = self._cache_kw(cached, cache_branch)
        self._prepare()
        if not guided:
            ops._sampler_update_cond(self.x, self._forward_cond(rt, cache), self.cond_frame, self.mask,
                                    self.coefs if multistep else None, self.d_prev if multistep else None, self.sigmas,
                                    self.step, num_steps, self.N, self.h, self.w)
            return
        net_out = self._forward(rt, cache)
        self._finish(net_out, num_steps, multistep, self._forward_img(rt, cache) if action else None)

    def runner(self, rt, num_steps: int, multistep: bool = False, action: bool = False, guided: bool = True,
               cached: bool = False, cache_branch: int = 0):
        """Callable advancing one step the fastest supported way; call after one eager step of the same kind (which
        allocates every buffer of the executor).  Without a collective inside the UNet the launch sequence is replayed
        from a CUDA graph: the whole step, or prepare + UNet in CFG-split mode (the pair exchange and the update stay
        eager)."""
        if not USE_GRAPH:
            return lambda: self.one_step(rt, num_steps, multistep, action, guided, cached, cache_branch)
        # NB: `rt.group is None` also names the DEFAULT process group; the runtime says whether its step holds collectives
        if getattr(rt, "has_collectives", False) and not USE_TAPE:
            return lambda: self.one_step(rt, num_steps, multistep, action)
        if getattr(rt, "has_collectives", False):
            # collectives inside the UNet: no graph; the first call records the step's C-ABI calls and host-side
            # collectives on a launch tape (vista_b200.lib), later calls replay it without the Python layers above
            def run_taped():
                if self.tape is None or self.tape_steps != num_steps:
                    _lib.begin_tape()
                    try:
                        self.one_step(rt, num_steps)
                    finally:
                        tape = _lib.end_tape()
                    self.tape, self.tape_steps = tape, num_steps
                else:
                    _lib.replay(self.tape)
            return run_taped
        if not guided:
            key = (num_steps, multistep, COND_SLOT)
        else:
            key = (num_steps, multistep, True) if action else (num_steps, multistep)
        if cached:
            key = key + ("cached", cache_branch)
        if key in self.graphs:
            self.graph, self.graph_steps = self.graphs[key], key
        if self.graph is None or self.graph_steps != key:
            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            whole = self.split is None or self.pair_peer is not None      # no host-side collective in the step
            with torch.cuda.graph(g):             # capture does not execute
                if whole:
                    self.one_step(rt, num_steps, multistep, action, guided, cached, cache_branch)
                else:
                    self._prepare()
                    self._fwd_out = self._forward(rt)
            self.graph, self.graph_steps = g, key
            self.graphs[key] = g
        if self.split is None or self.pair_peer is not None:
            return self.graph.replay

        def run():
            self.graph.replay()
            self._finish(self._fwd_out, num_steps)
        return run


def _expand(t: torch.Tensor, rows: int, T: int) -> torch.Tensor:
    if t.shape[0] == rows:
        return t
    assert t.shape[0] * T == rows, (t.shape, rows, T)
    return t.repeat_interleave(T, dim=0)


def fused_sample(sampler, den, x: torch.Tensor, cond: Dict, uc: Optional[Dict], cond_frame, cond_mask,
                 num_steps: Optional[int] = None) -> torch.Tensor:
    net = den.network
    T = den.denoiser.num_frames
    n = sampler.num_steps if num_steps is None else num_steps
    uc = cond if uc is None else uc
    dev = x.device
    N, zc, h, w = x.shape
    assert zc == 4 and N % T == 0
    from .diffusion import ActionCFG, DPMPP2MSampler, IdentityGuider, IntervalCFG, dpmpp2m_coefficients
    multistep = isinstance(sampler, DPMPP2MSampler)
    interval = sampler.guider if isinstance(sampler.guider, IntervalCFG) else None
    guider = interval.guider if interval is not None else sampler.guider
    action = isinstance(guider, ActionCFG)
    identity = isinstance(guider, IdentityGuider)
    if multistep and getattr(net, "frame_sharded", False):
        raise NotImplementedError("DPMPP2MSampler: the frame-sharded fused loop runs the Euler sampler only")
    if action and getattr(net, "frame_sharded", False):
        raise NotImplementedError("ActionCFG: the frame-sharded fused loop runs one guidance scale only")
    if (interval is not None or identity) and getattr(net, "frame_sharded", False):
        raise NotImplementedError(f"{type(sampler.guider).__name__}: the frame-sharded fused loop guides every step")
    cache_interval, cache_branch = sampler.cache_interval, sampler.cache_branch
    if cache_interval > 1 and getattr(net, "frame_sharded", False):
        raise NotImplementedError(f"{type(sampler).__name__}: the frame-sharded fused loop does not cache features")
    rt = net._rt_get(net.diffusion_model, T, dev)
    if getattr(net, "frame_sharded", False):
        return _fused_sample_sharded(sampler, rt, x, cond, uc, cond_frame, cond_mask, n, T, net)
    if cache_interval > 1 and not cache_branch < len(rt.plan.input_blocks):
        raise ValueError(f"cache_branch must be below the UNet's {len(rt.plan.input_blocks)} input blocks; got {cache_branch}")
    key = (N, h, w)
    states = rt.__dict__.setdefault("_loop_states", {})
    st: _LoopState = states.get(key)
    if st is None:
        st = states[key] = _LoopState(rt, N, h, w)
    assert n + 1 <= st.sigmas.numel()

    sigmas = sampler.discretization(n, device="cpu").to(torch.float32)
    x *= torch.sqrt(1.0 + sigmas[0] ** 2).to(x.device)            # sampling.py:36 (in place, like the reference)
    st.x.copy_(x)
    st.sigmas[: n + 1].copy_(sigmas)
    if multistep:
        st.enable_multistep()
        st.coefs[:n].copy_(dpmpp2m_coefficients(sigmas).to(torch.float32))
    st.step.zero_()
    if cond_frame is not None:
        st.cond_frame.copy_(cond_frame)
    if cond_mask is not None:
        st.mask.copy_(cond_mask)
    else:
        st.mask.zero_()
    st.mask2.copy_(torch.cat([st.mask, st.mask]))
    st.concat_u.copy_(_expand(uc["concat"], N, T))
    st.concat_c.copy_(_expand(cond["concat"], N, T))
    # which steps are guided, from the fp32 sigma table the kernels read; only the kinds of step that run are conditioned
    if identity:
        schedule = [False] * n
    elif interval is not None:
        schedule = [interval.guided(sigmas[i]) for i in range(n)]
    else:
        schedule = [True] * n
    if any(schedule):
        sv = guider.scale_vector(T).to(dev, torch.float32)
        st.scales.copy_(sv.repeat(N // T))
        context = torch.cat((_expand(uc["crossattn"], N, T), _expand(cond["crossattn"], N, T)), 0)
        y = torch.cat((_expand(uc["vector"], N, T), _expand(cond["vector"], N, T)), 0)
        rt.set_conditioning(context, y)
        if action:
            st.enable_action()
            st.action_scales.copy_(guider.action_scale_vector(T).to(dev, torch.float32).repeat(N // T))
            st.img_cond = (_expand(guider.action_free(cond)["crossattn"], N, T), y[N:])
            rt.set_conditioning(*st.img_cond)
    if not all(schedule):
        rt.set_conditioning(_expand(cond["crossattn"], N, T), _expand(cond["vector"], N, T), slot=COND_SLOT)
    if getattr(net, "_cond_cache", None) is not None:
        net._cond_cache = None      # the wrapper's own forward must set its conditioning again: this loop replaced it

    if cache_interval > 1:
        from .diffusion import cache_schedule
        _run_schedule(st, rt, n, multistep, action, schedule, cache_schedule(schedule, cache_interval), cache_branch)
    elif all(schedule):
        _run_steps(st, rt, n, multistep, action)
    else:
        _run_schedule(st, rt, n, multistep, action, schedule)
    x.copy_(st.x)
    return x


def _run_steps(st: _LoopState, rt, n: int, multistep: bool = False, action: bool = False):
    if n < 3:
        for _ in range(n):
            st.one_step(rt, n, multistep, action)
        return
    st.one_step(rt, n, multistep, action)       # eager first step: allocates every buffer of the executor
    step = st.runner(rt, n, multistep, action)
    for _ in range(n - 1):
        step()


def _run_schedule(st: _LoopState, rt, n: int, multistep: bool, action: bool, schedule, full=None, cache_branch: int = 0):
    """The steps of a schedule with unguided or cached steps: schedule[i] says whether step i is guided, full[i] (None:
    every step) whether it runs the whole UNet.  The first step of each kind runs eagerly, which allocates every buffer
    of the executor that kind of step uses; later ones replay its graph."""
    kinds = [(g, True if full is None else f) for g, f in zip(schedule, full or schedule)]
    if n < 3:
        for guided, whole in kinds:
            st.one_step(rt, n, multistep, action, guided, not whole, cache_branch)
        return
    seen = set()
    for kind in kinds:
        guided, whole = kind
        if kind not in seen:
            seen.add(kind)
            st.one_step(rt, n, multistep, action, guided, not whole, cache_branch)
        else:
            st.runner(rt, n, multistep, action, guided, not whole, cache_branch)()


def _fused_sample_sharded(sampler, rt, x, cond, uc, cond_frame, cond_mask, n: int, T: int, net=None) -> torch.Tensor:
    """One clip spread over the ranks (vista_b200/sharded.py): the frames are sharded, and with an even world size
    the two CFG halves too.  Every rank receives the same full-clip inputs, advances the frames it owns and the
    final latent is all-gathered."""
    from .sharded import gather_latent
    dev = x.device
    N, zc, h, w = x.shape
    assert N == T, "sharded sampling handles one clip"
    t0, t1 = rt.t0, rt.t1
    Tl = t1 - t0
    half = getattr(rt, "cfg_half", None)
    states = rt.__dict__.setdefault("_loop_states", {})
    st = states.get((Tl, h, w))
    if st is None:
        # NVLink peer window (collective on first use): the step's exchanges become kernels, the step a CUDA graph
        win = net.peer_window(T, h, w, rt.cfg.model_channels, dev) if net is not None else None
        if win is not None and hasattr(rt, "attach_window"):
            rt.attach_window(win)
        st = states[(Tl, h, w)] = _LoopState(rt, Tl, h, w)
        if half is not None:
            partner = (win.rank + win.world // 2) % win.world if win is not None else None
            st.configure_split(half, rt.pair_group, win, partner, rows_pad=getattr(rt, "T_pad", Tl) * h * w)
    sigmas = sampler.discretization(n, device="cpu").to(torch.float32)
    x *= torch.sqrt(1.0 + sigmas[0] ** 2).to(dev)
    st.x.copy_(x[t0:t1])
    st.sigmas[: n + 1].copy_(sigmas)
    st.step.zero_()
    if cond_frame is not None:
        st.cond_frame.copy_(cond_frame[t0:t1])
    if cond_mask is not None:
        st.mask.copy_(cond_mask[t0:t1])
    else:
        st.mask.zero_()
    st.mask2.copy_(torch.cat([st.mask, st.mask]))
    st.concat_u.copy_(_expand(uc["concat"], N, T)[t0:t1])
    st.concat_c.copy_(_expand(cond["concat"], N, T)[t0:t1])
    st.scales.copy_(sampler.guider.scale_vector(T).to(dev, torch.float32)[t0:t1])
    if half is None:
        context = torch.cat((_expand(uc["crossattn"], N, T), _expand(cond["crossattn"], N, T)), 0)
        y = torch.cat((_expand(uc["vector"], N, T), _expand(cond["vector"], N, T)), 0)
    else:
        src = uc if half == 0 else cond
        context, y = _expand(src["crossattn"], N, T), _expand(src["vector"], N, T)
    rt.set_conditioning(context, y)
    _run_steps(st, rt, n)
    if Tl == T:
        x.copy_(st.x)
    else:
        x.copy_(gather_latent(st.x, T, group=rt.group))
    return x
