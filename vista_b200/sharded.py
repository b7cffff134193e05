"""Frame-sharded execution of ONE clip over several GPUs (BASELINE config 5, SURVEY.md §8e).

Rank r owns a contiguous range of the T frames of the clip — for both CFG halves — and runs every
spatial operator (2-D convolutions, per-frame GroupNorm, spatial attention, feed-forwards) locally.
The three temporal couplings of the UNet cross ranks:

  * temporal self-attention (video_attention.py:127): each query frame needs K, V of all T frames of its
    pixel -> ONE all-gather of the K|V projection per SpatialVideoTransformer (the collective named in
    BASELINE.json), consumed in place by ``b200v_attention_temporal_sharded`` through a frame table;
  * the temporal ResBlock's GroupNorm over (C/32, T, H, W) (video_model.py:67-72): fixed-order local sums,
    an all-reduce of [clips, 32, 2] fp64 values, finalisation with the global element count;
  * the (3,1,1) convolution (video_model.py:38-52): the local zero-padded conv plus two one-frame halo
    corrections  out[first frame] += W_tap0 x prev-rank's last frame,  out[last frame] += W_tap2 x next-rank's
    first frame  (linearity of the convolution), the halos travelling by point-to-point send/recv.

Weights are replicated.  The sampler state is frame-local too; the latent is all-gathered once at the end.

Two transports.  With an NVLink peer window attached (``attach_window``; the CFG-split layouts, one clip per rank) the three
couplings are KERNELS over peer memory (csrc/peer.cu): the K|V projection writes its slab straight into the window and
``peer_put`` stores it into every peer's window; the GroupNorm sums go through the rank-ordered ``peer_allreduce_f64`` (fused
statistics stay on); the boundary frames are stored into the neighbours' halo slots of a halo-extended buffer and the
convolution runs ONCE (tap-GEMM ``h_pad``).  No communicator call is left in the step, which is replayed from a CUDA graph.
Otherwise (frames-only layouts, VISTA_B200_PEER=0) torch.distributed / NCCL carries them as described above and the step is
replayed from a launch tape.  Either way the math stays in the C-ABI kernels.

With an even number of ranks the classifier-free-guidance batch is split first (modules.enable_frame_sharding):
ranks [0, W/2) run the unconditional clip, ranks [W/2, W) the conditional one, each half sharding the frames
over W/2 ranks with the collectives above inside its own sub-group; the only traffic between the halves is the
4-channel network output of a rank's frames, exchanged pairwise once per step for the guidance (fused.py).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from . import lib as _lib
from . import ops
from .parallel import frame_shards, halo_neighbours
from .spec import UNetConfig
from .unet import Lin, UNetRuntime


class HaloExchange:
    """One-frame halo exchange of a (3,1,1) convolution between frame-shard neighbours: the first local frame goes to
    the previous rank, the last one to the next rank, their boundary frames come back.  `start` / `wait` are plain
    host callables so that they can sit on the launch tape (vista_b200.lib) between the kernels and be replayed;
    `first` / `last` = (staging view, source view, send buffer, receive buffer).  Peers are GLOBAL ranks."""

    def __init__(self, group, prev: Optional[int], nxt: Optional[int], first, last):
        self.copies, self.p2p, self.pending = [], [], []
        if prev is not None:
            stage, src, send, recv = first
            self.copies.append((stage, src))
            self.p2p.append(dist.P2POp(dist.isend, send, prev, group))
            self.p2p.append(dist.P2POp(dist.irecv, recv, prev, group))
        if nxt is not None:
            stage, src, send, recv = last
            self.copies.append((stage, src))
            self.p2p.append(dist.P2POp(dist.isend, send, nxt, group))
            self.p2p.append(dist.P2POp(dist.irecv, recv, nxt, group))

    def start(self):
        for dst, src in self.copies:
            dst.copy_(src)
        self.pending = list(dist.batch_isend_irecv(self.p2p)) if self.p2p else []

    def wait(self):
        for r in self.pending:
            r.wait()
        self.pending = []


class ShardedUNetRuntime(UNetRuntime):
    has_collectives = True        # its step issues NCCL calls: never CUDA-graph-captured, replayed from the launch tape

    def __init__(self, cfg: UNetConfig, sd: Dict[str, torch.Tensor], device, num_frames: int = 25, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.T_full = num_frames
        self.shards = frame_shards(num_frames, self.world)
        self.t0, self.t1 = self.shards[self.rank]
        self.T_pad = max(b - a for a, b in self.shards)
        super().__init__(cfg, sd, device, num_frames=self.t1 - self.t0)     # self.T = local frames per clip
        prev, nxt = halo_neighbours(self.rank, self.world)
        to_global = (lambda r: r) if group is None else (lambda r: dist.get_global_rank(group, r))
        self.prev = None if prev is None else to_global(prev)       # P2POp peers are global ranks
        self.next = None if nxt is None else to_global(nxt)
        self._tap_w: Dict[int, tuple] = {}
        self._frame_tables: Dict[tuple, torch.Tensor] = {}
        self.comm_bytes = 0
        self.win = None               # PeerWindow (attach_window): the exchanges below become kernels over NVLink
        self._ext: Dict[tuple, tuple] = {}
        self._ext_of: Dict[int, tuple] = {}
        self._peer_state: Dict[str, dict] = {}

    # ------------------------------------------------------------------ NVLink peer-memory path
    def attach_window(self, win):
        """win: vista_b200.peer.PeerWindow over the group the clip is spread over.  With it (and one clip per rank, the
        CFG-split layouts) the temporal couplings are stores into the neighbours' windows plus flags (csrc/peer.cu): no NCCL
        call in the step, which then is a fixed launch sequence and replayed from a CUDA graph like the single-GPU one."""
        self.win = win
        self.has_collectives = False
        # window ranks of the members of this runtime's frame group, in shard order
        granks = list(range(self.world)) if self.group is None else dist.get_process_group_ranks(self.group)
        wranks = list(range(win.world)) if win.group is None else dist.get_process_group_ranks(win.group)
        self.wr = [wranks.index(g) for g in granks]          # shard index -> window rank
        W = self.world
        # GroupNorm all-reduce: slots [2 parities][16][max doubles] + flags [2][16], in every window at the same offsets
        amax = ops._lib.load().b200v_peer_allreduce_max()
        self._ar = dict(slot=win.region("gn.ar.slots", 2 * 16 * amax * 8), flag=win.region("gn.ar.flags", 2 * 16 * 4), counter=win.counter("gn.ar"))
        # the all-reduce kernel indexes windows by SHARD index: hand it this group's windows in shard order
        self._ar["windows"] = win.ptr_array([win.bases[r] for r in self.wr])
        # halo flags: +0 raised by the previous shard (its last frame has landed in my slot 0), +256 by the next shard
        hf = win.region("halo.flags", 1024)
        me = self.rank
        st = dict(c_put_prev=win.counter("halo.put_prev"), t_put_prev=win.counter("halo.ticket_prev"),
                  c_put_next=win.counter("halo.put_next"), t_put_next=win.counter("halo.ticket_next"), c_wait=win.counter("halo.wait"))
        wait = []
        if me > 0:
            st["flag_on_prev"] = win.ptr_array([win.remote(self.wr[me - 1], hf + 256)])     # I am its next shard
            wait.append(win.local(hf))
        if me < W - 1:
            st["flag_on_next"] = win.ptr_array([win.remote(self.wr[me + 1], hf)])
            wait.append(win.local(hf + 256))
        st["wait"] = win.ptr_array(wait) if wait else None
        st["n_wait"] = len(wait)
        self._halo = st
        kf = win.region("kv.flags", 16 * 256)
        peers = [r for r in range(W) if r != me]
        self._kv = dict(flag_off=kf, peers=peers, c_put=win.counter("kv.put"), t_put=win.counter("kv.ticket"), c_wait=win.counter("kv.wait"),
                        flags_remote=win.ptr_array([win.remote(self.wr[r], kf + me * 256) for r in peers]),
                        flags_local=win.ptr_array([win.local(kf + r * 256) for r in peers]))

    def _peer_on(self, nb: int) -> bool:
        return self.win is not None and nb == 1

    def _ext_buffer(self, hw: int, Cc: int, which: int):
        """Halo-extended activation of a temporal convolution in the window: frames [prev halo | T local | next halo] (+ unused
        slots up to T_pad + 2 so that the layout is the same on every rank).  Zeroed at allocation: the clip ends keep their
        zero halo = the convolution's zero padding (openaimodel.py:190-193)."""
        key = (hw, Cc, which)
        hit = self._ext.get(key)
        if hit is None:
            fb = hw * Cc * 2
            off = self.win.region(f"ext.{hw}.{Cc}.{which}", (self.T_pad + 2) * fb)
            ext = self.win.tensor(off, ((self.T + 2) * hw, Cc), torch.float16)
            mid = ext[hw:(self.T + 1) * hw]
            hit = self._ext[key] = (ext, mid, off, fb)
            self._ext_of[mid.data_ptr()] = hit
        return hit

    # ------------------------------------------------------------------ conditioning
    def set_conditioning(self, context: torch.Tensor, y: torch.Tensor):
        """context / y hold the rows of the WHOLE clip(s): (nb*T_full, ...).  The frame-index embedding and the
        temporal cross-attention constant follow the global frame numbering (video_attention.py:256,270-279)."""
        Tf, T = self.T_full, self.T
        nb = context.shape[0] // Tf
        ctx = context.reshape(nb, Tf, -1)
        yy = y.reshape(nb, Tf, -1)
        local_ctx = ctx[:, self.t0:self.t1].reshape(nb * T, 1, -1)
        local_y = yy[:, self.t0:self.t1].reshape(nb * T, -1)
        # time context = context of the first frame of every clip, whoever owns it
        first_ctx = ctx[:, :1].reshape(nb, 1, -1)
        super().set_conditioning(local_ctx, local_y)
        cond = self.cond
        t16 = self.buf("cond.tctx", nb, first_ctx.numel() // nb)
        t16.copy_(first_ctx.reshape(nb, -1))
        frames = torch.arange(Tf, dtype=torch.float32, device=self.dev)
        for t in self.plan.transformers():
            L = self.layers[t.prefix]
            cond["tm"][t.prefix] = self._attn2_const(L["tattn2"], t16, f"cond.tm.{t.prefix}")
            temb = self.buf("cond.temb_full", Tf, t.ch)
            ops.timestep_embedding(frames, temb, t.ch)
            full = self._mlp(temb, *L["pos"], f"cond.posfull.{t.prefix}")
            cond["pos"][t.prefix] = full[self.t0:self.t1]          # rows of the local frames, contiguous view

    # ------------------------------------------------------------------ temporal GroupNorm
    def _fuse_stats(self, B, h, w) -> bool:
        # NCCL path: the (3,1,1) convolutions get their halo corrections AFTER the main launch, statistics taken in its epilogue
        # would miss them -> separate statistics pass.  Peer path: the halos are in place before the ONE launch, the fused
        # statistics are exact again.
        if self._peer_on(B // self.T):
            return super()._fuse_stats(B, h, w)
        return False

    def _gn_temporal(self, x, y, B, hw, norm, eps, silu, idx, fps, part=None):
        nb = B // fps
        Cc = norm[0].numel()
        sums = self.buf(f"gn.sums{nb}", nb * self.cfg.num_groups, 2, torch.float64)
        if part is not None:       # this rank's raw sums from the column partials its producing GEMM wrote
            ops.groupnorm_from_partials(part, B, hw, Cc, eps, None, fps, self.cfg.num_groups, raw_sums=sums)
        else:
            ops.groupnorm_sums(x, B, hw, Cc, sums, fps, groups=self.cfg.num_groups, ws=self.gn_ws)
        if self._peer_on(nb):
            ar = self._ar
            ops.peer_allreduce_f64(sums.view(-1), ar["windows"], ar["slot"], ar["flag"], self.rank, self.world, ar["counter"])
            # the normalised activation goes straight into the halo-extended buffer of the (3,1,1) convolution that follows
            which = 0 if y.data_ptr() == self.buf("rb.a1", y.shape[0], y.shape[1]).data_ptr() else 1
            y = self._ext_buffer(hw, Cc, which)[1]
        else:
            _lib.tape_host(lambda: dist.all_reduce(sums, group=self.group), "gn-sum all_reduce")
        self.comm_bytes += sums.numel() * 8
        count = float(Cc // self.cfg.num_groups) * hw * self.T_full
        return ops.groupnorm_finalize_apply(x, y, B, hw, norm[0], norm[1], eps, silu, sums, count,
                                            self.gn_stats[idx, :nb], fps, groups=self.cfg.num_groups)

    # ------------------------------------------------------------------ temporal convolution with halos
    def _tap_weights(self, lin: Lin):
        key = lin.w.data_ptr()
        tw = self._tap_w.get(key)
        if tw is None:
            Cc = lin.w.shape[1] // 3
            tw = (Lin(lin.w[:, :Cc].contiguous(), None, lin.tile_n), Lin(lin.w[:, 2 * Cc:].contiguous(), None, lin.tile_n))
            self._tap_w[key] = tw
        return tw

    def _tconv(self, a, lin: Lin, out, hw: int, nb: int, **epi):
        T, Cc = self.T, a.shape[1]
        ext = self._ext_of.get(a.data_ptr()) if self._peer_on(nb) else None
        if ext is not None:
            # my boundary frames -> the neighbours' halo slots (NVLink stores + flag), wait for theirs, ONE convolution over
            # the extended tensor (h_pad = 1): no correction GEMMs, fused statistics stay valid
            ext_t, _, off, fb = ext
            h, win, me = self._halo, self.win, self.rank
            if me > 0:          # first frame -> slot T_prev + 1 of the previous shard's buffer
                t_prev = self.shards[me - 1][1] - self.shards[me - 1][0]
                dst = self._peer_ptrs(("hp", off, fb), lambda: [win.remote(self.wr[me - 1], off + (t_prev + 1) * fb)])
                ops.peer_put(a.data_ptr(), fb, 1, fb, dst, fb, h["flag_on_prev"], 1, h["c_put_prev"], h["t_put_prev"], "halo->prev")
            if me < self.world - 1:   # last frame -> slot 0 of the next shard's buffer
                dst = self._peer_ptrs(("hn", off, fb), lambda: [win.remote(self.wr[me + 1], off)])
                ops.peer_put(a.data_ptr() + (T - 1) * fb, fb, 1, fb, dst, fb, h["flag_on_next"], 1, h["c_put_next"], h["t_put_next"], "halo->next")
            if h["n_wait"]:
                ops.peer_wait(h["wait"], h["n_wait"], h["c_wait"], "halo")
            self.comm_bytes += fb * ((me > 0) + (me < self.world - 1))
            return self.gemm(ext_t, lin, out, taps=ops.TAPS_T3, geom=(hw, T, nb), h_pad=1, **epi)
        # boundary frames of the input go to the neighbours while the local convolution runs
        send_first = self.buf("halo.sf", nb * hw, Cc)
        send_last = self.buf("halo.sl", nb * hw, Cc)
        recv_prev = self.buf("halo.rp", nb * hw, Cc)
        recv_next = self.buf("halo.rn", nb * hw, Cc)
        a4 = a.reshape(nb, T, hw, Cc) if a.is_contiguous() else None
        av = a4 if a4 is not None else a.as_strided((nb, T, hw, Cc), (T * hw * a.stride(0), hw * a.stride(0), a.stride(0), 1))
        halo = HaloExchange(self.group, self.prev, self.next,
                            first=(send_first.view(nb, hw, Cc), av[:, 0], send_first, recv_prev),
                            last=(send_last.view(nb, hw, Cc), av[:, T - 1], send_last, recv_next))
        start_halo, wait_halo = halo.start, halo.wait
        _lib.tape_host(start_halo, "halo copy + isend/irecv")
        self.comm_bytes += 2 * nb * hw * Cc * 2 * ((self.prev is not None) + (self.next is not None))
        self.gemm(a, lin, out, taps=ops.TAPS_T3, geom=(hw, T, nb), **epi)
        _lib.tape_host(wait_halo, "halo wait")
        s_acc = epi.get("s_acc", 1.0)
        w0, w2 = self._tap_weights(lin)
        ov = out.as_strided((nb, T, hw, out.shape[1]), (T * hw * out.stride(0), hw * out.stride(0), out.stride(0), 1))
        for b in range(nb):
            if self.prev is not None:      # frame t0-1 contributes through tap 0 to our first frame
                o = ov[b, 0]
                self.gemm(recv_prev[b * hw:(b + 1) * hw], w0, o, s_acc=s_acc, res1=o)
            if self.next is not None:      # frame t1 contributes through tap 2 to our last frame
                o = ov[b, T - 1]
                self.gemm(recv_next[b * hw:(b + 1) * hw], w2, o, s_acc=s_acc, res1=o)
        return out

    def _peer_ptrs(self, key, make):
        t = self._peer_state.get(key)
        if t is None:
            t = self._peer_state[key] = self.win.ptr_array(make())
        return t

    # ------------------------------------------------------------------ temporal attention with gathered K|V
    def _frame_table(self, nb: int, hw: int) -> torch.Tensor:
        key = (nb, hw)
        tab = self._frame_tables.get(key)
        if tab is None:
            rows = []
            for b in range(nb):
                for t in range(self.T_full):
                    r = next(i for i, (a, e) in enumerate(self.shards) if a <= t < e)
                    tl = t - self.shards[r][0]
                    rows.append(((r * nb + b) * self.T_pad + tl) * hw)
            tab = torch.tensor(rows, dtype=torch.int64, device=self.dev)
            self._frame_tables[key] = tab
        return tab

    def _kv_direct(self, nb: int) -> bool:
        """The K|V projection can be written straight into the all-gather's send layout when that layout has no padding
        rows between the clips of this rank: one clip (the CFG-split layouts), or every rank owning T_pad frames."""
        return nb == 1 or self.T == self.T_pad

    def _svt_tqkv(self, n, L, M: int, Cc: int, nb: int, hw: int):
        """q|k|v projection of the temporal attention.  Direct mode: two launches over the row blocks of the fused weight —
        q into the q buffer, K|V straight into the send buffer of the all-gather (no staging copy of the largest tensor of
        the exchange); otherwise the fused projection (the copy happens in _attn_temporal)."""
        if not self._kv_direct(nb):
            return super()._svt_tqkv(n, L, M, Cc, nb, hw)
        lin = L["tqkv"]
        sub = self._tap_w.get(("qkv", lin.w.data_ptr()))
        if sub is None:
            sub = (Lin(lin.w[:Cc], None, ops.pick_tile_n(Cc)), Lin(lin.w[Cc:], None, ops.pick_tile_n(2 * Cc)))
            self._tap_w[("qkv", lin.w.data_ptr())] = sub
        qkv = self.buf("tr.qkv", M, 3 * Cc)
        send = self._kv_recv(nb, hw, Cc)[1] if self._peer_on(nb) else self.buf("kv.send", nb * self.T_pad * hw, 2 * Cc)
        self.gemm(n, sub[0], qkv[:, :Cc])
        self.gemm(n, sub[1], send[:M])
        return qkv

    def _kv_recv(self, nb: int, hw: int, Cc: int):
        """(gathered K|V [W * T_pad * hw, 2C] in the window, this rank's slab of it, slab bytes, region offset)."""
        key = ("kv", hw, Cc)
        hit = self._peer_state.get(key)
        if hit is None:
            slab = self.T_pad * hw * 2 * Cc * 2
            # one region for every level: the first transformer met (highest resolution) has the largest K|V; region()
            # refuses a later, larger request instead of overlapping a neighbour
            off = self.win.region("kv.recv", self.world * slab)
            recv = self.win.tensor(off, (self.world * self.T_pad * hw, 2 * Cc), torch.float16)
            mine = recv[self.rank * self.T_pad * hw:(self.rank + 1) * self.T_pad * hw]
            dsts = self.win.ptr_array([self.win.remote(self.wr[r], off + self.rank * slab) for r in self._kv["peers"]])
            hit = self._peer_state[key] = (recv, mine, slab, off, dsts)
        return hit

    def _attn_temporal(self, qkv, o, nb: int, hw: int, heads: int, Cc: int):
        T, Tp, W = self.T, self.T_pad, self.world
        if self._peer_on(nb):
            # all-gather by stores: my K|V slab (written by the projection GEMM into my own window) goes to the same slab of
            # every peer's window, one flag per (peer, source); then wait for the W - 1 slabs addressed to me
            recv, mine, slab, off, dsts = self._kv_recv(nb, hw, Cc)
            kv = self._kv
            nbytes = T * hw * 2 * Cc * 2
            ops.peer_put(mine.data_ptr(), nbytes, 1, nbytes, dsts, nbytes, kv["flags_remote"], len(kv["peers"]), kv["c_put"], kv["t_put"],
                         f"kv C={Cc} hw={hw}")
            ops.peer_wait(kv["flags_local"], len(kv["peers"]), kv["c_wait"], "kv")
            self.comm_bytes += nbytes * len(kv["peers"])
            tab = self._frame_table(nb, hw)
            return ops.attention_temporal_sharded(qkv[:, :Cc], recv[:, :Cc], recv[:, Cc:], o, nb, T, self.T_full, hw, heads, tab)
        send = self.buf("kv.send", nb * Tp * hw, 2 * Cc)
        recv = self.buf("kv.recv", W * nb * Tp * hw, 2 * Cc)
        if not self._kv_direct(nb):
            # the K|V column block of the fused q|k|v projection as a strided (clip, frame, pixel, 2C) view
            kv = qkv.as_strided((nb, T, hw, 2 * Cc), (T * hw * qkv.stride(0), hw * qkv.stride(0), qkv.stride(0), 1),
                                qkv.storage_offset() + Cc)
            dst = send.view(nb, Tp, hw, 2 * Cc)[:, :T]
            _lib.tape_host(lambda: dst.copy_(kv), "kv staging copy")
        _lib.tape_host(lambda: dist.all_gather_into_tensor(recv, send, group=self.group), f"kv all_gather C={Cc} hw={hw}")
        self.comm_bytes += recv.numel() * 2
        tab = self._frame_table(nb, hw)
        return ops.attention_temporal_sharded(qkv[:, :Cc], recv[:, :Cc], recv[:, Cc:], o, nb, T, self.T_full, hw, heads, tab)


def gather_latent(x_local: torch.Tensor, num_frames: int, group=None) -> torch.Tensor:
    """All-gather of the frame-sharded latent (T_loc,4,h,w) -> (T,4,h,w) on every rank."""
    world = dist.get_world_size(group)
    shards = frame_shards(num_frames, world)
    pad = max(b - a for a, b in shards)
    buf = x_local.new_zeros((pad,) + tuple(x_local.shape[1:]))
    buf[: x_local.shape[0]] = x_local
    out = x_local.new_empty((world * pad,) + tuple(x_local.shape[1:]))
    dist.all_gather_into_tensor(out, buf, group=group)
    parts = out.reshape(world, pad, *x_local.shape[1:])
    return torch.cat([parts[r, : b - a] for r, (a, b) in enumerate(shards)], dim=0)


# ---------------------------------------------------------------------------------------------------------------
# Frame-sharded VAE decode: the frames of every decode chunk are spread over the ranks with the NCCL mechanisms of the
# UNet's round-1 path — the temporal GroupNorm's sums are all-reduced, the (3,1,1) convolutions get one-frame halo corrections,
# the closing 3-tap time mix (AE3DConv, temporal_ae.py:90-97) reads one halo frame of its 3-channel input on each side.
# Host-side orchestration only.  The engine picks it when there are more ranks than chunks, up to 4 ranks (validated on
# hardware at 2 and 4: 1.5e-3 against the serial decode at 4, one more fp16 rounding per halo correction; 0.115 s per clip).
# ---------------------------------------------------------------------------------------------------------------
from .vae import DecoderRuntime, _decode_chunks      # noqa: E402  (kept next to its only user)


class ShardedDecoderRuntime(DecoderRuntime):
    def __init__(self, cfg, sd, device, group=None):
        super().__init__(cfg, sd, device)
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self._to_global = (lambda r: r) if group is None else (lambda r: dist.get_global_rank(group, r))
        self._tap_w: Dict[int, tuple] = {}
        self.T_full, self.prev, self.next = 0, None, None

    def _set_chunk(self, n_frames: int):
        """Frame shards of an n_frames chunk; ranks beyond the frame count own nothing (and only take part in the
        collectives with zero contributions)."""
        self.T_full = n_frames
        self.shards = frame_shards(n_frames, min(self.world, n_frames))
        self.active = self.rank < len(self.shards)
        self.t0, self.t1 = self.shards[self.rank] if self.active else (0, 0)
        last = len(self.shards) - 1
        self.prev = self._to_global(self.rank - 1) if self.active and self.rank > 0 else None
        self.next = self._to_global(self.rank + 1) if self.active and self.rank < last else None

    # temporal GroupNorm: one statistic over ALL frames of the chunk
    def _fuse_stats(self, T, h, w) -> bool:
        return False        # halo corrections land after the main (3,1,1) launch: keep the separate statistics pass

    def _gn(self, x, y, T, hw, norm, eps, idx, fps=1, part=None, silu=True):
        if fps == 1:
            return super()._gn(x, y, T, hw, norm, eps, idx, fps, silu=silu)
        Cc, G = norm[0].numel(), self.cfg.num_groups
        sums = self.buf("gn.sums", G, 2, torch.float64)
        ops.groupnorm_sums(x, T, hw, Cc, sums, T, groups=G, ws=self.gn_ws)
        dist.all_reduce(sums, group=self.group)
        count = float(Cc // G) * hw * self.T_full
        return ops.groupnorm_finalize_apply(x, y, T, hw, norm[0], norm[1], eps, True, sums, count,
                                            self.gn_stats[idx, :1], T, groups=G)

    def _tap_weights(self, lin: Lin):
        key = lin.w.data_ptr()
        tw = self._tap_w.get(key)
        if tw is None:
            Cc = lin.w.shape[1] // 3
            tw = (Lin(lin.w[:, :Cc].contiguous(), None, lin.tile_n), Lin(lin.w[:, 2 * Cc:].contiguous(), None, lin.tile_n))
            self._tap_w[key] = tw
        return tw

    def _tconv(self, a, lin: Lin, out, T: int, hw: int, **epi):
        Cc = a.shape[1]
        send_first, send_last = self.buf("halo.sf", hw, Cc), self.buf("halo.sl", hw, Cc)
        recv_prev, recv_next = self.buf("halo.rp", hw, Cc), self.buf("halo.rn", hw, Cc)
        halo = HaloExchange(self.group, self.prev, self.next,
                            first=(send_first, a[:hw], send_first, recv_prev),
                            last=(send_last, a[(T - 1) * hw:T * hw], send_last, recv_next))
        halo.start()
        self.gemm(a, lin, out, taps=ops.TAPS_T3, geom=(hw, T, 1), **epi)
        halo.wait()
        s_acc = epi.get("s_acc", 1.0)
        w0, w2 = self._tap_weights(lin)
        if self.prev is not None:
            o = out[:hw]
            self.gemm(recv_prev, w0, o, s_acc=s_acc, res1=o)
        if self.next is not None:
            o = out[(T - 1) * hw:T * hw]
            self.gemm(recv_next, w2, o, s_acc=s_acc, res1=o)
        return out

    def _resblock(self, L, x, T, h, w, name):
        rb = L["spec"]
        hw, M, gi = h * w, T * h * w, L["gn_idx"]
        a1 = self._gn(x, self.buf("d.a1", M, rb.cin), T, hw, L["gn1"], 1e-6, gi)
        h1 = self.gemm(a1, L["conv1"], self.buf("d.h1", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, T))
        a2 = self._gn(h1, self.buf("d.a2", M, rb.cout), T, hw, L["gn2"], 1e-6, gi + 1)
        xs = x if L["skip"] is None else self.gemm(x, L["skip"], self.buf("d.xs", M, rb.cout))
        xsp = self.gemm(a2, L["conv2"], self.buf("d.xsp", M, rb.cout), taps=ops.TAPS_3X3, geom=(w, h, T), res1=xs)
        a3 = self._gn(xsp, self.buf("d.a1", M, rb.cout), T, hw, L["tgn1"], 1e-5, gi + 2, fps=T)
        h2 = self._tconv(a3, L["tconv1"], self.buf("d.h1", M, rb.cout), T, hw)
        a4 = self._gn(h2, self.buf("d.a2", M, rb.cout), T, hw, L["tgn2"], 1e-5, gi + 3, fps=T)
        out = self.buf(name, M, rb.cout)
        self._tconv(a4, L["tconv2"], out, T, hw, s_acc=L["alpha"], res1=xsp)       # xsp + alpha*(conv + bias)
        return out

    def forward_local(self, z_tokens: torch.Tensor, T: int, h: int, w: int) -> torch.Tensor:
        """z_tokens: rows of THIS rank's T frames of the chunk -> (T, 3, 8h, 8w) fp32 frames (time mix included)."""
        cfg = self.cfg
        if not hasattr(self, "gn_stats") or self.gn_stats.shape[1] < max(T, 1):
            self._bufs.setdefault(("gn.retired",), []).append(getattr(self, "gn_stats", None))   # tapes may still point at it
            self.gn_stats = torch.zeros(self.n_gn, max(T, 1), cfg.num_groups, 2, dtype=torch.float32, device=self.dev)
        if not hasattr(self, "gn_ws"):
            self.gn_ws = ops.GNWorkspace(self.dev)
        up_total = 2 ** (len(cfg.ch_mult) - 1)
        self.gn_ws.reserve(ops.groupnorm_scratch(T, h * w * up_total * up_total, cfg.num_groups))
        x = ops.conv3x3_small_cin(z_tokens, cfg.z_channels, self.conv_in_w, self.conv_in_b,
                                  self.buf("d.in", T * h * w, self.plan.block_in), T, h, w)
        x = self._resblock(self.res[self.plan.mid[0].prefix], x, T, h, w, "d.r0")
        x, _ = self._attn(x, T, h, w)
        x = self._resblock(self.res[self.plan.mid[1].prefix], x, T, h, w, "d.r1")
        for blocks, up, ch in self.plan.levels:
            for bi, rb in enumerate(blocks):
                x = self._resblock(self.res[rb.prefix], x, T, h, w, f"d.r{bi % 2}")
            if up is not None:
                xu = ops.upsample2x(x, self.buf("d.up", T * 4 * h * w, ch), T, h, w, ch)
                h, w = 2 * h, 2 * w
                x = self.gemm(xu, self.ups[up], self.buf("d.upc", T * h * w, ch), taps=ops.TAPS_3X3, geom=(w, h, T))
        hw, M = h * w, T * h * w
        a = ops.groupnorm(x, self.buf("d.a1", M, self.plan.final_ch), T, hw, self.norm_out[0], self.norm_out[1], 1e-6,
                          True, self.gn_stats[self.norm_out_idx, :T], groups=cfg.num_groups, ws=self.gn_ws)
        # 3-channel conv into the middle of a (T + 2)-frame buffer whose first / last frame are the neighbours' halos
        y_ext = self.buf("d.yext", (T + 2) * hw, 8, torch.float32)
        y_ext.zero_()
        y = y_ext[hw:(T + 1) * hw]
        self.gemm(a, self.out_conv, y, taps=ops.TAPS_3X3, geom=(w, h, T))
        send_first, send_last = self.buf("halo.yf", hw, 8, torch.float32), self.buf("halo.yl", hw, 8, torch.float32)
        halo = HaloExchange(self.group, self.prev, self.next,
                            first=(send_first, y[:hw], send_first, y_ext[:hw]),
                            last=(send_last, y[(T - 1) * hw:], send_last, y_ext[(T + 1) * hw:]))
        halo.start()
        halo.wait()
        ext = torch.empty(T + 2, cfg.out_ch, h, w, dtype=torch.float32, device=self.dev)
        ops.time_mix_small(y_ext, self.tmix_w, self.tmix_b, ext, None, T + 2, hw, cfg.out_ch, 0, 0)
        return ext[1:T + 1]


def decode_first_stage_sharded(rt: ShardedDecoderRuntime, z: torch.Tensor, scale_factor: float = 0.18215,
                               n_samples: Optional[int] = 14, overlap: int = 3) -> torch.Tensor:
    """decode_first_stage with the FRAMES of every chunk sharded over the ranks of rt.group; every rank passes the same
    z and receives the whole clip.  Chunk / overlap rule as in the serial path (vwm/models/diffusion.py:150-180)."""
    F_, zc, h, w = z.shape
    n_samples = F_ if n_samples is None else n_samples
    up = 2 ** (len(rt.cfg.ch_mult) - 1)
    H, W = h * up, w * up
    out = torch.empty(F_, rt.cfg.out_ch, H, W, dtype=torch.float32, device=z.device)
    zs = (z.float() / scale_factor).contiguous()
    chunks = _decode_chunks(F_, n_samples, overlap)
    if any(nov > n or o0 != f0 for f0, n, o0, nov in chunks):
        raise NotImplementedError("decode_first_stage_sharded: chunks shorter than the overlap")
    for f0, n, o0, nov in chunks:
        rt._set_chunk(n)
        pad = max(b - a for a, b in rt.shards)
        mine = torch.zeros(pad, rt.cfg.out_ch, H, W, dtype=torch.float32, device=z.device)
        if rt.active:
            T = rt.t1 - rt.t0
            tok = rt.buf("d.z", T * h * w, 8)
            tok.zero_()
            ops.nchw_to_tokens(zs[f0 + rt.t0:f0 + rt.t1].contiguous(), tok, T, zc, h, w)
            mine[:T] = rt.forward_local(tok, T, h, w)
        else:                                   # more ranks than frames: join the collectives with empty hands
            raise NotImplementedError("decode_first_stage_sharded: more ranks than frames in a chunk")
        gathered = torch.empty(rt.world * pad, rt.cfg.out_ch, H, W, dtype=torch.float32, device=z.device)
        dist.all_gather_into_tensor(gathered, mine, group=rt.group)
        parts = gathered.reshape(rt.world, pad, rt.cfg.out_ch, H, W)
        chunk = torch.cat([parts[r, : b - a] for r, (a, b) in enumerate(rt.shards)], dim=0)
        if nov:
            out[o0:o0 + nov] = 0.5 * (out[o0:o0 + nov] + chunk[:nov])
        out[o0 + nov:o0 + n] = chunk[nov:]
    return out
