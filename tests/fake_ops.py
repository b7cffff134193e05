"""CPU emulation of the C-ABI operators, for testing the HOST-side executors (buffer plumbing, weight packing,
tap / gather conventions) without a GPU.  Test infrastructure only: it patches vista_b200.ops inside a context
manager; nothing under vista_b200/ imports it.  Numerics: fp16 operands, fp32 accumulation and statistics, fp16 (or
fp32) outputs — the same rounding points as the kernels, so the executors can be compared with the golden fixtures
at the GPU tolerance."""
import contextlib

import torch
import torch.nn.functional as F


def _f(t):
    return t.float()


def gemm(a, w, out, *, taps=((0, 0),), geom=None, bias=None, rowvec=None, rv_div=1, rv_mod=1, res1=None, s_res1=1.0,
         res2=None, s_res2=1.0, s_acc=1.0, act=0, tile_n=None, cin=None, stats=None, h_pad=0):
    if h_pad:
        # `a` holds h_pad halo rows of H before and after the H output rows: fold them in as real neighbours, i.e. run the
        # plain tap-GEMM over the extended image and keep the middle rows
        W_, H_, NB_ = geom
        He = H_ + 2 * h_pad
        assert a.shape[0] == NB_ * He * W_
        assert act == 0
        tmp32 = torch.empty(NB_ * He * W_, out.shape[1], dtype=torch.float32)      # s_acc * (conv + bias), unrounded
        gemm(a, w, tmp32, taps=taps, geom=(W_, He, NB_), bias=bias, s_acc=s_acc, act=0, tile_n=tile_n, cin=cin)
        acc = tmp32.reshape(NB_, He, W_, -1)[:, h_pad:h_pad + H_].reshape(NB_ * H_ * W_, -1)
        tokens = acc.shape[0]
        if rowvec is not None:
            rows = (torch.arange(tokens) // rv_div) % rv_mod
            acc = acc + _f(rowvec)[rows][:, :acc.shape[1]]
        assert act == 0
        if res1 is not None:
            acc = acc + s_res1 * _f(res1)
        if res2 is not None:
            acc = acc + s_res2 * _f(res2)
        out.copy_(acc.to(out.dtype))
        if stats is not None:
            pad = (-tokens) % 128
            v = F.pad(acc, (0, 0, 0, pad)).reshape(-1, 32, acc.shape[1])
            stats[: v.shape[0], :acc.shape[1], 0] = v.sum(dim=1)
            stats[: v.shape[0], :acc.shape[1], 1] = (v * v).sum(dim=1)
        return out
    tokens = a.shape[0]
    N, K = w.shape
    ntaps = len(taps)
    cin = cin if cin is not None else K // ntaps
    x = _f(a[:, :cin])
    if geom is None:
        cols = x
    else:
        W, H, NB = geom
        assert W * H * NB == tokens
        img = x.reshape(NB, H, W, cin)
        parts = []
        for dh, dw in taps:                      # out[b,h,w] reads in[b, h+dh, w+dw], zero outside
            sh = torch.zeros_like(img)
            hs, he = max(0, -dh), min(H, H - dh)
            ws, we = max(0, -dw), min(W, W - dw)
            if hs < he and ws < we:
                sh[:, hs:he, ws:we] = img[:, hs + dh:he + dh, ws + dw:we + dw]
            parts.append(sh.reshape(tokens, cin))
        cols = torch.cat(parts, dim=1)
    acc = cols @ _f(w).t()
    if bias is not None:
        acc = acc + _f(bias)[:N]
    acc = acc * s_acc
    if rowvec is not None:
        rows = (torch.arange(tokens) // rv_div) % rv_mod
        acc = acc + _f(rowvec)[rows][:, :N]
    if act == 1:
        acc = F.silu(acc)
    elif act == 2:                               # value | gate halves per tile of tile_n columns (weights.permute_geglu)
        tn = tile_n if tile_n is not None else N
        hh = tn // 2
        t = acc.reshape(tokens, N // tn, 2, hh)
        acc = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(tokens, N // 2)
    elif act == 3:                               # erf-GELU
        acc = F.gelu(acc)
    if res1 is not None:
        acc = acc + s_res1 * _f(res1)
    if res2 is not None:
        acc = acc + s_res2 * _f(res2)
    n_out = out.shape[1]
    out.copy_(acc[:, :n_out].to(out.dtype))
    if stats is not None:              # column partials per (128-token tile, 32-row quarter) of the fp32 values, like the kernel
        pad = (-tokens) % 128
        v = F.pad(acc[:, :n_out], (0, 0, 0, pad)).reshape(-1, 32, n_out)
        stats[: v.shape[0], :n_out, 0] = v.sum(dim=1)
        stats[: v.shape[0], :n_out, 1] = (v * v).sum(dim=1)
    return out


class GNWorkspace:
    def __init__(self, device, max_stats=4096):
        self.device = device

    def reserve(self, n):
        pass


def groupnorm_scratch(frames, tokens_per_frame, groups=32):
    return 0


def groupnorm(x, y, frames, tokens_per_frame, gamma, beta, eps, silu, stats=None, frames_per_stat=1, groups=32, ws=None):
    C = gamma.numel()
    xs = _f(x[:, :C]).reshape(frames // frames_per_stat, frames_per_stat * tokens_per_frame, groups, C // groups)
    mean = xs.mean(dim=(1, 3), keepdim=True)
    var = xs.var(dim=(1, 3), unbiased=False, keepdim=True)
    if stats is not None:                        # the kernel's (mean, rstd) output
        stats[..., 0] = mean.reshape(stats.shape[:2])
        stats[..., 1] = torch.rsqrt(var + eps).reshape(stats.shape[:2])
    o = ((xs - mean) * torch.rsqrt(var + eps)).reshape(-1, C) * _f(gamma) + _f(beta)
    if silu:
        o = F.silu(o)
    y.copy_(o.to(y.dtype))
    return y


def groupnorm_from_partials(partials, frames, tokens_per_frame, Cc, eps, stats, frames_per_stat=1, groups=32, raw_sums=None):
    n_stat = frames // frames_per_stat
    rows = frames_per_stat * (tokens_per_frame // 128) * 4
    p = partials[: n_stat * rows, :Cc].double().reshape(n_stat, rows, groups, Cc // groups, 2).sum(dim=(1, 3))
    if raw_sums is not None:
        raw_sums.copy_(p.reshape(raw_sums.shape))
        return stats
    count = float(Cc // groups) * tokens_per_frame * frames_per_stat
    mean = p[..., 0] / count
    var = (p[..., 1] / count - mean * mean).clamp_min(0.0)
    stats[..., 0] = mean.float()
    stats[..., 1] = torch.rsqrt(var + eps).float()
    return stats


def groupnorm_apply(x, y, frames, tokens_per_frame, gamma, beta, silu, stats, frames_per_stat=1, groups=32):
    C = gamma.numel()
    n_stat = frames // frames_per_stat
    xs = _f(x[:, :C]).reshape(n_stat, frames_per_stat * tokens_per_frame, groups, C // groups)
    o = (xs - stats[..., 0][:, None, :, None]) * stats[..., 1][:, None, :, None]
    o = o.reshape(-1, C) * _f(gamma) + _f(beta)
    if silu:
        o = F.silu(o)
    y.copy_(o.to(y.dtype))
    return y


def conv3x3_small_cin(x8, cin, w, bias, out, NB, H, W):
    img = _f(x8[:, :cin]).reshape(NB, H, W, cin).permute(0, 3, 1, 2)
    o = F.conv2d(img, _f(w), None if bias is None else _f(bias), padding=1)
    out.copy_(o.permute(0, 2, 3, 1).reshape(NB * H * W, -1).to(out.dtype))
    return out


def im2col_s2_asym(x, out, NB, H, W, Cc):
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    img = F.pad(x[:, :Cc].reshape(NB, H, W, Cc), (0, 0, 0, 2, 0, 2))          # zero beyond the right / bottom edge
    parts = [img[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)]
    out.copy_(torch.cat(parts, dim=-1).reshape(NB * Ho * Wo, 9 * Cc))
    return out


def upsample2x(x, out, NB, H, W, Cc):
    img = x[:, :Cc].reshape(NB, H, W, Cc)
    out.copy_(img.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(NB * 4 * H * W, Cc))
    return out


def softmax_rows(x, y):
    y.copy_(torch.softmax(_f(x), dim=-1).to(y.dtype))
    return y


def nchw_to_tokens(x, out, NB, Cc, H, W):
    out[:, :Cc] = x.permute(0, 2, 3, 1).reshape(NB * H * W, Cc).to(out.dtype)
    return out


def tokens_to_nchw(x, out, NB, Cc, H, W):
    out.copy_(_f(x[:, :Cc]).reshape(NB, H, W, Cc).permute(0, 3, 1, 2))
    return out


def time_mix_small(x, w, bias, out, blend, T, HW, Cc, out_frame0=0, skip_frames=0):
    v = _f(x[:, :Cc]).reshape(T, HW, Cc)
    acc = torch.zeros(T, HW, Cc) + (0 if bias is None else _f(bias))
    for kt in range(3):
        for t in range(T):
            tt = t + kt - 1
            if 0 <= tt < T:
                acc[t] += v[tt] @ _f(w)[:, :, kt].t()
    hh = out.shape[2]
    img = acc.reshape(T, hh, HW // hh, Cc).permute(0, 3, 1, 2)
    for t in range(skip_frames, T):
        if blend is not None and int(blend[t]) != 0:
            out[out_frame0 + t] = 0.5 * (out[out_frame0 + t] + img[t])
        else:
            out[out_frame0 + t] = img[t]
    return out


def time_mix_small_u8(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0=0, skip_frames=0, keep_f32_from=-1):
    tmp = out.clone()
    time_mix_small(x, w, bias, tmp, blend, T, HW, Cc, out_frame0, skip_frames)
    for t in range(skip_frames, T):
        f = out_frame0 + t
        s = ((tmp[f] + 1.0) / 2.0).clamp(0.0, 1.0)
        out_u8[f] = (255.0 * s).to(torch.uint8).permute(1, 2, 0)          # float -> uint8 truncates, like numpy astype
        if keep_f32_from < 0 or t >= keep_f32_from:
            out[f] = tmp[f]
    return out_u8


def rollout_advance(sample, z0, samples_z, filled, dst_frame0, src_frame0, n_cond):
    T = sample.shape[0]
    if z0 is not None:
        sample[0] = z0[0]
    samples_z[dst_frame0 + src_frame0:dst_frame0 + T] = sample[src_frame0:]
    if filled is not None:
        filled.zero_()
        filled[:n_cond] = sample[T - n_cond:]
    return samples_z


def ensemble_reward(members):
    K = len(members)
    u = torch.mean(torch.stack(members), 0)
    diff = torch.zeros_like(members[0])
    for m in members:
        diff.add_((m - u) ** 2)
    mv = (diff / (K - 1)).double().mean().float()
    return torch.stack([mv, torch.exp(-mv)])


def groupnorm_sums(x, frames, tokens_per_frame, Cc, sums, frames_per_stat, groups=32, ws=None):
    xs = x[:, :Cc].double().reshape(frames // frames_per_stat, frames_per_stat * tokens_per_frame, groups, Cc // groups)
    sums.copy_(torch.stack([xs.sum(dim=(1, 3)), (xs * xs).sum(dim=(1, 3))], dim=-1).reshape(sums.shape))
    return sums


def groupnorm_finalize_apply(x, y, frames, tokens_per_frame, gamma, beta, eps, silu, sums, count, stats, frames_per_stat,
                             groups=32):
    C = gamma.numel()
    n_stat = frames // frames_per_stat
    sm = sums.reshape(n_stat, groups, 2)
    mean = sm[..., 0] / count
    var = (sm[..., 1] / count - mean * mean).clamp_min(0.0)
    xs = _f(x[:, :C]).reshape(n_stat, frames_per_stat * tokens_per_frame, groups, C // groups)
    o = (xs - mean.float()[:, None, :, None]) * torch.rsqrt(var.float() + eps)[:, None, :, None]
    o = o.reshape(-1, C) * _f(gamma) + _f(beta)
    if silu:
        o = F.silu(o)
    y.copy_(o.to(y.dtype))
    return y


def layernorm(x, y, gamma, beta, eps=1e-5, addvec=None, av_div=1, av_mod=1):
    C = gamma.numel()
    v = _f(x[:, :C])
    if addvec is not None:
        rows = (torch.arange(v.shape[0]) // av_div) % av_mod
        v = v + _f(addvec)[rows][:, :C]
    y.copy_(F.layer_norm(v, (C,), _f(gamma), _f(beta), eps).to(y.dtype))
    return y


def attention_spatial(q, k, v, out, frames, seq, heads, impl=None):
    def sp(t):
        return _f(t).reshape(frames, seq, heads, 64).permute(0, 2, 1, 3)
    o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v))
    out.copy_(o.permute(0, 2, 1, 3).reshape(frames * seq, heads * 64).to(out.dtype))
    return out


def attention_temporal(q, k, v, out, nb, T, S, heads):
    def tp(t):                                   # tokens (b, t, s) -> (b, s, head, t, 64)
        return _f(t).reshape(nb, T, S, heads, 64).permute(0, 2, 3, 1, 4)
    o = F.scaled_dot_product_attention(tp(q), tp(k), tp(v))
    out.copy_(o.permute(0, 3, 1, 2, 4).reshape(nb * T * S, heads * 64).to(out.dtype))
    return out


def attention_temporal_sharded(q, k, v, out, nb, Tq, T, S, heads, kv_frame_tok):
    C = heads * 64
    rows = (kv_frame_tok.reshape(nb, T, 1) + torch.arange(S).reshape(1, 1, S)).reshape(-1)      # (b, t, s) -> gathered row
    kk = _f(k)[rows].reshape(nb, T, S, heads, 64).permute(0, 2, 3, 1, 4)
    vv = _f(v)[rows].reshape(nb, T, S, heads, 64).permute(0, 2, 3, 1, 4)
    qq = _f(q).reshape(nb, Tq, S, heads, 64).permute(0, 2, 3, 1, 4)
    o = F.scaled_dot_product_attention(qq, kk, vv)
    out.copy_(o.permute(0, 3, 1, 2, 4).reshape(nb * Tq * S, C).to(out.dtype))
    return out


def timestep_embedding(t, out, dim, max_period=10000.0):
    half = dim // 2
    freq = torch.exp(-torch.log(torch.tensor(float(max_period))) * torch.arange(half, dtype=torch.float32) / half)
    a = _f(t).reshape(-1, 1) * freq
    out[:, :dim] = torch.cat([torch.cos(a), torch.sin(a)], dim=1).to(out.dtype)
    return out


def blend_emb(e_plain, e_cond, label, mask, emb, silu_emb):
    m = torch.zeros(e_plain.shape[0], 1) if mask is None else _f(mask).reshape(-1, 1)
    e = _f(e_plain) * (1.0 - m)
    if e_cond is not None:
        e = e + _f(e_cond) * m
    if label is not None:
        e = e + _f(label)
    if emb is not None:
        emb.copy_(e)
    if silu_emb is not None:
        silu_emb.copy_(F.silu(e).to(silu_emb.dtype))


def im2col_s2(x, out, NB, H, W, Cc):
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    img = F.pad(x[:, :Cc].reshape(NB, H, W, Cc), (0, 0, 1, 2, 1, 2))
    parts = [img[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)]
    out.copy_(torch.cat(parts, dim=-1).reshape(NB * Ho * Wo, 9 * Cc))
    return out


def sampler_prepare(x, cond_frame, mask, concat_u, concat_c, sigmas, step_idx, unet_in, c_noise, T, h, w):
    sigma = float(sigmas[int(step_idx[0])])
    c_in = (sigma * sigma + 1.0) ** -0.5
    if mask is not None and cond_frame is not None:
        m = _f(mask).reshape(T, 1, 1, 1)
        x.copy_(x * (1.0 - m) + cond_frame * m)
    if c_noise is not None:
        c_noise.fill_(0.25 * float(torch.log(torch.tensor(sigma))))
    xs = (x * c_in).permute(0, 2, 3, 1).reshape(T * h * w, 4)
    zu = torch.zeros_like(xs) if concat_u is None else concat_u.permute(0, 2, 3, 1).reshape(T * h * w, 4)
    zc = torch.zeros_like(xs) if concat_c is None else concat_c.permute(0, 2, 3, 1).reshape(T * h * w, 4)
    unet_in[: T * h * w, :8] = torch.cat([xs, zu], 1).to(unet_in.dtype)
    unet_in[T * h * w:, :8] = torch.cat([xs, zc], 1).to(unet_in.dtype)


def sampler_update(x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w):
    step = int(step_idx[0])
    sigma, sigma_next = float(sigmas[step]), float(sigmas[step + 1])
    c_skip, c_out = 1.0 / (sigma * sigma + 1.0), -sigma * (sigma * sigma + 1.0) ** -0.5
    hw = h * w
    nu = _f(net_out[: T * hw, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    nc = _f(net_out[T * hw:, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    du, dc = nu * c_out + x * c_skip, nc * c_out + x * c_skip
    den = du + _f(scales).reshape(T, 1, 1, 1) * (dc - du)
    xn = x + (x - den) / sigma * (sigma_next - sigma)
    if step + 1 == num_steps and mask is not None and cond_frame is not None:
        m = _f(mask).reshape(T, 1, 1, 1)
        xn = xn * (1.0 - m) + cond_frame * m
    x.copy_(xn)
    step_idx += 1


from fake_peer import peer_allreduce_f64, peer_put, peer_wait      # noqa: E402  (emulated NVLink peer kernels)

_PATCHED = ["gemm", "GNWorkspace", "groupnorm_scratch", "groupnorm", "conv3x3_small_cin", "im2col_s2_asym", "upsample2x",
            "softmax_rows", "nchw_to_tokens", "tokens_to_nchw", "time_mix_small", "groupnorm_sums",
            "groupnorm_finalize_apply", "groupnorm_from_partials", "groupnorm_apply", "layernorm", "attention_spatial", "attention_temporal",
            "attention_temporal_sharded", "timestep_embedding", "blend_emb", "im2col_s2", "sampler_prepare",
            "sampler_update", "time_mix_small_u8", "rollout_advance", "ensemble_reward", "peer_put", "peer_wait", "peer_allreduce_f64"]
_NOT_TAPED = {"GNWorkspace", "groupnorm_scratch", "rollout_advance", "ensemble_reward", "peer_put", "peer_wait", "peer_allreduce_f64"}


@contextlib.contextmanager
def patched_ops():
    """Swap the emulations into vista_b200.ops for the duration of the block.  Every emulated launch goes through
    lib.tape_host, so that a launch tape recorded by the executors replays them like real C-ABI calls."""
    from vista_b200 import lib, ops

    def taped(fn):
        def call(*a, **k):
            return lib.tape_host(lambda: fn(*a, **k))
        return call
    saved = {k: getattr(ops, k) for k in _PATCHED}
    try:
        for k in _PATCHED:
            setattr(ops, k, globals()[k] if k in _NOT_TAPED else taped(globals()[k]))
        yield
    finally:
        for k, v in saved.items():
            setattr(ops, k, v)
