"""Gain conformance on the H100: the launch harness of tests/shadow.py (gain check on) over production launch
configurations of 576 x 1024 (latent 72 x 128, 50 frames) on the real kernels, clean and with the five systematic
defects of test_bias_conformance_cpu.py planted in wrappers around vista_b200.ops (never in a kernel).  Clean, every key
passes; each defect passes the element / rel-L2 rule and fails the gain check at twice its bound or more, naming the op,
the key and the term.  Each case prints the harness's census."""
import pytest
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

import shadow
from test_bias_conformance_cpu import GN_RSTD_GAIN, S_ACC, S_RES1, U16, fp16_scale, rz16_after_extra_bit
from test_conformance_cpu import U24
from test_conformance_small_cpu import u8_path

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
B, H0, W0 = 50, 72, 128               # the UNet's CFG batch and level-0 latent of 576 x 1024


def rnd(*shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


# ==================================================================================================================
# Production launches
# ==================================================================================================================
def gemm_conv(ops):
    """The level-0 ResBlock convolution: 3x3 taps over 50 frames of 72 x 128, 320 -> 320 channels, bias, a residual,
    with blend scales s_acc = 1/3 and s_res1 = 2/3."""
    C = 320
    a, w = rnd(B * H0 * W0, C, seed=1), rnd(C, 9 * C, seed=2, scale=(9 * C) ** -0.5)
    res = rnd(B * H0 * W0, C, seed=3, scale=0.5)
    out = torch.empty(B * H0 * W0, C, dtype=torch.float16, device=DEV)
    ops.gemm(a, w, out, taps=ops.TAPS_3X3, geom=(W0, H0, B), bias=rnd(C, seed=4, dtype=torch.float32), res1=res,
             s_res1=S_RES1, s_acc=S_ACC)


def attention_l1(ops):
    """Level-1 spatial self-attention: 50 frames of 36 x 64 tokens, 10 heads."""
    seq, heads = (H0 // 2) * (W0 // 2), 10
    C = 64 * heads
    qkv = rnd(B * seq, 3 * C, seed=5, scale=1.5)
    out = torch.empty(B * seq, C, dtype=torch.float16, device=DEV)
    ops.attention_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, B, seq, heads)


def groupnorm_apply_clip(ops):
    """The decoder's temporal GroupNorm: a 14-frame clip at 72 x 128, 512 channels, statistics over the clip from the
    fused partials of the GEMM that wrote it, then the apply (without SiLU: the normalised term alone)."""
    T, C = 14, 512
    tpf = H0 * W0
    a, w = rnd(T * tpf, C, seed=6), rnd(C, C, seed=7, scale=C ** -0.5)
    x = torch.empty(T * tpf, C, dtype=torch.float16, device=DEV)
    partials = torch.zeros(T * tpf // 128 * 4, C, 2, device=DEV)
    ops.gemm(a, w, x, bias=rnd(C, seed=8, dtype=torch.float32, scale=0.3), stats=partials)
    stats = torch.zeros(1, 32, 2, device=DEV)
    ops.groupnorm_from_partials(partials, T, tpf, C, 1e-5, stats, frames_per_stat=T)
    gamma = rnd(C, seed=9, dtype=torch.float32, scale=0.2) + 1
    ops.groupnorm_apply(x, torch.empty_like(x), T, tpf, gamma, rnd(C, seed=10, dtype=torch.float32, scale=0.3), False,
                        stats, frames_per_stat=T)


def time_mix_decode(ops):
    """The decoder's output time mix on the second 14-frame chunk of a 25-frame decode at 576 x 1024: frames 11..24,
    the first three blended with the previous chunk's, every fp32 frame kept."""
    T, HW = 14, 576 * 1024
    x = rnd(T * HW, 8, seed=11, dtype=torch.float32, scale=0.8)
    w, b = rnd(3, 3, 3, seed=12, dtype=torch.float32, scale=0.5), rnd(3, seed=13, dtype=torch.float32, scale=0.1)
    out = rnd(25, 3, 576, 1024, seed=14, dtype=torch.float32, scale=0.7)
    out8 = torch.zeros(25, 576, 1024, 3, dtype=torch.uint8, device=DEV)
    blend = torch.tensor([1] * 3 + [0] * (T - 3), dtype=torch.int32, device=DEV)
    ops.time_mix_small_u8(x, w, b, out, out8, blend, T, HW, 3, out_frame0=11, skip_frames=0, keep_f32_from=-1)


LAUNCHES = {"gemm": gemm_conv, "attention_spatial": attention_l1, "groupnorm_apply": groupnorm_apply_clip,
            "time_mix_small_u8": time_mix_decode}


# ==================================================================================================================
# Defects: wrappers around the real entry points
# ==================================================================================================================
def scales_fp16(real):
    def gemm(a, w, out, **kw):
        return real(a, w, out, **dict(kw, s_acc=fp16_scale(kw.get("s_acc", 1.0)),
                                      s_res1=fp16_scale(kw.get("s_res1", 1.0))))
    return gemm


def store_toward_zero(real):
    def gemm(a, w, out, **kw):
        tmp = torch.empty(out.shape, dtype=torch.float32, device=out.device)     # the epilogue's value before the store
        real(a, w, tmp, **kw)
        out.copy_(rz16_after_extra_bit(tmp))
        return out
    return gemm


def attention_scaled(real):
    """A twin, not the kernel plus a defect: the kernel stores fp16 and its value before rounding is not reachable, and
    scaling that fp16 output would add a second rounding (a shift of one ulp, not a gain).  So the defective launch is
    fp32 SDPA with the scaled store; the clean case holds the real kernel on the same key."""
    def attention_spatial(q, k, v, out, frames, seq, heads, impl=None):
        sp = lambda t: t.float().reshape(frames, seq, heads, 64).permute(0, 2, 1, 3)
        with sdpa_kernel(SDPBackend.MATH):
            for f in range(frames):            # fp32 attention one frame at a time, then the scaled store
                o = F.scaled_dot_product_attention(sp(q)[f:f + 1], sp(k)[f:f + 1], sp(v)[f:f + 1])
                out[f * seq:(f + 1) * seq] = (o.permute(0, 2, 1, 3).reshape(seq, heads * 64) * (1 - U16)).half()
        return out
    return attention_spatial


def rstd_high(real):
    def groupnorm_apply(x, y, frames, tokens_per_frame, gamma, beta, silu, stats, frames_per_stat=1, groups=32):
        s = stats.clone()
        s[..., 1] *= 1 + GN_RSTD_GAIN
        return real(x, y, frames, tokens_per_frame, gamma, beta, silu, s, frames_per_stat, groups)
    return groupnorm_apply


def blend_high(real):
    def time_mix_small_u8(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0=0, skip_frames=0, keep_f32_from=-1):
        real(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0, skip_frames, keep_f32_from)
        for t in range(skip_frames, T):
            if blend is not None and int(blend[t]):
                f = out_frame0 + t
                out[f] *= 1 + 2 * U24                 # the blend weight 0.5 one fp32 ulp high
                out_u8[f] = u8_path(out[f]).permute(1, 2, 0)
        return out_u8
    return time_mix_small_u8


# defect -> (op, wrapper, the term the failure must name)
DEFECTS = {"scales_fp16": ("gemm", scales_fp16, "acc"), "store_toward_zero": ("gemm", store_toward_zero, "acc"),
           "attention_scaled": ("attention_spatial", attention_scaled, "ref"),
           "rstd_high": ("groupnorm_apply", rstd_high, "norm"), "blend_high": ("time_mix_small_u8", blend_high, "prev")}


def test_production_keys_clean():
    """Every production launch above, on the real kernels: every key passes, gain check included."""
    from vista_b200 import lib, ops
    lib.load()
    with torch.no_grad(), shadow.Shadow() as sh:
        for fn in LAUNCHES.values():
            fn(ops)
        torch.cuda.synchronize()
    print(f"\n[clean] {torch.cuda.get_device_name(DEV)}\n" + sh.report())
    sh.assert_ok()
    fams = sh.families()
    assert {"gemm", "attention_spatial", "groupnorm_apply", "groupnorm_from_partials", "time_mix_small_u8"} <= set(fams)


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_defect_fails_the_gain_check(defect, monkeypatch):
    """The defect's op fails on one key, on the gain check alone, at 2x its bound or more, naming the term; every
    other launch passes."""
    from vista_b200 import lib, ops
    lib.load()
    op, wrap, term = DEFECTS[defect]
    monkeypatch.setattr(ops, op, wrap(getattr(ops, op)))
    with torch.no_grad(), shadow.Shadow() as sh:
        LAUNCHES[op](ops)
        torch.cuda.synchronize()
    print(f"\n[{defect}] {torch.cuda.get_device_name(DEV)}\n" + sh.report())
    for msg in sh.failures.values():
        print("   ", msg)
    assert len(sh.failures) == 1, sh.failures
    (key, msg), = sh.failures.items()
    assert key[0] == op and "systematic gain on" in msg and f"{term}: beta" in msg, msg
    worst = sh.worst_gain(op)
    assert worst.ratio >= 2.0, f"{defect}: fails at only {worst.ratio:.2f} x the bound: {worst}"


# ==================================================================================================================
# Planted layer defects at 576 x 1024: one Euler step of the full-size UNet under the layer harness
# ==================================================================================================================
@pytest.mark.parametrize("defect,direction", [("residual", "res"), ("alpha", "d_alpha")])
def test_planted_layer_defect_production(defect, direction, monkeypatch):
    """trajectory.DEFECTS on the full-size engine (B = 50 CFG forward, T = 25, 576 x 1024): each layer's partition rule
    passes, and the gain check fails at 2x its bound or more, naming a layer and the direction."""
    import time
    import trajectory as tj
    from block_shadow import BlockShadow
    from test_block_conformance_gpu import ACTION, UC_KEYS, T, H, W, weights
    from test_production_conformance_gpu import sampler
    from tools.bench_session import build_engine
    from vista_b200 import fused, lib, ops, synth
    from oracle.make_golden_clip import clip_frames
    monkeypatch.setattr(fused, "USE_GRAPH", False)
    lib.load()
    eng = build_engine(DEV)
    frame = torch.from_numpy(clip_frames(12, "block_conformance", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "block_conformance.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "block_conformance.noise", (T, 4, H // 8, W // 8))).to(DEV)
    with torch.no_grad():
        c, uc = eng.condition({**vd, **ACTION}, T, UC_KEYS)
    monkeypatch.setattr(eng, "sampler", sampler(eng, "euler_vanilla", 1))
    unet, _, _ = weights(eng)
    t0 = time.perf_counter()
    with torch.no_grad(), tj.planted(defect, ops, eng.model), BlockShadow(unet=unet) as bs:
        eng.sample(c, uc=uc, N=T, shape=tuple(z.shape[1:]), noise=noise.clone(), cond_frame=z)
        torch.cuda.synchronize()
    print(f"\n[layer {defect}] {torch.cuda.get_device_name(DEV)}: wall {time.perf_counter() - t0:.1f} s\n" + bs.report())
    for msg in bs.failures.values():
        print("   ", msg)
    assert bs.failures and all(k[0] == "gain" for k in bs.failures), list(bs.failures)
    hits = [bs.census[k[1]].gain for k in bs.failures if bs.census[k[1]].gain_term.name.startswith(direction)]
    assert hits and max(hits) >= 2.0, f"{defect}: {list(bs.failures.values())}"
