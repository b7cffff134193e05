"""Conformance of the small kernels of the single-GPU path against fp64 references: the fused sampler step, the thin
direct convolution, the decoder's output kernels (fp32 and uint8), the rollout glue, the embedding helpers, the layout
converters and the CLIP attention.  This file holds the case tables, the references and the bounds, and runs every table
on the operator twins of tests/fake_ops.py (tests/clip_fake_ops.py for attention_d80); it also holds KERNEL_TESTS, the
map from every __global__ kernel of vista_b200/csrc/ to the conformance tests that hold it.

tests/test_conformance_small_gpu.py runs the same tables on the kernels, with the twin beside each on the same inputs.

The tolerance rule is the one of tests/test_conformance_cpu.py: per element |out - ref| <= ulp_out(|ref|) + eps * mag,
mag an fp64 magnitude of the operation's terms, eps derived from the roundings the operation performs (written next to
each reference); data movement and byte bookkeeping match exactly."""
import ast
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

import clip_fake_ops
import fake_ops
from test_conformance_cpu import (ATTN_EPS, CPU, FAMILY, U24, assert_conform, attention_reference, gemm_reference,
                                  padded, rel_l2, rnd, ulp)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAPS_3X3 = [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]
NAN = float("nan")


def gen(seed: int, device=CPU) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def randn(shape, seed, device, scale=1.0):
    """fp32 normal values drawn on `device` (the production-size inputs are drawn where they are used)."""
    return torch.randn(*shape, generator=gen(seed, device), device=device) * scale


def assert_elements(out, ref, tol, name):
    """Element bound only: for short vectors (c_noise, a scalar), where an L2 floor of the fp16 rounding means nothing."""
    err = (out.double() - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err - tol, torch.zeros_like(err))))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; worst flat index {i}: "
                             f"out {float(out.flatten()[i]):.9g} ref {float(ref.flatten()[i]):.9g} "
                             f"tol {float(tol.flatten()[i]):.3g}")


def sync(device):
    if device.type == "cuda":
        torch.cuda.synchronize()


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bit-for-bit equality (NaN sentinels included, which torch.equal treats as unequal)."""
    return a.shape == b.shape and a.dtype == b.dtype and \
        torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ==================================================================================================================
# A. Sampler step (b200v_sampler_prepare, b200v_sampler_update)
# ==================================================================================================================
IN_PAD = 64      # row stride of vista_b200.unet.padded_input_rows
NUM_STEPS = 50


def edm_sigmas(n=NUM_STEPS):
    from oracle.vista_oracle import edm_sigmas as _e
    return _e(n)


def triangle_scales(T):
    from oracle.vista_oracle import triangle_scales as _t
    return _t(T)


# (T, h, w, mask kind, concat_u given, concat_c given, scale kind); mask kind: 'none' (mask and cond_frame NULL), 'init'
# (the initial mask [1, 0, ...]) or 'rollout' (frames 0..2 of a later round)
SAMPLER_CASES = [(25, 72, 128, "init", True, True, "triangle"),
                 (25, 8, 16, "rollout", False, True, "const"),
                 (25, 8, 16, "none", True, False, "triangle"),
                 (3, 5, 7, "rollout", True, True, "triangle"),     # 105 tokens: not a multiple of 256; every frame masked
                 (3, 5, 7, "init", False, False, "const"),
                 (1, 1, 1, "init", True, True, "const"),           # one token: c_noise is written by threads >= total
                 (1, 1, 1, "none", False, False, "triangle")]
SAMPLER_STEPS = (0, 24, NUM_STEPS - 1)                             # the last one goes to sigma = 0 and re-imposes


def sampler_case_id(c):
    return "T{}x{}x{}-{}-u{}c{}-{}".format(c[0], c[1], c[2], c[3], int(c[4]), int(c[5]), c[6])


def make_sampler_inputs(case, device, seed=1):
    """fp32 state and arguments of one case, in the layouts the fused sampler uses: unet_in a [2 T h w, 8] view of rows of
    IN_PAD halves whose pad columns hold NaN sentinels, net_out [2 T h w, 8] fp32 whose columns 4..7 are NaN."""
    T, h, w, mk, cu, cc, sk = case
    hw = h * w
    d = dict(T=T, h=h, w=w)
    d["x"] = randn((T, 4, h, w), seed, device, 3.0)
    d["cond_frame"] = d["mask"] = None
    if mk != "none":
        m = torch.zeros(T, device=device)
        m[:1 if mk == "init" else 3] = 1.0
        d["mask"], d["cond_frame"] = m, randn((T, 4, h, w), seed + 1, device)
    d["concat_u"] = randn((T, 4, h, w), seed + 2, device) if cu else None
    d["concat_c"] = randn((T, 4, h, w), seed + 3, device) if cc else None
    d["scales"] = (triangle_scales(T) if sk == "triangle" else torch.full((T,), 2.5)).to(device)
    d["sigmas"] = edm_sigmas().to(device)
    d["in_buf"] = torch.full((2 * T * hw, IN_PAD), NAN, dtype=torch.float16, device=device)
    d["unet_in"] = d["in_buf"][:, :8]
    d["c_noise_buf"] = torch.full((2 * T + 4,), NAN, device=device)
    d["c_noise"] = d["c_noise_buf"][:2 * T]
    net = randn((2 * T * hw, 8), seed + 4, device)
    net[:, 4:] = NAN
    d["net"] = net
    return d


def prepare_reference(d, sigma):
    """fp64 of what sampler_prepare writes: the masked x (x (1 - m) + cond m, exact in fp32 for 0/1 masks: the kernel must
    match the fp32 formula bit for bit), unet_in columns 0..3 = x c_in with c_in = (s^2 + 1)^-1/2 and their magnitude,
    columns 4..7 the fp16 rounding of concat_u (first T h w rows) / concat_c (last T h w rows), or zeros."""
    T, h, w = d["T"], d["h"], d["w"]
    x = d["x"]
    if d["mask"] is not None:
        m = d["mask"].reshape(T, 1, 1, 1)
        x = x * (1.0 - m) + d["cond_frame"] * m
    s = float(sigma)
    c_in = (s * s + 1.0) ** -0.5
    tok = lambda t: t.permute(0, 2, 3, 1).reshape(T * h * w, 4)
    xs = tok(x.double()) * c_in
    cat = [torch.zeros(T * h * w, 4, dtype=torch.float16, device=x.device) if c is None else tok(c).half()
           for c in (d["concat_u"], d["concat_c"])]
    return x, torch.cat([xs, xs]), torch.cat(cat)


# rsqrtf (2 ulp: 4 U24 relative), s^2 and s^2 + 1 rounded (2 U24, halved by the square root: U24), the product (U24)
PREP_EPS = 6 * U24


def c_noise_reference(sigma, n, device):
    """0.25 ln s and its bound: logf is within 1 ulp (2 U24 relative), the factor 0.25 is exact."""
    ref = torch.full((n,), 0.25 * math.log(float(sigma)), dtype=torch.float64, device=device)
    return ref, ulp(ref, torch.float32) + 2 * U24 * ref.abs()


def update_reference(x, d, step, num_steps=NUM_STEPS):
    """fp64 Euler step of the V-scaled EDM denoiser under the per-frame guider, from fp32 inputs:
    D = x c_skip + c_out (u + scale_t (c - u)), x' = x + (x - D) / s (s' - s), c_skip = 1 / (s^2 + 1),
    c_out = -s (s^2 + 1)^-1/2; the conditioning frames re-imposed on the final step.  Returns (x', mag, a) with
    a = dx'/dx = 1 + (1 - c_skip)(s' - s) / s, in (0, 1].

    Bound (UPDATE_EPS * mag), counting roundings of the kernel's fp32 evaluation against
    M = |x| + (1 + 2|scale_t|)(c_skip |x| + |c_out| (|u| + |c|)), which bounds |x|, |D| (D = (1 - scale) du + scale dc) and
    |x - D| / 2, with (s' - s) / s in [-1, 0):  c_skip 3 U24 (s^2, + 1, division), c_out 6 U24 (as c_in, times s), du and
    dc 2 U24 each, dc - du, the scale product and the sum 1 U24 each: 14 U24 M on D; x - D, / s, s' - s, the product
    2 U24 M each, the final sum 3 U24 M: 25 U24 M in all."""
    T, h, w = d["T"], d["h"], d["w"]
    hw = h * w
    s, s1 = float(d["sigmas"][step]), float(d["sigmas"][step + 1])
    c_skip, c_out = 1.0 / (s * s + 1.0), -s * (s * s + 1.0) ** -0.5
    nch = lambda t: t[:, :4].double().reshape(T, h, w, 4).permute(0, 3, 1, 2)
    u, c = nch(d["net"][:T * hw]), nch(d["net"][T * hw:2 * T * hw])
    sc = d["scales"].double().reshape(T, 1, 1, 1)
    x64 = x.double()
    den = x64 * c_skip + c_out * (u + sc * (c - u))
    xn = x64 + (x64 - den) / s * (s1 - s)
    mag = x64.abs() + (1 + 2 * sc.abs()) * (c_skip * x64.abs() + abs(c_out) * (u.abs() + c.abs()))
    if step + 1 == num_steps and d["mask"] is not None:
        m = d["mask"].double().reshape(T, 1, 1, 1)
        xn = xn * (1 - m) + d["cond_frame"].double() * m
        mag = mag * (1 - m)
    return xn, mag, 1.0 + (1.0 - c_skip) * (s1 - s) / s


UPDATE_EPS = 32 * U24      # the 25 U24 derived in update_reference, rounded up


def check_sampler_step(case, step, prepare, update, device):
    """One prepare -> update at `step` of the 50-step schedule through `prepare` / `update` (ops or their twins)."""
    d = make_sampler_inputs(case, device, seed=10 + step)
    T, h, w = d["T"], d["h"], d["w"]
    name = f"{sampler_case_id(case)} step {step}"
    idx = torch.tensor([step], dtype=torch.int32, device=device)
    sigma = d["sigmas"][step]
    x_ref, in_ref, cat_ref = prepare_reference(d, sigma)
    x = d["x"].clone()
    prepare(x, d["cond_frame"], d["mask"], d["concat_u"], d["concat_c"], d["sigmas"], idx, d["unet_in"], d["c_noise"],
            T, h, w)
    sync(device)
    # the 0/1 mask is exact: the masked x is the fp32 formula, bit for bit
    assert torch.equal(x, x_ref), f"{name}: masked x differs from x (1 - m) + cond m"
    assert_conform(d["unet_in"][:, :4], in_ref, in_ref.abs(), PREP_EPS, "elementwise", f"{name}: unet_in x c_in")
    assert torch.equal(d["unet_in"][:, 4:], cat_ref), f"{name}: concat columns are not the fp16 rounding of concat_u / c"
    assert bool(torch.isnan(d["in_buf"][:, 8:]).all()), f"{name}: pad columns of the padded input rows written"
    cn_ref, cn_tol = c_noise_reference(sigma, 2 * T, device)
    assert_elements(d["c_noise"], cn_ref, cn_tol, f"{name}: c_noise")
    if device.type == "cuda":         # the twin fills its view; the kernel must stop at 2 T
        assert bool(torch.isnan(d["c_noise_buf"][2 * T:]).all()), f"{name}: c_noise written past 2 T"
    xn_ref, mag, _ = update_reference(x, d, step)
    update(x, d["net"], d["cond_frame"], d["mask"], d["scales"], d["sigmas"], idx, NUM_STEPS, T, h, w)
    sync(device)
    assert int(idx[0]) == step + 1, f"{name}: step_idx {int(idx[0])}"
    assert_conform(x, xn_ref, mag, UPDATE_EPS, "elementwise", f"{name}: update")
    if step + 1 == NUM_STEPS and d["mask"] is not None:
        m = d["mask"].bool()
        assert torch.equal(x[m], d["cond_frame"][m]), f"{name}: conditioning frames not re-imposed exactly"


def trajectory_inputs(T, h, w, device):
    """The rollout configuration: frames 0..2 conditioned, both concat inputs, the triangle guider scales."""
    return make_sampler_inputs((T, h, w, "rollout", True, True, "triangle"), device, seed=77)


def trajectory_reference(d, num_steps=NUM_STEPS):
    """50 fp64 prepare -> update steps from the fp32 start state with the fixed network output, and the per-element bound
    accumulated through the affine update: e' = a e + UPDATE_EPS * mag(|x| + e), a = dx'/dx in (0, 1] (errors of earlier
    steps do not grow), reset to zero where prepare / the final step re-impose the conditioning frames."""
    T = d["T"]
    x = d["x"].double()
    e = torch.zeros_like(x)
    m = d["mask"].double().reshape(T, 1, 1, 1)
    cf = d["cond_frame"].double()
    for k in range(num_steps):
        x = x * (1 - m) + cf * m
        e = e * (1 - m)
        dd = dict(d)
        xn, mag, a = update_reference(x, dd, k, num_steps)
        mag_e = update_reference(x.abs() + e, dd, k, num_steps)[1]        # the magnitude at the perturbed state
        e = abs(a) * e + UPDATE_EPS * torch.maximum(mag, mag_e)
        if k + 1 == num_steps:
            e = e * (1 - m)
        x = xn
    return x, e


def run_trajectory(d, prepare, update, num_steps=NUM_STEPS):
    T, h, w = d["T"], d["h"], d["w"]
    x = d["x"].clone()
    idx = torch.zeros(1, dtype=torch.int32, device=x.device)
    for _ in range(num_steps):
        prepare(x, d["cond_frame"], d["mask"], d["concat_u"], d["concat_c"], d["sigmas"], idx, d["unet_in"], d["c_noise"],
                T, h, w)
        update(x, d["net"], d["cond_frame"], d["mask"], d["scales"], d["sigmas"], idx, num_steps, T, h, w)
    return x, idx


def check_trajectory(x, ref, bound, name):
    rel = rel_l2(x, ref)
    print(f"{name}: 50-step trajectory rel-L2 {rel:.3e}, worst error / bound "
          f"{float(((x.double() - ref).abs() / bound.clamp_min(1e-300)).max()):.3f}")
    assert_elements(x, ref, bound, name)


# ==================================================================================================================
# B. Thin direct convolution (b200v_conv3x3_small_cin)
# ==================================================================================================================
# (NB, H, W, cin, cout, bias, output a column slice of a wider buffer)
CONV_CASES = [(1, 5, 7, 4, 257, True, True),      # 35 tokens: a last block of 3; cout 257: one channel in a second pass
              (2, 1, 9, 3, 100, False, False),    # H = 1, bias NULL
              (3, 6, 1, 8, 256, True, True),      # W = 1; cout 256: exactly one pass of the 256 threads
              (1, 1, 1, 4, 1, True, False),       # one token, one output channel
              (2, 3, 11, 1, 512, False, True),    # cin 1, 66 tokens (3 blocks, the last of 2), two full passes
              (1, 4, 8, 4, 512, True, False)]     # 32 tokens: one full block


def conv_case_id(c):
    return "{}x{}x{}-{}to{}".format(*c[:5]) + ("-bias" if c[5] else "") + ("-slice" if c[6] else "")


def make_conv_inputs(NB, H, W, cin, cout, bias, sliced, device, seed, pad_fill=None):
    """x8 [tokens, 8] fp16 with random values in channels >= cin too (the convolution must ignore them; `pad_fill`
    overrides them), w fp32 [cout, cin, 3, 3], output view with NaN sentinel columns on both sides when `sliced`."""
    M = NB * H * W
    x8 = randn((M, 8), seed, device).half()
    if pad_fill is not None:
        x8[:, cin:] = pad_fill
    w = randn((cout, cin, 3, 3), seed + 1, device, (9 * cin) ** -0.5)
    b = randn((cout,), seed + 2, device) if bias else None
    ex = 16 if sliced else 0
    obuf = torch.full((M, cout + ex), NAN, dtype=torch.float16, device=device)
    out = obuf[:, ex // 2:ex // 2 + cout]
    return x8, w, b, obuf, out


def conv_reference(x8, w, b, NB, H, W, rows=None):
    """fp64 3x3 convolution, padding 1, of channels 0..cin-1 (the tap-GEMM reference with K = 9 cin, tap-major)."""
    cout, cin = w.shape[:2]
    wm = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    return gemm_reference(x8, wm, taps=TAPS_3X3, geom=(W, H, NB), bias=b, rows=rows)


def conv_eps(cin):
    return FAMILY["gemm"].c_acc * math.sqrt(9 * cin) * U24


def check_conv_case(c, op, device, seed=500):
    NB, H, W, cin, cout, bias, sliced = c
    x8, w, b, obuf, out = make_conv_inputs(NB, H, W, cin, cout, bias, sliced, device, seed)
    op(x8, cin, w, b, out, NB, H, W)
    sync(device)
    ref, mag = conv_reference(x8, w, b, NB, H, W)
    assert_conform(out, ref, mag, conv_eps(cin), "gemm", conv_case_id(c))
    if sliced:
        assert bool(torch.isnan(obuf[:, :8]).all()) and bool(torch.isnan(obuf[:, 8 + cout:]).all()), \
            f"{conv_case_id(c)}: sentinel columns overwritten"


# the defect-1 inputs: NaN and Inf in the channels the convolution must ignore
NONFINITE_PAD = (NAN, float("inf"), -float("inf"))


def check_conv_ignores_nonfinite_pad(op, device, cin, fill):
    """Channels cin..7 holding NaN / Inf: the output must be bit-equal to the output with zeros there."""
    NB, H, W, cout = 2, 5, 9, 40
    x0, w, b, _, out0 = make_conv_inputs(NB, H, W, cin, cout, True, False, device, 600 + cin, pad_fill=0.0)
    x1 = x0.clone()
    x1[:, cin:] = fill
    out1 = torch.empty_like(out0)
    op(x0, cin, w, b, out0, NB, H, W)
    op(x1, cin, w, b, out1, NB, H, W)
    sync(device)
    assert torch.equal(out0, out1), f"cin {cin}: {fill} in channels >= cin changes {int((out0 != out1).sum())} outputs"


# ==================================================================================================================
# C. Decoder output (b200v_time_mix_small, b200v_time_mix_small_u8)
# ==================================================================================================================
# (T, H, W, out_frame0, skip_frames, blended frames, keep_f32_from, bias)
TMIX_CASES = [(1, 5, 7, 0, 0, 0, -1, True),      # T = 1: no neighbour frame on either side; HW = 35
              (2, 5, 7, 1, 0, 1, 1, False),      # T = 2, bias NULL, one blended frame, fp32 kept from frame 1
              (5, 5, 7, 2, 1, 2, 3, True),       # a skipped frame, then a blended one
              (14, 8, 16, 11, 0, 3, 14, True)]   # the last chunk of a 25-frame decode: nothing kept

# eps of the time mix: at most 3 taps x 3 channels fused multiply-adds (9 roundings), and up to 3 more in the twin's
# per-tap sums
TMIX_EPS = 12 * U24


def tmix_case_id(c):
    return "T{}-{}x{}-f0{}-skip{}-blend{}-keep{}".format(*c[:7]) + ("-bias" if c[7] else "")


def tmix_weights(device, seed, bias=True):
    w = randn((3, 3, 3), seed, device, 0.5)
    return w, (randn((3,), seed + 1, device, 0.1) if bias else None)


def tmix_reference(x, w, bias, T, HW, prev, out_frame0, blend, skip, terms=None):
    """fp64 AE3DConv time mix, 3 -> 3 channels, kernel (3,1,1), zero padded over frames, of the token-major fp32 x
    [T HW, >= 3], as NCHW frames [T, 3, HW], then the chunk-overlap blend: frames with blend[t] != 0 are
    0.5 (prev + mix) with `prev` the fp32 frames `out` held before the call.  Returns (ref, mag, extra) for
    frames skip..T-1: mag = sum |w||x| + |b| (halved when blended), extra = half an ulp of the blend's sum.  ``terms``
    receives the blend's branches (tests/bias.py): 'mix' (the taps), 'bias' and 'prev', each as it enters the output."""
    C = 3
    v = x[:, :C].double().reshape(T, HW, C)
    w64 = w.double()
    acc = torch.zeros(T, HW, C, dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(acc)
    for kt in range(3):
        for t in range(T):
            tt = t + kt - 1
            if 0 <= tt < T:
                acc[t] += v[tt] @ w64[:, :, kt].t()
                mag[t] += v[tt].abs() @ w64[:, :, kt].abs().t()
    mix = acc.permute(0, 2, 1)[skip:]
    b = torch.zeros_like(mix) if bias is None else bias.double().reshape(1, C, 1).expand_as(mix)
    acc, mag = mix + b, (mag.permute(0, 2, 1)[skip:] + b.abs())
    extra = torch.zeros_like(acc)
    p = torch.zeros_like(acc)
    half = torch.ones_like(acc[:, :1, :1])
    if blend is not None:
        bl = blend.bool()[skip:].reshape(-1, 1, 1)
        p = torch.where(bl, prev.reshape(prev.shape[0], C, HW)[out_frame0 + skip:out_frame0 + T].double(), p)
        extra = torch.where(bl, 0.5 * ulp(p.abs() + acc.abs(), torch.float32), extra)
        half = torch.where(bl, 0.5, 1.0)
        acc = torch.where(bl, 0.5 * (p + acc), acc)
        mag = torch.where(bl, 0.5 * mag, mag)
    if terms is not None:
        terms.update(mix=half * mix, bias=half * b, prev=0.5 * p)
    return acc, mag, extra


def u8_path(v: torch.Tensor) -> torch.Tensor:
    """The reference's output path on fp32 frames: (255 * clamp((v + 1) / 2, 0, 1)).astype(uint8), in fp32."""
    return (255.0 * torch.clamp((v.float() + 1.0) / 2.0, 0.0, 1.0)).to(torch.uint8)


def u8_exact(v64: torch.Tensor) -> torch.Tensor:
    """The same path in fp64: floor(255 clamp((v + 1) / 2, 0, 1))."""
    return torch.floor(255.0 * torch.clamp((v64 + 1.0) / 2.0, 0.0, 1.0)).to(torch.uint8)


def check_u8_bytes(got, ref, tol, name):
    """Every byte between u8(ref - tol') and u8(ref + tol') (u8 is monotone), tol' the fp32 bound of the frame value plus
    the output path's own fp32 roundings ((v + 1) and 255 s: 2 U24 |v + 1|).  Only bytes whose fp64 value is within that
    bound of a truncation boundary may differ from u8(ref), and only by one.  Returns the count of those that do."""
    t = tol + 2 * U24 * (ref + 1.0).abs()
    lo, hi, mid = u8_exact(ref - t), u8_exact(ref + t), u8_exact(ref)
    bad = (got < lo) | (got > hi)
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} bytes outside [u8(ref - tol), u8(ref + tol)]"
    n = int((got != mid).sum())
    print(f"{name}: {n} of {got.numel()} bytes differ from the fp64 truncation (by one, at a boundary)")
    return n


def check_tmix_call(fp32_op, u8_op, x, w, bias, out, out8, blend, T, HW, out_frame0, skip, keep, name, device):
    """One call of the fp32 and of the uint8 kernel on the same `out` state: fp32 frames against the fp64 mix, bytes
    against the fp64 output path and bit-equal to the fp32 output path on the fp32 kernel's frames, and untouched memory:
    fp32 frames outside [out_frame0 + skip, out_frame0 + T) and below keep_f32_from, bytes outside the written frames."""
    C = 3
    F_ = out.shape[0]
    prev, prev8 = out.clone(), out8.clone()
    ref, mag, extra = tmix_reference(x, w, bias, T, HW, prev, out_frame0, blend, skip)
    lo, hi = out_frame0 + skip, out_frame0 + T
    # fp32 kernel on a copy of the state
    o32 = prev.clone()
    fp32_op(x, w, bias, o32, blend, T, HW, C, out_frame0, skip)
    sync(device)
    got = o32.reshape(F_, C, HW)[lo:hi]
    assert_conform(got, ref, mag, TMIX_EPS, "elementwise", f"{name}: fp32 frames", extra=extra)
    assert same_bits(o32[:lo], prev[:lo]) and same_bits(o32[hi:], prev[hi:]), f"{name}: fp32 kernel wrote outside"
    # uint8 kernel on the real state
    u8_op(x, w, bias, out, out8, blend, T, HW, C, out_frame0, skip, keep)
    sync(device)
    b = out8[lo:hi].permute(0, 3, 1, 2).reshape(hi - lo, C, HW)
    tol = ulp(ref, torch.float32) + TMIX_EPS * mag + extra
    check_u8_bytes(b, ref, tol, f"{name}: bytes")
    assert torch.equal(b, u8_path(got)), f"{name}: bytes are not the output path applied to the fp32 frames"
    assert torch.equal(out8[:lo], prev8[:lo]) and torch.equal(out8[hi:], prev8[hi:]), f"{name}: bytes written outside"
    k0 = lo if keep < 0 else max(lo, out_frame0 + keep)
    assert same_bits(out[:k0], prev[:k0]) and same_bits(out[hi:], prev[hi:]), f"{name}: fp32 frames not kept written"
    assert same_bits(out[k0:hi], o32[k0:hi]), f"{name}: kept fp32 frames differ from the fp32 kernel's"


def tmix_inputs(T, H, W, device, seed, ld=8):
    """x [T H W, ld] fp32 token rows, columns 3.. NaN (the decoder's output rows: 8 columns, 3 used)."""
    x = randn((T * H * W, ld), seed, device, 0.8)
    x[:, 3:] = NAN
    return x


def check_tmix_case(c, fp32_op, u8_op, device):
    T, H, W, f0, skip, nb, keep, bias = c
    HW = H * W
    F_ = f0 + T + 2
    x = tmix_inputs(T, H, W, device, 900 + T)
    w, b = tmix_weights(device, 910 + T, bias)
    out = randn((F_, 3, H, W), 920 + T, device)
    out8 = torch.full((F_, H, W, 3), 0xA5, dtype=torch.uint8, device=device)
    blend = None
    if nb:
        blend = torch.zeros(T, dtype=torch.int32, device=device)
        blend[:nb] = 1
    check_tmix_call(fp32_op, u8_op, x, w, b, out, out8, blend, T, HW, f0, skip, keep, tmix_case_id(c), device)


def boundary_values():
    """Frame values at and beyond +-1 and at exact truncation boundaries of the output path: v_k = 2 k / 255 - 1 in fp32
    and its two fp32 neighbours, for every k."""
    k = torch.arange(256, dtype=torch.float64)
    vk = (2.0 * k / 255.0 - 1.0).float()
    up = torch.nextafter(vk, torch.full_like(vk, 2.0))
    dn = torch.nextafter(vk, torch.full_like(vk, -2.0))
    special = torch.tensor([-3.0, -1.5, -1.0 - 2 ** -23, -1.0, -1.0 + 2 ** -24, 0.0, 1.0 - 2 ** -24, 1.0, 1.0 + 2 ** -23,
                            1.5, 3.0, 1e30, -1e30])
    return torch.cat([vk, up, dn, special])


def check_tmix_boundaries(fp32_op, u8_op, device):
    """The time mix as the identity (middle tap = I, bias NULL): the frames are x exactly, so the bytes are the output
    path of chosen values: +-1, beyond, every truncation boundary and its fp32 neighbours."""
    vals = boundary_values()
    T, H, W = 3, 8, 33
    n = T * H * W * 3
    v = vals.repeat(-(-n // vals.numel()))[:n].reshape(T, 3, H * W).permute(0, 2, 1).reshape(-1, 3)
    x = torch.full((T * H * W, 8), NAN)
    x[:, :3] = v
    w = torch.zeros(3, 3, 3)
    w[:, :, 1] = torch.eye(3)
    x, w = x.to(device), w.to(device)
    out = torch.zeros(T, 3, H, W, device=device)
    out8 = torch.zeros(T, H, W, 3, dtype=torch.uint8, device=device)
    check_tmix_call(fp32_op, u8_op, x, w, None, out, out8, None, T, H * W, 0, 0, -1, "identity mix at boundaries", device)
    want = v.reshape(T, H * W, 3).permute(0, 2, 1).to(device)
    assert torch.equal(out.reshape(T, 3, H * W), want), "the identity mix must reproduce its input exactly"
    # at a boundary the fp32 path may truncate to either side of the fp64 one: the bytes are the fp32 path's
    assert torch.equal(out8.permute(0, 3, 1, 2).reshape(T, 3, H * W), u8_path(want))


def decode_chunk_plan(F_=25, n_samples=14, overlap=3):
    """decode_first_stage(u8=True)'s calls: (first input frame, frames, out_frame0, blended frames, keep_f32_from)."""
    from vista_b200.vae import _decode_chunks
    chunks = _decode_chunks(F_, n_samples, overlap)
    plan = []
    for ci, (f0, n, o0, nov) in enumerate(chunks):
        keep = n if ci + 1 == len(chunks) else max(0, chunks[ci + 1][2] - o0)
        plan.append((f0, n, o0, nov, keep))
    return plan


def check_decode_sequence(fp32_op, u8_op, H, W, device):
    """The chunk calls of decode_first_stage(u8=True) at T = 25 on one (out, out8) pair, in order: each call against the
    state the previous ones left (the blend reads the fp32 frames the previous chunk kept)."""
    F_, HW = 25, H * W
    out = torch.full((F_, 3, H, W), NAN, device=device)
    out8 = torch.full((F_, H, W, 3), 0xA5, dtype=torch.uint8, device=device)
    w, b = tmix_weights(device, 950)
    for i, (f0, n, o0, nov, keep) in enumerate(decode_chunk_plan()):
        x = tmix_inputs(n, H, W, device, 960 + i)
        blend = None
        if nov:
            blend = torch.zeros(n, dtype=torch.int32, device=device)
            blend[:nov] = 1
        check_tmix_call(fp32_op, u8_op, x, w, b, out, out8, blend, n, HW, o0, 0, keep, f"decode chunk {i}", device)
    assert not bool((out8 == 0xA5).all(dim=(1, 2, 3)).any()), "a frame of the decode was never written"


def check_session_round(fp32_op, u8_op, H, W, device):
    """RolloutSession._decode of a round after the first: two chunks of 14 frames into a 14-frame fp32 buffer, each
    blending its first 3 frames with the carried fp32 frames and keeping frames 11..13 for the next chunk; the bytes of
    chunk k go to out8[11 k:]."""
    HW = H * W
    f32 = torch.empty(14, 3, H, W, device=device)
    out8 = torch.full((25, H, W, 3), 0xA5, dtype=torch.uint8, device=device)
    carry = randn((3, 3, H, W), 970, device)
    w, b = tmix_weights(device, 971)
    blend = torch.zeros(14, dtype=torch.int32, device=device)
    blend[:3] = 1
    for k, o0 in enumerate((0, 11)):
        f32[:3].copy_(carry)
        x = tmix_inputs(14, H, W, device, 980 + k)
        check_tmix_call(fp32_op, u8_op, x, w, b, f32, out8[o0:], blend, 14, HW, 0, 0, 11, f"session chunk {k}", device)
        carry = f32[11:].clone()


# ==================================================================================================================
# D. Rollout glue (b200v_rollout_advance, b200v_ensemble_reward)
# ==================================================================================================================
def rollout_advance_reference(sample, z0, samples_z, filled, dst0, src0, n_cond):
    """sample[0] = z0[0] (first round), samples_z[dst0 + t] = sample[t] for t >= src0, filled = the last n_cond rows of
    sample then zeros.  Pure data movement: the kernel must match exactly."""
    T = sample.shape[0]
    s, sz = sample.clone(), samples_z.clone()
    if z0 is not None:
        s[0] = z0[0]
    sz[dst0 + src0:dst0 + T] = s[src0:]
    f = None
    if filled is not None:
        f = torch.zeros_like(filled)
        f[:n_cond] = s[T - n_cond:]
    return s, sz, f


def rollout_cases(T=25):
    """(n_cond, round r, src0, z0 given, filled given): every n_cond in {0, 1, 3, T} over rounds 0..3 at destination
    r (T - n), the source frame rotating over {0, n_cond, T}, z0 on round 0 (and with filled NULL on round 3)."""
    cases = []
    for n in (0, 1, 3, T):
        for r in range(4):
            cases.append((n, r, (0, n, T)[r % 3], r in (0, 3), r != 3))
    return cases


def check_rollout_advance(op, E, device, T=25):
    """Every case on one samples_z per n_cond, sentinel rows everywhere nothing may be written."""
    for n, r, src0, with_z0, with_filled in rollout_cases(T):
        name = f"E {E} n_cond {n} round {r} src0 {src0} z0 {with_z0} filled {with_filled}"
        dst0 = r * (T - n)
        seed = 1000 + 17 * n + r
        sample = randn((T, E), seed, device)
        z0 = randn((2, E), seed + 1, device) if with_z0 else None
        samples_z = torch.full((dst0 + T + 2, E), -777.0, device=device)
        filled = torch.full((T, E), 555.0, device=device) if with_filled else None
        s_ref, sz_ref, f_ref = rollout_advance_reference(sample, z0, samples_z, filled, dst0, src0, n)
        op(sample, z0, samples_z, filled, dst0, src0, n)
        sync(device)
        assert torch.equal(sample, s_ref), f"{name}: sample"
        assert torch.equal(samples_z, sz_ref), f"{name}: samples_z (rows outside [dst0 + src0, dst0 + T) are sentinels)"
        if with_filled:
            assert torch.equal(filled, f_ref), f"{name}: filled"
        if n == T and with_z0 and with_filled:
            assert torch.equal(filled[0], z0[0]), f"{name}: filled row 0 must come from z0"


def reward_reference(members):
    """fp64 mean variance of reward_utils (mean over the ensemble, unbiased variance, mean over elements) and its bound.

    The kernel evaluates per element, in fp32: u = (sum_k m_k) / K, within U24 S1 of the exact mean (K - 1 roundings of
    a sum bounded by S1 = sum_k |m_k|, then / K); e_k = m_k - u within du + U24 |e_k|; sum_k e_k^2 within
    2 du sum_k |e_k| + (K + 2) U24 sum_k e_k^2 + K du^2; / (K - 1) one more rounding.  The mean over n elements is fp64
    (n 2^-53 relative), the store rounds to fp32 (one ulp)."""
    K, n = len(members), members[0].numel()
    u = sum(x.reshape(-1).double() for x in members) / K
    s1, se, se2 = (torch.zeros_like(u) for _ in range(3))
    for x in members:
        x = x.reshape(-1).double()
        e = x - u
        s1 += x.abs()
        se += e.abs()
        se2 += e * e
    var = se2 / (K - 1)
    du = U24 * s1
    bound = (2 * du * se + (K + 2) * U24 * se2 + K * du * du) / (K - 1) + U24 * var
    mv = var.mean()
    tol = bound.mean() + n * 2.0 ** -53 * mv
    return float(mv), float(tol)


# (K, n, common offset in standard deviations)
REWARD_CASES = [(2, 1, 0), (3, 255, 0), (5, 256, 0), (64, 257, 0), (5, 25 * 4 * 72 * 128, 0), (2, 25 * 4 * 72 * 128, 30),
                (64, 25 * 4 * 72 * 128, 30), (3, 2 * 4096 * 256 + 37, 0)]     # the last: every thread of the capped grid loops


def reward_members(K, n, offset, device, seed):
    base = randn((n,), seed, device, 0.5)
    return [(base + randn((n,), seed + 1 + k, device, 1.0 + 0.05 * k) + offset).contiguous() for k in range(K)]


def check_reward(out, members, name):
    """out = [mean variance, reward]: mv within its bound of the fp64 reference, the reward within 2 ulp of exp(-mv) of
    the returned mv (expf is documented within 2 ulp) and close to the fp64 reward."""
    mv_ref, tol = reward_reference(members)
    mv, r = float(out[0]), float(out[1])
    tol_mv = tol + float(ulp(torch.tensor(mv_ref, dtype=torch.float64), torch.float32))
    assert abs(mv - mv_ref) <= tol_mv, f"{name}: mean variance {mv!r} vs {mv_ref!r} (bound {tol_mv:.3g})"
    e = math.exp(-mv)
    u = float(ulp(torch.tensor(e, dtype=torch.float64), torch.float32))
    assert abs(r - e) <= 2 * u, f"{name}: reward {r!r} vs exp(-mv) {e!r}"
    assert abs(r - math.exp(-mv_ref)) <= 2 * u + math.exp(-mv_ref) * tol_mv * 1.01, f"{name}: reward vs fp64"
    print(f"{name}: mv {mv:.8g} ref {mv_ref:.8g} (|err| {abs(mv - mv_ref):.3g}, bound {tol_mv:.3g}); reward {r:.8g}")


def identical_members(K, n, device):
    """K copies of values with 11 significant bits: every partial sum k m (k <= 64) is exact, so u == m exactly."""
    m = randn((n,), 1234, device).half().float()
    return [m.clone() for _ in range(K)]


# ==================================================================================================================
# E. Embedding helpers and layout converters
# ==================================================================================================================
def timestep_embedding_reference(t, dim, max_period=10000.0):
    """fp64 [cos(t f_k) | sin(t f_k)], f_k = exp(-ln(P) k / (dim / 2)) (the reference's frequencies), and the magnitude
    for eps = U24: logf (2 U24 relative) and the two roundings of -ln(P) k / half put 4 U24 |ln P| on the exponent, expf
    4 U24 (2 ulp) and t f one U24 on the argument a: (4 |ln P| + 5) U24 |a| through cos / sin (slope <= 1), plus
    cosf / sinf within 2 ulp (<= 4 U24 absolute)."""
    half = dim // 2
    k = torch.arange(half, dtype=torch.float64, device=t.device)
    a = t.double().reshape(-1, 1) * torch.exp(-math.log(max_period) * k / half)
    ref = torch.cat([torch.cos(a), torch.sin(a)], dim=1)
    m = a.abs() * (4 * abs(math.log(max_period)) + 5) + 4
    return ref, torch.cat([m, m], dim=1)


def temb_cases():
    """(name, t, dim): c_noise over the 50-step schedule at width 320, frame indices 0..24 at 320 / 640 / 1280."""
    s = edm_sigmas()[:NUM_STEPS]
    c_noise = 0.25 * torch.log(s)
    frames = torch.arange(25, dtype=torch.float32)
    return [("c_noise-320", c_noise, 320), ("frames-320", frames, 320), ("frames-640", frames, 640),
            ("frames-1280", frames, 1280)]


def check_temb(op, name, t, dim, device):
    """Strided output with NaN sentinel columns on both sides."""
    t = t.to(device).contiguous()
    buf = torch.full((t.numel(), dim + 16), NAN, dtype=torch.float16, device=device)
    out = buf[:, 8:8 + dim]
    op(t, out, dim)
    sync(device)
    ref, mag = timestep_embedding_reference(t, dim)
    assert_conform(out, ref, mag, U24, "elementwise", f"timestep_embedding {name}")
    assert bool(torch.isnan(buf[:, :8]).all()) and bool(torch.isnan(buf[:, 8 + dim:]).all()), f"{name}: sentinels"


# blend_emb: e = e_plain (1 - m) + e_cond m + label; (1 - m), two products and two sums: 5 U24 on the magnitude
BLEND_EPS = 5 * U24


def blend_emb_combos():
    """Every combination of the arguments the ABI allows to be NULL (e_plain is required)."""
    return [(ec, lb, mk, em, se) for ec in (0, 1) for lb in (0, 1) for mk in (0, 1) for em in (0, 1) for se in (0, 1)]


def check_blend_emb(op, combo, device, rows=7, dim=320):
    ec, lb, mk, em, se = combo
    name = "blend_emb e_cond {} label {} mask {} emb {} silu {}".format(*combo)
    e_plain = randn((rows, dim), 1300, device)
    e_cond = randn((rows, dim), 1301, device) if ec else None
    label = randn((rows, dim), 1302, device) if lb else None
    mask = torch.rand(rows, generator=gen(1303)).to(device) if mk else None
    if mask is not None:
        mask[:2] = torch.tensor([0.0, 1.0])
    emb = torch.full((rows, dim), NAN, device=device) if em else None
    semb = torch.full((rows, dim), NAN, dtype=torch.float16, device=device) if se else None
    op(e_plain, e_cond, label, mask, emb, semb)
    sync(device)
    m = torch.zeros(rows, 1, dtype=torch.float64, device=device) if mask is None else mask.double().reshape(-1, 1)
    ref = e_plain.double() * (1 - m)
    mag = e_plain.double().abs() * (1 - m).abs()
    if e_cond is not None:
        ref, mag = ref + e_cond.double() * m, mag + e_cond.double().abs() * m.abs()
    if label is not None:
        ref, mag = ref + label.double(), mag + label.double().abs()
    if emb is not None:
        assert_conform(emb, ref, mag, BLEND_EPS, "elementwise", f"{name}: emb")
    if semb is not None:
        # silu_f: ex2.approx of a rounded -x log2 e (|x| + 4 U24 relative on exp(-x)), 1 + e, rcp.approx (2 U24), the
        # product: (|x| + 8) U24 relative on silu; the input's BLEND_EPS mag through silu' <= 1.1
        s = F.silu(ref)
        assert_conform(semb, s, 1.1 * BLEND_EPS / U24 * mag + (ref.abs() + 8) * s.abs(), U24, "elementwise",
                       f"{name}: silu_emb")


# (NB, C, H, W, row stride of the token buffer, source dtype of tokens_to_nchw)
LAYOUT_CASES = [(50, 4, 72, 128, 64, torch.float16),       # the UNet input rows: 64-column padded layout
                (3, 3, 5, 7, 8, torch.float32),            # encoder moments / decoder output rows, odd sizes
                (2, 8, 9, 11, 16, torch.float16),
                (1, 1, 1, 1, 8, torch.float32)]


def check_layout(nchw_op, tok_op, case, device):
    NB, C, H, W, ld, dt = case
    name = f"layout {NB}x{C}x{H}x{W} ld {ld} {dt}"
    x = randn((NB, C, H, W), 1400 + C, device, 2.0)
    buf = torch.full((NB * H * W, ld), NAN, dtype=torch.float16, device=device)
    nchw_op(x, buf[:, :max(C, 1)], NB, C, H, W)
    sync(device)
    want = x.permute(0, 2, 3, 1).reshape(NB * H * W, C).half()
    assert torch.equal(buf[:, :C], want), f"{name}: nchw_to_tokens"
    assert bool(torch.isnan(buf[:, C:]).all()), f"{name}: columns >= C written"
    src = randn((NB * H * W, ld), 1410 + C, device).to(dt)
    out = torch.full((NB, C, H, W), NAN, device=device)
    tok_op(src, out, NB, C, H, W)
    sync(device)
    assert torch.equal(out, src[:, :C].float().reshape(NB, H, W, C).permute(0, 3, 1, 2)), f"{name}: tokens_to_nchw"


IM2COL_S2_CASES = [(2, 5, 7, 64), (1, 9, 3, 8), (3, 1, 1, 16), (1, 8, 8, 32)]


def im2col_s2_reference(x, NB, H, W, C):
    """Zero padding of one on every side, a 3x3 stride-2 unfold, tap-major columns: Ho = (H - 1) // 2 + 1."""
    img = x[:, :C].reshape(NB, H, W, C).permute(0, 3, 1, 2).float()
    u = F.unfold(F.pad(img, (1, 1, 1, 1)), kernel_size=3, stride=2)
    L = u.shape[-1]
    return u.reshape(NB, C, 9, L).permute(0, 3, 2, 1).reshape(NB * L, 9 * C).to(x.dtype)


def check_im2col_s2(op, case, device):
    NB, H, W, C = case
    x = padded(NB * H * W, C, 16, 1500 + H, device, offset=8)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.full((NB * Ho * Wo, 9 * C), NAN, dtype=torch.float16, device=device)
    op(x, out, NB, H, W, C)
    sync(device)
    assert torch.equal(out, im2col_s2_reference(x, NB, H, W, C)), f"im2col_s2 {case}"


UPSAMPLE_CASES = [(2, 3, 5, 16), (1, 1, 1, 8), (3, 4, 7, 64)]


def check_upsample2x(op, case, device):
    """x and out with row strides C + 8 and C + 16 (views), sentinel columns of out untouched."""
    NB, H, W, C = case
    x = padded(NB * H * W, C, 8, 1600 + W, device)
    obuf = torch.full((NB * 4 * H * W, C + 16), NAN, dtype=torch.float16, device=device)
    out = obuf[:, 8:8 + C]
    op(x, out, NB, H, W, C)
    sync(device)
    img = x.reshape(NB, H, W, C)
    want = img.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, C)
    assert torch.equal(out, want), f"upsample2x {case}"
    assert bool(torch.isnan(obuf[:, :8]).all()) and bool(torch.isnan(obuf[:, 8 + C:]).all())


# ==================================================================================================================
# F. CLIP attention (b200v_attention_d80)
# ==================================================================================================================
# (batch, seq, heads): seq 1 / 2, one short of / exactly / one past a 64-key block, two blocks, 257 = the CLIP tokens
D80_CASES = [(1, 1, 1), (25, 2, 1), (1, 63, 16), (25, 64, 1), (1, 65, 16), (1, 128, 1), (2, 129, 16), (1, 257, 1),
             (25, 257, 16)]
D80_SCALE = 80 ** -0.5


def d80_inputs(batch, seq, heads, device, seed, qk_scale=1.0, identical_keys=False):
    """q / k / v as column blocks of one fused in-projection output [tokens, 3 C + 16] (padded row stride)."""
    C = heads * 80
    qkv = randn((batch * seq, 3 * C + 16), seed, device).half()
    if qk_scale != 1.0:
        qkv[:, :2 * C] = (qkv[:, :2 * C].float() * qk_scale).half()
    if identical_keys:
        qkv[:, C:2 * C] = qkv[:1, C:2 * C]
    return qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:3 * C]


def d80_reference(q, k, v, batch, seq, heads):
    """The spatial attention's bound with scale 1/sqrt(80): P is rounded unnormalised (exp(s - running max) <= 1), so
    the absolute subnormal term is divided by the fp64 row sum."""
    sp = lambda t: t.double().reshape(batch, seq, heads, 80).permute(0, 2, 1, 3)
    o, m = attention_reference(sp(q), sp(k), sp(v), p_normalised=False, scale=D80_SCALE)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(batch * seq, heads * 80)
    return back(o), back(m)


def check_d80(op, batch, seq, heads, device, seed=1700, qk_scale=1.0, identical_keys=False, name="d80"):
    C = heads * 80
    q, k, v = d80_inputs(batch, seq, heads, device, seed, qk_scale, identical_keys)
    obuf = torch.full((batch * seq, C + 16), NAN, dtype=torch.float16, device=device)
    out = obuf[:, 8:8 + C]
    op(q, k, v, out, batch, seq, heads)
    sync(device)
    ref, mag = d80_reference(q, k, v, batch, seq, heads)
    assert_conform(out, ref, mag, ATTN_EPS, "attn", f"{name} {batch}x{seq}x{heads}")
    assert bool(torch.isnan(obuf[:, :8]).all()) and bool(torch.isnan(obuf[:, 8 + C:]).all()), f"{name}: sentinels"
    return ref


# logits of about +-30: q and k scaled so that q.k / sqrt(80) has a standard deviation of about 12
D80_LARGE_QK = 12.0 ** 0.5


# ==================================================================================================================
# G. Which conformance tests hold each kernel
# ==================================================================================================================
_G = "test_conformance_gpu.py::"
_S = "test_conformance_small_gpu.py::"
_P = "test_production_conformance_gpu.py::"
_STEP, _DEC, _COND, _SESS = (_P + "test_sampler_step_production", _P + "test_decode_production",
                             _P + "test_condition_and_encode_production", _P + "test_session_production")
_N = "test_norm_statistics_gpu.py::"
_B = "test_bias_conformance_gpu.py::"
_BIAS = [_B + "test_production_keys_clean", _B + "test_planted_defect_fails_the_gain_check"]
KERNEL_TESTS = {
    "tapgemm_kernel": [_G + "test_gemm_sweep", _G + "test_gemm_production_conv_sampled", _STEP, _DEC, _COND,
                       _N + "test_gemm_stats_offset_and_flat", _N + "test_gemm_stats_partial_last_tile"] + _BIAS,
    "attn_spatial_kernel": [_G + "test_attention_spatial_edges", _G + "test_attention_spatial_level0_sampled", _STEP] + _BIAS,
    "attn_temporal_kernel": [_G + "test_attention_temporal_conformance", _G + "test_attention_temporal_sharded", _STEP],
    "gn_stats_kernel": [_G + "test_groupnorm_conformance", _G + "test_groupnorm_sums_finalize_sharded", _STEP, _COND,
                        _N + "test_groupnorm_offset_and_flat", _N + "test_groupnorm_offset_and_flat_decoder_scale",
                        _N + "test_sharded_offset_and_flat"],
    "gn_apply_kernel": [_G + "test_groupnorm_conformance", _G + "test_groupnorm_sums_finalize_sharded", _STEP, _DEC,
                        _N + "test_groupnorm_offset_and_flat", _N + "test_gemm_stats_offset_and_flat",
                        _N + "test_sharded_offset_and_flat"] + _BIAS,
    "gn_finalize_kernel": [_G + "test_groupnorm_sums_finalize_sharded", _N + "test_sharded_offset_and_flat"],
    "gn_from_partials_kernel": [_G + "test_groupnorm_from_partials_raw_sums_sharded", _STEP, _DEC,
                                _N + "test_gemm_stats_offset_and_flat", _N + "test_sharded_offset_and_flat"] + _BIAS,
    "layernorm_kernel": [_G + "test_layernorm_conformance", _STEP, _COND, _N + "test_layernorm_offset_and_flat"],
    "layernorm40_kernel": [_G + "test_layernorm_conformance", _STEP, _N + "test_layernorm_offset_and_flat"],
    "softmax_rows_kernel": [_G + "test_softmax_rows_conformance", _DEC, _COND],
    "im2col_s2_asym_kernel": [_G + "test_im2col_s2_asym_exact", _COND],
    "clip_preprocess_kernel": ["test_clip_gpu.py::test_preprocess_matches_oracle", _COND],
    "sinusoid_embed_kernel": ["test_conditioner_gpu.py::test_sinusoid_embed_matches_formula", _COND],
    "sampler_prepare_kernel": [_S + "test_sampler_step", _S + "test_sampler_trajectory_and_graph_replay", _STEP],
    "sampler_update_kernel": [_S + "test_sampler_step", _S + "test_sampler_trajectory_and_graph_replay", _STEP],
    "conv3x3_small_cin_kernel": [_S + "test_conv3x3_small_cin_edges", _S + "test_conv3x3_small_cin_production",
                                 _S + "test_conv3x3_small_cin_ignores_nonfinite_pad_channels", _DEC, _COND],
    "time_mix_small_kernel": [_S + "test_time_mix_cases", _S + "test_time_mix_decode_and_session_chunks"],
    "time_mix_small_u8_kernel": [_S + "test_time_mix_cases", _S + "test_time_mix_boundaries",
                                 _S + "test_time_mix_decode_and_session_chunks", _DEC] + _BIAS,
    "rollout_advance_kernel": [_S + "test_rollout_advance", _SESS],
    "ensemble_reward_kernel": [_S + "test_ensemble_reward", _S + "test_ensemble_reward_identical_members",
                               _S + "test_ensemble_reward_back_to_back", _SESS],
    "timestep_embedding_kernel": [_S + "test_timestep_embedding", _STEP],
    "blend_emb_kernel": [_S + "test_blend_emb", _STEP],
    "nchw_to_tokens_kernel": [_S + "test_layout_converters", _DEC, _COND],
    "tokens_to_nchw_kernel": [_S + "test_layout_converters", _COND],
    "im2col_s2_kernel": [_S + "test_im2col_s2", _STEP],
    "upsample2x_kernel": [_S + "test_upsample2x", _STEP],
    "attn_d80_kernel": [_S + "test_attention_d80", _S + "test_attention_d80_identical_keys_and_large_logits", _COND],
}
NOT_HELD = {
    "peer_put_kernel": "needs two or more GPUs; test_sharded_gpu.py covers the peer-memory transport",
    "peer_wait_kernel": "needs two or more GPUs; test_sharded_gpu.py covers the peer-memory transport",
    "peer_allreduce_f64_kernel": "needs two or more GPUs; test_sharded_gpu.py covers the peer-memory transport",
    "conv3x3_small_cout_kernel": "no caller on the product path",
    "step_inc_kernel": "its one effect, the step counter, is checked through step_idx by the sampler tests",
}
# kernels of NOT_HELD the single-GPU product path does launch (checked indirectly, as the reason says)
LAUNCHED_NOT_HELD = {"step_inc_kernel"}


def source_kernels():
    """Names of every __global__ function in vista_b200/csrc/."""
    csrc = os.path.join(ROOT, "vista_b200", "csrc")
    pat = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(")
    names = set()
    for f in sorted(os.listdir(csrc)):
        if f.endswith((".cu", ".cuh")):
            names.update(pat.findall(open(os.path.join(csrc, f)).read()))
    return names


def _test_functions(path):
    tree = ast.parse(open(path).read())
    return {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}


# ==================================================================================================================
# CPU run: the twins on the case tables
# ==================================================================================================================
@pytest.mark.parametrize("step", SAMPLER_STEPS)
@pytest.mark.parametrize("case", [c for c in SAMPLER_CASES if c[1] * c[2] <= 128], ids=sampler_case_id)
def test_sampler_step_twin(case, step):
    """The sampler twins at the schedule's first, middle and last step (sigma' = 0, conditioning frames re-imposed)."""
    check_sampler_step(case, step, fake_ops.sampler_prepare, fake_ops.sampler_update, CPU)


def test_sampler_trajectory_twin():
    """50 twin steps at 25 x 8 x 16 against the fp64 trajectory, within the accumulated per-step bound."""
    d = trajectory_inputs(25, 8, 16, CPU)
    ref, bound = trajectory_reference(d)
    x, idx = run_trajectory(d, fake_ops.sampler_prepare, fake_ops.sampler_update)
    assert int(idx[0]) == NUM_STEPS
    check_trajectory(x, ref, bound, "twin")


def test_sampler_reference_is_the_oracle_step():
    """The fp64 update restates the oracle's Euler step: vscaling_edm_cnoise's coefficients and the guider mix."""
    from oracle import vista_oracle as vo
    d = make_sampler_inputs((3, 5, 7, "none", False, False, "triangle"), CPU)
    for step in SAMPLER_STEPS:
        s = d["sigmas"][step].double()
        c_skip, c_out, c_in, c_noise = vo.vscaling_edm_cnoise(s)
        assert abs(float(c_in) - (float(s) ** 2 + 1) ** -0.5) < 1e-15
        assert abs(float(c_noise) - 0.25 * math.log(float(s))) < 1e-12
        xn, _, _ = update_reference(d["x"], d, step)
        T = d["T"]
        hw = d["h"] * d["w"]
        u = d["net"][:T * hw, :4].double().reshape(T, d["h"], d["w"], 4).permute(0, 3, 1, 2)
        c = d["net"][T * hw:, :4].double().reshape(T, d["h"], d["w"], 4).permute(0, 3, 1, 2)
        x = d["x"].double()
        du, dc = u * float(c_out) + x * float(c_skip), c * float(c_out) + x * float(c_skip)
        den = du + d["scales"].double().reshape(T, 1, 1, 1) * (dc - du)
        want = x + (x - den) / float(s) * (float(d["sigmas"][step + 1]) - float(s))
        assert torch.allclose(xn, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("case", CONV_CASES, ids=conv_case_id)
def test_conv3x3_small_cin_twin(case):
    check_conv_case(case, fake_ops.conv3x3_small_cin, CPU)


@pytest.mark.parametrize("fill", NONFINITE_PAD)
def test_conv3x3_small_cin_twin_ignores_nonfinite_pad(fill):
    for cin in (1, 3, 4):
        check_conv_ignores_nonfinite_pad(fake_ops.conv3x3_small_cin, CPU, cin, fill)


@pytest.mark.parametrize("case", TMIX_CASES, ids=tmix_case_id)
def test_time_mix_twin(case):
    check_tmix_case(case, fake_ops.time_mix_small, fake_ops.time_mix_small_u8, CPU)


def test_time_mix_twin_boundaries_and_decode():
    check_tmix_boundaries(fake_ops.time_mix_small, fake_ops.time_mix_small_u8, CPU)
    check_decode_sequence(fake_ops.time_mix_small, fake_ops.time_mix_small_u8, 4, 8, CPU)
    check_session_round(fake_ops.time_mix_small, fake_ops.time_mix_small_u8, 4, 8, CPU)


def test_decode_chunk_plan():
    """The plan the decode tests replay: two chunks of 14 frames, the second blending 3 frames and starting at frame 11;
    the first keeps fp32 from frame 11 on, the last keeps nothing."""
    assert decode_chunk_plan() == [(0, 14, 0, 0, 11), (11, 14, 11, 3, 14)]


@pytest.mark.parametrize("E", [37, 4 * 8 * 16])
def test_rollout_advance_twin(E):
    check_rollout_advance(fake_ops.rollout_advance, E, CPU)


@pytest.mark.parametrize("K,n,offset", REWARD_CASES)
def test_ensemble_reward_twin(K, n, offset):
    members = reward_members(K, n, offset, CPU, 1100 + K)
    check_reward(fake_ops.ensemble_reward(members), members, f"twin K {K} n {n} offset {offset}")


def test_ensemble_reward_bound_detects_biased_variance():
    """The mv bound is tight enough to tell K from K - 1 at K = 64 with a 30-sigma common offset (a factor 63 / 64)."""
    members = reward_members(64, 4096, 30, CPU, 1200)
    mv, tol = reward_reference(members)
    assert mv / 64 > 10 * (tol + float(ulp(torch.tensor(mv, dtype=torch.float64), torch.float32)))


@pytest.mark.parametrize("K", [2, 3, 5, 64])
def test_ensemble_reward_twin_identical_members(K):
    out = fake_ops.ensemble_reward(identical_members(K, 1000, CPU))
    assert torch.equal(out, torch.tensor([0.0, 1.0]))


@pytest.mark.parametrize("name,t,dim", temb_cases(), ids=[c[0] for c in temb_cases()])
def test_timestep_embedding_twin(name, t, dim):
    check_temb(fake_ops.timestep_embedding, name, t, dim, CPU)


@pytest.mark.parametrize("combo", blend_emb_combos())
def test_blend_emb_twin(combo):
    check_blend_emb(fake_ops.blend_emb, combo, CPU)


@pytest.mark.parametrize("case", LAYOUT_CASES[1:])
def test_layout_twins(case):
    check_layout(fake_ops.nchw_to_tokens, fake_ops.tokens_to_nchw, case, CPU)


@pytest.mark.parametrize("case", IM2COL_S2_CASES)
def test_im2col_s2_twin(case):
    check_im2col_s2(fake_ops.im2col_s2, case, CPU)


@pytest.mark.parametrize("case", UPSAMPLE_CASES)
def test_upsample2x_twin(case):
    check_upsample2x(fake_ops.upsample2x, case, CPU)


@pytest.mark.parametrize("batch,seq,heads", D80_CASES[:-1])
def test_attention_d80_twin(batch, seq, heads):
    """The table without its production case (25 images x 16 heads, run on the GPU only: its fp64 scores are 200 MB)."""
    check_d80(clip_fake_ops.attention_d80, batch, seq, heads, CPU, name="d80 twin")


def test_attention_d80_twin_identical_keys_and_large_logits():
    check_d80(clip_fake_ops.attention_d80, 2, 129, 2, CPU, identical_keys=True, name="d80 twin identical keys")
    check_d80(clip_fake_ops.attention_d80, 2, 257, 2, CPU, qk_scale=D80_LARGE_QK, name="d80 twin large logits")


def test_every_kernel_has_a_conformance_test():
    """Every __global__ kernel of vista_b200/csrc/ is held by a conformance test (KERNEL_TESTS) or left out with a reason
    (NOT_HELD); no entry names a kernel that no longer exists or a test function that does not exist."""
    kernels = source_kernels()
    assert len(kernels) >= 30, sorted(kernels)
    held, out = set(KERNEL_TESTS), set(NOT_HELD)
    assert not held & out, sorted(held & out)
    assert not kernels - held - out, f"kernels without a conformance test: {sorted(kernels - held - out)}"
    assert not (held | out) - kernels, f"stale entries: {sorted((held | out) - kernels)}"
    assert LAUNCHED_NOT_HELD <= out
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    for k, ids in KERNEL_TESTS.items():
        assert ids, k
        for tid in ids:
            f, fn = tid.split("::")
            path = os.path.join(tests_dir, f)
            assert os.path.isfile(path), f"{k}: {f} does not exist"
            assert fn in _test_functions(path), f"{k}: {tid} does not exist"
