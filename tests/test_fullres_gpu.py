"""Full-resolution rollout on one 80 GB H100: the upsampling tap-GEMM mode (a_mode 2) against upsample2x + the image-tap
convolution, the decoder on its planned scratch, and the native-YAML engine at 576 x 1024 (ViT-H/14, the vista encoder,
UNet and decoder, seeded synthetic weights) running a 2-round session within a memory budget."""
import ctypes
import importlib.util
import os

import pytest
import torch

from helpers import decoder_weights, rel_l2, to_t
from vista_b200 import lib, ops, spec, synth, vae

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GIB = 2 ** 30
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _conv_inputs(W, H, T, C, N, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(T * H * W, C, generator=g).to(DEV, torch.float16)
    w = (torch.randn(N, 9 * C, generator=g) / (9 * C) ** 0.5).to(DEV, torch.float16)
    b = torch.randn(N, generator=g).to(DEV)
    return x, w, b


def _two_launch(x, w, b, W, H, T, stats):
    """The decoder's up-convolution before the upsampling mode: upsample2x, then the image-tap convolution."""
    C, N = x.shape[1], w.shape[0]
    up = ops.upsample2x(x, torch.empty(4 * x.shape[0], C, dtype=x.dtype, device=DEV), T, H, W, C)
    out = torch.empty(4 * x.shape[0], N, dtype=torch.float16, device=DEV)
    return ops.gemm(up, w, out, bias=b, taps=ops.TAPS_3X3, geom=(2 * W, 2 * H, T), stats=stats)


def _partials(tokens, N):
    return torch.full((-(-tokens // 128) * 4, N, 2), float("nan"), dtype=torch.float32, device=DEV)


# the decoder's three transitions at 576 x 1024 (14-frame chunk), a small odd frame count, and widths below 128
@pytest.mark.parametrize("W,H,T,C,N", [(128, 72, 14, 512, 512), (256, 144, 14, 512, 512), (512, 288, 14, 256, 256),
                                       (128, 3, 5, 64, 96), (32, 16, 3, 128, 128), (16, 8, 7, 64, 64)])
def test_upsample_conv_equals_upsample_then_conv(W, H, T, C, N):
    x, w, b = _conv_inputs(W, H, T, C, N, seed=W + H + T)
    M = 4 * T * H * W
    want = _two_launch(x, w, b, W, H, T, None)
    got = ops.gemm(x, w, torch.empty(M, N, dtype=torch.float16, device=DEV), bias=b, taps=ops.TAPS_3X3,
                   geom=(W, H, T), upsample=True)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    if ops.upsample_stats_box(W, H) is None or ops.stats_box(2 * W, 2 * H, T) is None:
        return
    # with fused statistics: the same output; per-frame column sums equal up to the fp32 summation order
    pw, pg = _partials(M, N), _partials(M, N)
    want = _two_launch(x, w, b, W, H, T, pw)
    got = ops.gemm(x, w, torch.empty(M, N, dtype=torch.float16, device=DEV), bias=b, taps=ops.TAPS_3X3,
                   geom=(W, H, T), upsample=True, stats=pg)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert not torch.isnan(pg).any()
    fw, fg = (p.double().reshape(T, -1, N, 2).sum(1) for p in (pw, pg))
    scale = got.double().abs().reshape(T, -1, N).sum(1)
    assert ((fw[..., 0] - fg[..., 0]).abs() <= 1e-5 * scale + 1e-3).all()
    assert ((fw[..., 1] - fg[..., 1]).abs() <= 1e-5 * fw[..., 1].abs() + 1e-3).all()
    sw, sg = (torch.empty(T, 32, 2, device=DEV) for _ in range(2))
    ops.groupnorm_from_partials(pw, T, 4 * H * W, N, 1e-6, sw)
    ops.groupnorm_from_partials(pg, T, 4 * H * W, N, 1e-6, sg)
    torch.cuda.synchronize()
    torch.testing.assert_close(sg, sw, rtol=1e-5, atol=1e-6)


def test_upsample_mode_rejects_other_epilogues():
    W, H, T, C, N = 128, 2, 2, 64, 64
    x, w, b = _conv_inputs(W, H, T, C, N, seed=1)
    M = 4 * T * H * W
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    res = torch.zeros(M, N, dtype=torch.float16, device=DEV)
    for kw in (dict(res1=res), dict(act=1), dict(s_acc=0.5), dict(rowvec=torch.zeros(1, N, device=DEV))):
        with pytest.raises(RuntimeError, match="upsampling mode"):
            ops.gemm(x, w, out, bias=b, taps=ops.TAPS_3X3, geom=(W, H, T), upsample=True, **kw)
    with pytest.raises(RuntimeError, match="upsampling mode"):
        ops.gemm(x, w, torch.empty(M, N, dtype=torch.float32, device=DEV), taps=ops.TAPS_3X3, geom=(W, H, T),
                 upsample=True)
    # statistics need boxes that tile every frame: the launcher refuses a box that does not
    d = lib.GemmDesc()
    d.a, d.lda, d.tokens, d.a_mode = x.data_ptr(), C, T * H * W, 2
    d.W, d.H, d.NB, d.box_w, d.box_h, d.box_b = W, H, T, 32, 4, 1
    d.cin, d.ntaps = C, 9
    for i, (dh, dw) in enumerate(ops.TAPS_3X3):
        d.dh[i], d.dw[i] = dh, dw
    d.b, d.N, d.tile_n, d.out, d.ldo, d.s_acc = w.data_ptr(), N, 64, out.data_ptr(), N, 1.0
    p = _partials(M, N)
    d.stats, d.stats_ld = p.data_ptr(), N
    with pytest.raises(RuntimeError, match="tile each frame"):
        lib.check(lib.load().b200v_gemm(ctypes.byref(d), torch.cuda.current_stream().cuda_stream), "b200v_gemm")
    torch.cuda.synchronize()


def _parent_upconv(monkeypatch):
    """Makes DecoderRuntime's up-convolutions run as before the upsampling mode: upsample2x into a full-resolution
    tensor, then the image-tap convolution with its statistics over 128 consecutive tokens."""
    gemm = vae.DecoderRuntime.gemm

    def two_launch(self, a, lin, out, upsample=False, geom=None, stats=None, **kw):
        if not upsample:
            return gemm(self, a, lin, out, geom=geom, stats=stats, **kw)
        W, H, T = geom
        up = ops.upsample2x(a, torch.empty(4 * a.shape[0], a.shape[1], dtype=a.dtype, device=a.device), T, H, W, a.shape[1])
        return gemm(self, up, lin, out, geom=(2 * W, 2 * H, T), stats=stats, **kw)
    monkeypatch.setattr(vae.DecoderRuntime, "gemm", two_launch)


def test_decoder_fullres_chunk_against_two_launch_path_and_peak(monkeypatch):
    cfg, sd = decoder_weights("vista")
    T, h, w = 14, 72, 128
    gemm_new = vae.DecoderRuntime.gemm
    rt = vae.DecoderRuntime(cfg, to_t(sd, DEV), DEV)
    z = torch.from_numpy(synth.normal(9, "fullres.z", (T, cfg.z_channels, h, w), std=1.0 / 0.18215)).to(DEV)
    tok = rt.buf("d.z", T * h * w, 8)
    tok.zero_()
    ops.nchw_to_tokens(z, tok, T, cfg.z_channels, h, w)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    out = torch.empty(T, cfg.out_ch, 8 * h, 8 * w, device=DEV)
    rt.forward(tok, T, h, w, out)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    plan = vae.decoder_scratch_plan(cfg, T, h, w)
    small = 64 * 2 ** 20        # GroupNorm statistics and workspace (a few MB at this size)
    print(f"decoder chunk {T} x {8 * h} x {8 * w}: peak {peak / GIB:.2f} GiB, planned scratch {plan.total / GIB:.2f} GiB, "
          f"output {out.numel() * 4 / GIB:.2f} GiB")
    assert peak <= plan.total + out.numel() * 4 + small
    _parent_upconv(monkeypatch)
    ref = torch.empty_like(out)
    rt.forward(tok, T, h, w, ref)
    torch.cuda.synchronize()
    d, r = float((out - ref).abs().max()), rel_l2(out, ref)
    # only the fp32 order of the up-convolutions' statistics partials differs; the last-bit changes of mean / rstd flip
    # fp16 roundings that some 40 further layers carry on (1.1e-3 rel-L2 measured): well inside the 5e-3 fp16 bound
    print(f"decoder chunk vs the two-launch up-convolution: max abs diff {d:.3e}, rel-L2 {r:.3e}")
    assert torch.isfinite(out).all() and r < 2.5e-3, (d, r)
    # with the statistics of the up-convolutions' outputs taken by their own pass, both paths are bit-identical
    monkeypatch.setattr(ops, "upsample_stats_box", lambda W, H: None)
    monkeypatch.setattr(vae.DecoderRuntime, "gemm", gemm_new)
    rt.forward(tok, T, h, w, out)
    _parent_upconv(monkeypatch)
    rt.forward(tok, T, h, w, ref)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def _bench_session():
    spec_ = importlib.util.spec_from_file_location("bench_session", os.path.join(ROOT, "tools", "bench_session.py"))
    mod = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(mod)
    return mod


def test_native_engine_session_at_576x1024_fits_and_equals_rollout():
    """The native YAML engine at Vista's resolution, 2 rounds of 2 steps: RolloutSession bytes equal engine.rollout's,
    two seeded runs are bit-identical, and the peak allocation stays within 72 GiB."""
    from oracle.make_golden_clip import clip_frames
    from vista_b200.rollout import conditioner_recondition
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    eng.sampler.num_steps = 2
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)        # the run's peak, with the weights and executors resident
    T, H, W, rounds = eng.num_frames, 576, 1024, 2
    frame = torch.from_numpy(clip_frames(12, "fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame,
          "trajectory": bs.TRAJECTORY}
    z = torch.from_numpy(synth.normal(7, "fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)

    def session():
        torch.manual_seed(5)
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
        frames = torch.cat([sess.step(None) for _ in range(rounds)] + [sess.close()])
        return frames, sess.samples_z.clone()

    f1, z1 = session()
    f2, z2 = session()
    c, uc = eng.condition(vd, T, bs.UC_KEYS)
    torch.manual_seed(5)
    fb, zb = eng.rollout(c, uc, z, rounds, recondition=conditioner_recondition(eng, vd, bs.UC_KEYS), u8=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV)
    print(f"576 x 1024 session, {rounds} rounds: peak allocated {peak / GIB:.2f} GiB")
    assert f1.shape == (rounds * (T - 3) + 3, H, W, 3)
    assert torch.equal(f1, f2) and torch.equal(z1, z2)
    assert torch.equal(f1, fb) and torch.equal(z1, zb)
    assert peak <= 72 * GIB
