"""The decoder's planned scratch (vae.decoder_scratch_plan) and the upsampling tap-GEMM mode, without a GPU: the plan's
size at the production chunk, that no two views live at the same op share bytes, that the runtime takes exactly the views
the plan lists, and that the decoder on the emulated operators (tests/fake_ops.py, plus the upsampling mode emulated
here) still matches the reference's fixtures."""
import contextlib

import pytest
import torch

from fake_ops import patched_ops
from helpers import decoder_weights, golden, golden_rel, to_t
from vista_b200 import ops, spec, synth, vae

GIB = 2 ** 30


def _nbytes(shape, dtype):
    n = dtype.itemsize
    for s in shape:
        n *= s
    return n


def test_vista_chunk_scratch_fits_budget():
    """One 14-frame chunk of 72 x 128 latents (576 x 1024 frames): at most 24 GiB of scratch.  One buffer per
    (role, shape), as before the plan, plus the materialised 2x upsample, would take about 45 GiB."""
    cfg = spec.decoder_preset("vista")
    plan = vae.decoder_scratch_plan(cfg, 14, 72, 128)
    per_shape = {(r, s, d): _nbytes(s, d) for r, s, d, _, _ in plan.uses}
    print(f"planned {plan.total / GIB:.2f} GiB; one buffer per role and shape {sum(per_shape.values()) / GIB:.2f} GiB")
    assert plan.total <= 24 * GIB
    assert "d.up" not in plan.roles


@pytest.mark.parametrize("preset,T,h,w", [("vista", 14, 72, 128), ("vista", 5, 72, 128), ("vista", 14, 16, 32),
                                          ("tiny", 14, 8, 16), ("small", 3, 8, 16), ("vista", 11, 9, 12)])
def test_scratch_views_fit_and_live_views_are_disjoint(preset, T, h, w):
    plan = vae.decoder_scratch_plan(spec.decoder_preset(preset), T, h, w)
    spans = []
    for role, shape, dtype, first, last in plan.uses:
        off, size = plan.roles[role]
        n = _nbytes(shape, dtype)
        assert n <= size and off % 4096 == 0 and off + size <= plan.total, (role, shape)
        assert first <= last
        spans.append((first, last, off, off + n, role))
    for i, (f1, l1, b1, e1, r1) in enumerate(spans):
        for f2, l2, b2, e2, r2 in spans[i + 1:]:
            if f1 <= l2 and f2 <= l1:
                assert e1 <= b2 or e2 <= b1, f"{r1} [{f1},{l1}] and {r2} [{f2},{l2}] overlap in bytes"


@pytest.mark.parametrize("preset,T,h,w", [("tiny", 14, 8, 16), ("small", 3, 8, 16)])
def test_runtime_takes_exactly_the_planned_views(preset, T, h, w, monkeypatch):
    """Every view DecoderRuntime.forward takes is one the plan lists (role, shape, dtype), and every listed one is taken:
    the plan and the executor cannot drift apart."""
    cfg, sd = decoder_weights(preset)
    plan = vae.decoder_scratch_plan(cfg, T, h, w)
    taken = set()
    scratch = vae.DecoderRuntime._scratch

    def record(self, role, shape, dtype):
        taken.add((role, tuple(shape), dtype))
        return scratch(self, role, shape, dtype)
    monkeypatch.setattr(vae.DecoderRuntime, "_scratch", record)
    with patched_ops(), torch.no_grad():
        rt = vae.DecoderRuntime(cfg, to_t(sd), "cpu")
        z = torch.from_numpy(synth.normal(9, "dec.z", (T, cfg.z_channels, h, w), std=1.0))
        tok = rt.buf("d.z", T * h * w, 8)
        tok.zero_()
        ops.nchw_to_tokens(z, tok, T, cfg.z_channels, h, w)
        up = 2 ** (len(cfg.ch_mult) - 1)
        rt.forward(tok, T, h, w, torch.empty(T, cfg.out_ch, up * h, up * w))
    assert taken == {(r, s, d) for r, s, d, _, _ in plan.uses}
    assert rt._arena.numel() == plan.total


@contextlib.contextmanager
def upsampling_ops():
    """tests/fake_ops.py's emulation plus the tap-GEMM's upsampling mode (``gemm(..., upsample=True)``): the nearest-2x
    upsample of the low-resolution operand, then the emulated image-tap GEMM over NB x 2H x 2W."""
    with patched_ops():
        fake = ops.gemm

        def gemm(a, w, out, *, upsample=False, geom=None, **kw):
            if not upsample:
                return fake(a, w, out, geom=geom, **kw)
            W, H, NB = geom
            assert kw.get("act", 0) == 0 and kw.get("s_acc", 1.0) == 1.0 and not kw.get("h_pad", 0)
            assert all(kw.get(k) is None for k in ("rowvec", "res1", "res2"))
            up = ops.upsample2x(a, torch.empty(4 * a.shape[0], a.shape[1], dtype=a.dtype), NB, H, W, a.shape[1])
            return fake(up, w, out, geom=(2 * W, 2 * H, NB), **kw)
        ops.gemm = gemm
        try:
            yield
        finally:
            ops.gemm = fake


def _decode_emulated(cfg, sd, upsample_in_gemm, monkeypatch):
    monkeypatch.setattr(vae.DecoderRuntime, "_upsample_in_gemm", lambda self: upsample_in_gemm)
    z = torch.from_numpy(synth.normal(9, "dec.z", (14, cfg.z_channels, 8, 16), std=1.0))
    with upsampling_ops(), torch.no_grad():
        dec = vae.DecoderRuntime(cfg, to_t(sd), "cpu")
        tok = dec.buf("d.z", 14 * 8 * 16, 8)
        tok.zero_()
        ops.nchw_to_tokens(z, tok, 14, cfg.z_channels, 8, 16)
        up = 2 ** (len(cfg.ch_mult) - 1)
        return dec.forward(tok, 14, 8, 16, torch.empty(14, cfg.out_ch, 8 * up, 16 * up))


@pytest.mark.parametrize("name,preset", [("decoder_tiny", "tiny"), ("decoder_small", "small")])
def test_planned_decoder_on_emulated_ops_matches_reference(name, preset, monkeypatch):
    """The decoder forward on the planned scratch, with its up-convolutions in the upsampling mode (as on CUDA), on the
    emulated operators against the REAL reference's fp32 outputs at the GPU tolerance; and equal to the same forward
    with the upsample materialised (the path a runtime on the CPU emulation takes)."""
    cfg, sd = decoder_weights(preset)
    out = _decode_emulated(cfg, sd, True, monkeypatch)
    r = golden_rel(out, golden(name))
    assert max(r) < 5e-3, r
    assert torch.equal(out, _decode_emulated(cfg, sd, False, monkeypatch))


def test_arena_grows_only_for_a_larger_geometry():
    cfg, sd = decoder_weights("tiny")
    with patched_ops(), torch.no_grad():
        rt = vae.DecoderRuntime(cfg, to_t(sd), "cpu")
        z = torch.from_numpy(synth.normal(9, "decfs.z", (25, cfg.z_channels, 8, 16), std=0.18215))
        vae.decode_first_stage(rt, z)                 # chunks of 14 and 14 frames
        big = rt._arena
        vae.decode_first_stage(rt, z[:6])             # one chunk of 6 frames: fits the arena of 14
        assert rt._arena is big
    assert big.numel() == vae.decoder_scratch_plan(cfg, 14, 8, 16).total
    assert rt._roles is None                          # views are handed out only while forward runs


@pytest.mark.parametrize("W,H,box", [(128, 72, (128, 1, 1)), (32, 16, (32, 4, 1)), (12, 9, None), (64, 3, None)])
def test_upsample_stats_box(W, H, box):
    assert ops.upsample_stats_box(W, H) == box
