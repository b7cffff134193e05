"""The layer-level harness of tests/block_shadow.py without a GPU: the tiny and small UNet, the tiny decoder and the tiny
encoder run on the operator twins of tests/fake_ops.py under the harness, and every layer, segment, conditioning
vector and hand-off passes with complete coverage.  Then composition defects are planted, each by recompiling one
runtime method with one argument or one routing changed (never a twin or a kernel): each run must fail naming the
layer (for a hand-off, the producer and the consumer), at three times the bound or more.  For each defect the figure
of the existing whole-network golden comparison on the same run is printed beside it."""
import inspect
import textwrap

import numpy as np
import pytest
import torch

import block_shadow
from fake_ops import patched_ops
from helpers import decoder_weights, golden, rel_l2, to_t, unet_inputs, unet_weights
from vista_b200 import ops, spec, synth
from vista_b200 import unet as unet_mod
from vista_b200 import vae as vae_mod

GOLDEN_BOUND = 5e-3        # the whole-network comparisons' rel-L2 bound (test_executor_cpu.py, test_unet_gpu.py)


@pytest.fixture(autouse=True)
def eager(monkeypatch):
    from vista_b200 import fused
    monkeypatch.setattr(fused, "USE_GRAPH", False)


# ==================================================================================================================
# The three networks on the twins
# ==================================================================================================================
def run_unet(preset="tiny", h=8, w=16, T=25, sigma=5.0, vector_delta=0.0):
    """One CFG forward (B = 2T) with the inputs of the unet_tiny golden; ``vector_delta`` shifts the unconditional
    clip's vector so that the two clips' embeddings differ.  Returns (harness, net output NCHW)."""
    cfg, sd = unet_weights(preset)
    sdt = to_t(sd)
    x, cc, mask2 = unet_inputs(7, cfg, h, w, T)
    vec = torch.from_numpy(cc["vector"]).clone()
    vec[:T] += vector_delta
    B = 2 * T
    with patched_ops(), torch.no_grad(), block_shadow.BlockShadow(unet=(cfg, sdt)) as bs:
        rt = unet_mod.UNetRuntime(cfg, sdt, "cpu", num_frames=T)
        c_in = 1.0 / np.sqrt(sigma * sigma + 1.0)
        xin = torch.from_numpy(np.concatenate([x * np.float32(c_in), cc["concat"]], 1))
        tok = unet_mod.padded_input_rows(B * h * w, "cpu")
        ops.nchw_to_tokens(xin.contiguous(), tok, B, 8, h, w)
        rt.set_conditioning(torch.from_numpy(cc["crossattn"]), vec)
        c_noise = torch.full((B,), 0.25 * float(np.log(sigma)))
        out = rt.forward(tok, c_noise, torch.from_numpy(mask2), h, w)
        res = torch.empty(B, cfg.out_channels, h, w)
        ops.tokens_to_nchw(out, res, B, cfg.out_channels, h, w)
    return bs, res


def run_decoder():
    """decode_first_stage of 25 latents (two 14-frame chunks), the decode_first_stage_tiny golden's inputs."""
    cfg, sd = decoder_weights("tiny")
    sdt = to_t(sd)
    z = torch.from_numpy(synth.normal(9, "decfs.z", (25, cfg.z_channels, 8, 16), std=0.18215))
    with patched_ops(), torch.no_grad(), block_shadow.BlockShadow(decoder=(cfg, sdt)) as bs:
        rt = vae_mod.DecoderRuntime(cfg, sdt, "cpu")
        out = vae_mod.decode_first_stage(rt, z)
    return bs, out


def run_encoder():
    """The conditioning encode of the cond_embedder_tiny golden: three frames through the tiny encoder with its
    quant_conv folded into conv_out (one forward per frame)."""
    from oracle.make_golden import cond_embedder_inputs
    cfg = spec.encoder_preset("tiny")
    sd = to_t(synth.synth_state_dict(spec.encoder_param_specs(cfg), seed=3))
    x, qw, qb = cond_embedder_inputs(cfg, 32, 64, 3)
    post = (torch.from_numpy(qw).flatten(1), torch.from_numpy(qb))
    x = torch.from_numpy(x)
    n, cin, H, W = x.shape
    with patched_ops(), torch.no_grad(), block_shadow.BlockShadow(encoder=(cfg, sd, post)) as bs:
        rt = vae_mod.EncoderRuntime(cfg, sd, "cpu", post=post)
        mom = torch.empty(n, 8, H // 2, W // 2)
        tok = rt.buf("e.x", H * W, 8)
        for i in range(n):
            tok.zero_()
            ops.nchw_to_tokens(x[i:i + 1].float().contiguous(), tok, 1, cin, H, W)
            ops.tokens_to_nchw(rt.forward(tok, 1, H, W), mom[i:i + 1], 1, 8, H // 2, W // 2)
    return bs, mom[:, :cfg.z_channels]


def unet_golden(res):
    return rel_l2(res, torch.from_numpy(golden("unet_tiny")["raw"]))


def decoder_golden(out):
    return rel_l2(out, torch.from_numpy(golden("decode_first_stage_tiny")["out"]))


def encoder_golden(mean):
    """cond_embedder_tiny holds mean * scale_factor (0.5) of the three frames, n_copies = 2 repeats."""
    ref = torch.from_numpy(golden("cond_embedder_tiny")["out"])
    return rel_l2((mean * 0.5).repeat_interleave(2, dim=0).reshape(ref.shape), ref)


def test_tiny_unet_every_layer_passes():
    bs, res = run_unet()
    print("\n" + bs.report())
    bs.assert_ok()
    assert unet_golden(res) < GOLDEN_BOUND
    assert bs.checked["unet"] >= set(block_shadow.unet_graph(unet_mod.build_unet_plan(spec.unet_preset("tiny"))))


def test_small_unet_every_layer_passes():
    """The vista topology (four levels, two ResBlocks per level, skips from three blocks per level) at 64 channels."""
    bs, _ = run_unet("small", 16, 32, T=5)
    print("\n" + bs.report())
    bs.assert_ok()


def test_tiny_decoder_every_layer_passes():
    bs, out = run_decoder()
    print("\n" + bs.report())
    bs.assert_ok()
    assert decoder_golden(out) < GOLDEN_BOUND
    assert bs.n_forward["dec"] == 2


def test_tiny_encoder_every_layer_passes():
    bs, mean = run_encoder()
    print("\n" + bs.report())
    bs.assert_ok()
    assert encoder_golden(mean) < GOLDEN_BOUND


def test_decoder_reference_pieces_equal_the_oracle():
    """The decoder's fp64 reference in pieces (per frame, row bands, clip statistics merged band by band) is the oracle's
    dec_video_res_block / up-convolution / head to fp64 re-association, with bands of 3 rows over 8 (a short last band)."""
    import torch.nn.functional as F
    from oracle import vista_oracle as vo
    cfg, sd = decoder_weights("tiny")
    sd = {k: v.double() for k, v in to_t(sd).items()}
    T, H, W = 5, 8, 16
    rb = next(b for b in vae_mod.build_decoder_plan(cfg).levels[-1][0] if b.has_skip)
    x = torch.randn(T, rb.cin, H, W, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    want = vo.dec_video_res_block(sd, rb.prefix, x, True, T)
    got = torch.zeros_like(want)

    def sink(ref, r0):
        got[:, :, r0:r0 + ref.shape[2]] = ref
    block_shadow.dec_video_res_block_pieces(sd, rb.prefix, lambda f: x[f:f + 1], T, True, sink,
                                            band_bytes=3 * rb.cout * T * W * 8)
    assert float((got - want).abs().max() / want.abs().max()) < 1e-12

    up = vae_mod.build_decoder_plan(cfg).levels[0][1]
    xu = torch.randn(T, cfg.ch * cfg.ch_mult[-1], H, W, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    want = F.conv2d(F.interpolate(xu, scale_factor=2, mode="nearest"), sd[f"{up}.weight"], sd[f"{up}.bias"], padding=1)
    got = torch.zeros_like(want)
    block_shadow.upconv_pieces(sd[f"{up}.weight"], sd[f"{up}.bias"], lambda f: xu[f:f + 1], T,
                               lambda ref, f: got.__setitem__(slice(f, f + 1), ref))
    assert float((got - want).abs().max() / want.abs().max()) < 1e-12

    xh = torch.randn(T, cfg.ch, H, W, dtype=torch.float64, generator=torch.Generator().manual_seed(7))
    y = F.conv2d(vo._swish(vo._gn(sd, "norm_out", xh, 1e-6)), sd["conv_out.weight"], sd["conv_out.bias"], padding=1)
    want = F.conv3d(y.permute(1, 0, 2, 3)[None], sd["conv_out.time_mix_conv.weight"], sd["conv_out.time_mix_conv.bias"],
                    padding=(1, 0, 0))[0].permute(1, 0, 2, 3)
    got = block_shadow.decoder_head_pieces(sd, lambda f: xh[f:f + 1], T)
    assert float((got - want).abs().max() / want.abs().max()) < 1e-12


# ==================================================================================================================
# Planted composition defects
# ==================================================================================================================
def recompiled(fn, old, new):
    """``fn`` (a runtime method or function) recompiled from its source with the one occurrence of ``old`` replaced by
    ``new``, in its own module's globals."""
    src = textwrap.dedent(inspect.getsource(fn))
    assert src.count(old) == 1, (fn.__qualname__, old)
    ns = {}
    exec(compile(src.replace(old, new), inspect.getsourcefile(fn), "exec"), fn.__globals__, ns)
    return ns[fn.__name__]


def plant(monkeypatch, cls, name, old, new):
    monkeypatch.setattr(cls, name, recompiled(getattr(cls, name), old, new))


def expect_failure(bs, figure, what, names):
    """The run failed naming one of ``names`` (a layer prefix, or the producer and the consumer of a hand-off), at 3x
    the bound or more for a layer; prints the harness's message and the golden comparison's figure."""
    print(f"\n{what}: golden rel-L2 {figure}")
    for msg in bs.failures.values():
        print("   ", msg.splitlines()[0])
    with pytest.raises(AssertionError):
        bs.assert_ok()
    hits = [m for m in bs.failures.values() if any(n in m for n in names)]
    assert hits, f"{what}: no failure names {names}: {list(bs.failures.values())}"
    layer = [bs.census[k[1]].ratio for k in bs.failures if k[0] == "layer" and any(n in k[1] for n in names)]
    if layer:
        assert max(layer) >= 3.0, f"{what}: fails at only {max(layer):.2f} x the bound"
    return hits


def _fmt(r):
    return f"{r:.2e} ({'passes' if r < GOLDEN_BOUND else 'fails'} the {GOLDEN_BOUND} bound)"


def test_planted_temporal_groupnorm_per_frame(monkeypatch):
    """1. The temporal GroupNorm of the ResBlocks with frames_per_stat 1 instead of T."""
    plant(monkeypatch, unet_mod.UNetRuntime, "_resblock", "gi + 2, fps=T, part=p2)", "gi + 2, fps=1, part=p2)")
    bs, res = run_unet()
    expect_failure(bs, _fmt(unet_golden(res)), "temporal GroupNorm per frame", ["input_blocks.1.0"])


def test_planted_resblock_alpha_swapped(monkeypatch):
    """2. The ResBlock time mixer's alpha and 1 - alpha swapped."""
    plant(monkeypatch, unet_mod.UNetRuntime, "_resblock", 's_acc=1.0 - L["alpha"]', 's_acc=L["alpha"]')
    bs, res = run_unet()
    expect_failure(bs, _fmt(unet_golden(res)), "alpha / 1 - alpha swapped", ["input_blocks.1.0"])


def test_planted_next_frame_position(monkeypatch):
    """3. The temporal block of the transformers adds the positional embedding of the next frame."""
    plant(monkeypatch, unet_mod.UNetRuntime, "_svt", 'pos = self.cond["pos"][p]', 'pos = self.cond["pos"][p].roll(-1, 0)')
    bs, res = run_unet()
    expect_failure(bs, _fmt(unet_golden(res)), "next frame's position", ["input_blocks.1.1"])


def test_planted_unconditional_time_context_for_both_clips(monkeypatch):
    """4. The unconditional clip's cond["tm"] row applied to both CFG clips."""
    plant(monkeypatch, unet_mod.UNetRuntime, "_svt", 'rv_div=T * hw, rv_mod=nb)', 'rv_div=T * hw, rv_mod=1)')
    bs, res = run_unet()
    expect_failure(bs, _fmt(unet_golden(res)), "uc time context for both clips", ["input_blocks.1.1"])


def test_planted_emb_rows_modulo_frames(monkeypatch):
    """5. One ResBlock's emb_out rows taken modulo T instead of B: the second clip reads the first clip's embedding.
    The golden's two clips share one vector (its embeddings are equal, the defect is invisible there), so this run gives
    the unconditional clip its own vector."""
    clean = run_unet(vector_delta=0.5)[1]
    plant(monkeypatch, unet_mod.UNetRuntime, "_resblock", 'L["emb_off"] + rb.cout], rv_div=hw, rv_mod=B',
          'L["emb_off"] + rb.cout], rv_div=hw, rv_mod=(T if rb.prefix == "output_blocks.0.0" else B)')
    bs, res = run_unet(vector_delta=0.5)
    expect_failure(bs, f"n/a on the golden's inputs; {rel_l2(res, clean):.2e} against the same run without the defect",
                   "emb_out rows modulo T", ["output_blocks.0.0"])


def test_planted_skip_from_wrong_input_block(monkeypatch):
    """6. Output blocks 2 and 3 read their skips from each other's input block (input blocks 0 and 1, one level)."""
    plant(monkeypatch, unet_mod.UNetRuntime, "forward", "j = n_out - 1 - i\n", "j = n_out - 1 - {0: 1, 1: 0}.get(i, i)\n")
    bs, res = run_unet()
    expect_failure(bs, _fmt(unet_golden(res)), "skip from the wrong input block",
                   ["input_blocks.1.1 -> output_blocks.2.0", "input_blocks.0.0 -> output_blocks.3.0"])


def test_planted_stale_skip_partials(monkeypatch):
    """7. The skip producers fill a copy of their GroupNorm partials: the concat buffer's skip half keeps stale ones
    while it is marked filled."""
    plant(monkeypatch, unet_mod.UNetRuntime, "forward", "cat_bufs[j][:, ch_in_h[j]:], hh, ww, xp=cur_p, dp=dp)",
          "cat_bufs[j][:, ch_in_h[j]:], hh, ww, xp=cur_p, dp=None if dp is None else dp.clone())")
    bs, res = run_unet()
    # the fused statistics run at 8 x 16 only: the stale halves are the skips of output blocks 3 (from input block 0)
    # and 2 (from input block 1), and input block 1 reads input block 0's partials through the same stale view
    consumers = ["output_blocks.2.0", "output_blocks.3.0", "input_blocks.1.0"]
    expect_failure(bs, _fmt(unet_golden(res)), "stale skip partials", consumers)
    failing = {k[1] for k in bs.failures if k[0] == "layer"}
    assert failing == set(consumers), failing


def test_planted_decoder_temporal_blend(monkeypatch):
    """8. The decoder's temporal conv blended with 1 - alpha instead of alpha."""
    plant(monkeypatch, vae_mod.DecoderRuntime, "_resblock", 's_acc=L["alpha"]', 's_acc=1.0 - L["alpha"]')
    bs, out = run_decoder()
    expect_failure(bs, _fmt(decoder_golden(out)), "decoder 1 - alpha", ["dec:mid.block_1", "dec:up."])


def test_planted_decoder_attention_without_v_bias(monkeypatch):
    """9. The decoder attention's V bias dropped."""
    plant(monkeypatch, vae_mod.DecoderRuntime, "_attn", 'bias=A["v_b"])', "bias=None)")
    bs, out = run_decoder()
    expect_failure(bs, _fmt(decoder_golden(out)), "attention V bias dropped", ["dec:mid.attn_1"])


def test_planted_decoder_arena_roles_share_bytes(monkeypatch):
    """10. Two arena roles that are live together share bytes: the attention's q over the ResBlock output it still
    has to add back."""
    real = vae_mod.decoder_scratch_plan

    def plan(cfg, T, h, w):
        p = real(cfg, T, h, w)
        roles = dict(p.roles)
        roles["d.q"] = (roles["d.r0"][0], roles["d.q"][1])
        return p._replace(roles=roles)
    monkeypatch.setattr(vae_mod, "decoder_scratch_plan", plan)
    bs, out = run_decoder()
    expect_failure(bs, _fmt(decoder_golden(out)), "d.q over d.r0", ["dec:mid.attn_1"])


def test_planted_encoder_symmetric_downsample(monkeypatch):
    """11. The encoder's Downsample gathered with im2col_s2 (padding 1 on every side) instead of im2col_s2_asym."""
    plant(monkeypatch, vae_mod.EncoderRuntime, "forward", "ops.im2col_s2_asym(x,", "ops.im2col_s2(x,")
    bs, mean = run_encoder()
    expect_failure(bs, _fmt(encoder_golden(mean)), "symmetric Downsample", ["enc:down.0.downsample.conv"])


def test_planted_quant_conv_not_folded(monkeypatch):
    """12. quant_conv not folded into the encoder's conv_out."""
    plant(monkeypatch, vae_mod.EncoderRuntime, "_pack", 'if getattr(self, "_post", None) is not None:', "if False:")
    bs, mean = run_encoder()
    expect_failure(bs, _fmt(encoder_golden(mean)), "quant_conv not folded", ["enc:out"])
