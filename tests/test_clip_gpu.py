"""The conditioner's CLIP image branch on the H100: the head-width-80 attention, the erf-GELU GEMM epilogue and the
preprocess kernel against torch / the CPU oracle, the native embedder against the reference fixtures, and engine.rollout
with CLIP re-conditioning between rounds against the same loop over the CPU oracle."""
import pytest
import torch
import torch.nn.functional as F

from helpers import golden, rel_l2, to_t
from oracle import clip_oracle as co
from oracle.make_golden_clip import CASES, clip_frames, clip_weights
from vista_b200 import spec, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as o
    lib.load()
    return o


@pytest.mark.parametrize("images", [1, 25])
@pytest.mark.parametrize("heads", [1, 16])
@pytest.mark.parametrize("seq", [1, 77, 257, 300])
def test_attention_d80_matches_sdpa(ops, seq, heads, images):
    torch.manual_seed(seq * 100 + heads * 10 + images)
    C = heads * 80
    qkv = (torch.randn(images * seq, 3 * C + 16, device=DEV) * 1.5).half()      # fused in-proj rows, padded stride
    out = torch.full((images * seq, C + 8), float("nan"), dtype=torch.float16, device=DEV)
    ops.attention_d80(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:3 * C], out[:, :C], images, seq, heads)
    torch.cuda.synchronize()
    sp = lambda t: t.float().reshape(images, seq, heads, 80).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sp(qkv[:, :C]), sp(qkv[:, C:2 * C]), sp(qkv[:, 2 * C:3 * C]))
    ref = ref.transpose(1, 2).reshape(images * seq, C)
    got = out[:, :C].float()
    assert torch.isfinite(got).all() and torch.isnan(out[:, C:].float()).all()     # nothing written past the heads
    assert rel_l2(got.cpu(), ref.cpu()) < 2e-3 and float((got - ref).abs().max()) < 2e-2


@pytest.mark.parametrize("tokens,N,K", [(771, 200, 320), (77, 1288, 64), (514, 5120, 1280)])
def test_gemm_gelu_epilogue(ops, tokens, N, K):
    torch.manual_seed(tokens + N)
    a = torch.randn(tokens, K, device=DEV).half()
    w = (torch.randn(N, K, device=DEV) / K ** 0.5 * 2).half()
    b = torch.randn(N, device=DEV) * 0.5
    out = torch.empty(tokens, N, dtype=torch.float16, device=DEV)
    ops.gemm(a, w, out, bias=b, act=3)
    torch.cuda.synchronize()
    ref = F.gelu(a.float() @ w.float().t() + b)
    assert float((out.float() - ref).abs().max()) < 2e-3 * max(1.0, float(ref.abs().max()))
    assert rel_l2(out.float().cpu(), ref.cpu()) < 1e-3


@pytest.mark.parametrize("H,W,aa", [(576, 1024, True), (576, 1024, False), (300, 500, True), (64, 128, True),
                                    (224, 224, True)])
def test_preprocess_matches_oracle(ops, H, W, aa):
    n = 2
    x = torch.from_numpy(clip_frames(5, f"pre{H}x{W}", n, H, W))
    want = co.preprocess(x, aa)
    rows32 = torch.full((n * 257, 640), float("nan"), device=DEV)
    ops.clip_preprocess(x.to(DEV), rows32, aa)
    rows16 = torch.full((n * 257, 640), float("nan"), dtype=torch.float16, device=DEV)
    ops.clip_preprocess(x.to(DEV), rows16, aa)
    torch.cuda.synchronize()
    r = rows32.cpu().reshape(n, 257, 640)
    assert torch.equal(r[:, 0], torch.zeros(n, 640)) and torch.equal(r[:, :, 588:], torch.zeros(n, 257, 52))
    got = r[:, 1:, :588].reshape(n, 16, 16, 3, 14, 14).permute(0, 3, 1, 4, 2, 5).reshape(n, 3, 224, 224)
    err = float((got - want).abs().max())
    print(f"preprocess {H}x{W} antialias={aa}: max abs error {err:.2e}")
    assert err <= 1e-5
    assert torch.equal(rows16, rows32.half())           # the fp16 rows are the fp32 values rounded once


def _embedder(cfg, sd, antialias=True, n_copies=1):
    from vista_b200.clip import FrozenOpenCLIPImagePredictionEmbedder
    emb = FrozenOpenCLIPImagePredictionEmbedder(
        {"target": "vista_b200.clip.FrozenOpenCLIPImageEmbedder", "params": {"arch": cfg, "antialias": antialias}},
        n_cond_frames=1, n_copies=n_copies)
    emb.load_state_dict({"open_clip.model.visual." + k: torch.from_numpy(v) for k, v in sd.items()})
    return emb.to(DEV)


@pytest.mark.parametrize("name", ["clip_tiny", "clip_vith_14"])
def test_embedder_matches_reference(ops, name):
    g = golden(name)
    preset, seed, frames = CASES[name]
    cfg, sd = clip_weights(preset, seed)
    assert str(g["weights_crc"]) == synth.state_dict_checksum(sd)
    for fname, n, H, W, aa in frames:
        x = torch.from_numpy(clip_frames(seed, fname, n, H, W))
        assert str(g[f"{fname}_frames_crc"]) == synth.checksum([x.numpy()])
        emb = _embedder(cfg, sd, aa)
        z = emb(x.to(DEV))
        z2 = emb(x.to(DEV)).clone()
        torch.cuda.synchronize()
        assert torch.equal(z, z2)                       # same input twice: bit-identical
        want = torch.from_numpy(g[f"{fname}_emb"])
        assert z.shape == want.shape and z.dtype == torch.float32
        r = rel_l2(z.cpu(), want)
        print(f"{name}/{fname} ({n} x {H}x{W}, antialias={aa}): rel-L2 vs reference {r:.3e}")
        assert r <= 5e-3


def test_rollout_with_clip_recondition_vs_oracle():
    from oracle import vista_oracle as vo
    from test_glue_gpu import _engine
    from vista_b200.rollout import clip_recondition
    T, h, w, steps, rounds = 25, 8, 16, 3, 3
    eng, (ucfg, usd), (dcfg, dsd) = _engine(steps)
    ccfg, csd = clip_weights("tiny", 11)
    emb = _embedder(ccfg, csd)
    c, uc = synth.synth_conditioning(7, T, h, w, trajectory=True, context_dim=ucfg.context_dim, adm=ucfg.adm_in_channels)
    _, z, _ = synth.synth_latents(7, T, h, w)
    zt = torch.from_numpy(z)
    noises = [torch.from_numpy(synth.normal(80 + i, "rollout.noise", (T, 4, h, w), std=1.0)) for i in range(rounds)]
    seen = []
    cb = clip_recondition(emb, to_t(c, DEV), to_t(uc, DEV), eng.scale_factor)

    def recording(n, sample, decode_tail):
        cc, uu = cb(n, sample, decode_tail)
        seen.append(cc["crossattn"].cpu().clone())
        return cc, uu
    _, samples_z = eng.rollout(to_t(c, DEV), to_t(uc, DEV), zt.to(DEV), rounds, noises=noises, recondition=recording,
                               decode=False)
    torch.cuda.synchronize()
    assert len(seen) == rounds - 1
    c1 = torch.from_numpy(c["crossattn"])
    assert not torch.equal(seen[0][..., :1024], c1[..., :1024])      # round 2 sees a new CLIP embedding
    assert torch.equal(seen[0][..., 1024:], c1[..., 1024:])          # the action slots are kept

    # the same loop over the CPU oracle (sample_utils.py:318-365 with the CLIP re-conditioning of :339-350)
    sdt, dsdt, csdt = to_t(usd), to_t(dsd), to_t(csd)
    fn = lambda nz, cc, cf, m: vo.euler_edm_sample(sdt, ucfg, nz, cc, to_t(uc), cf, m, steps, T)
    init_mask, pred_mask = torch.zeros(T), torch.zeros(T)
    init_mask[0] = 1
    pred_mask[[0, 1, 2]] = 1
    ref_z = torch.zeros_like(samples_z.cpu())
    cc = to_t(c)
    ref_cross = []
    with torch.no_grad():
        sample = fn(noises[0].clone(), cc, zt, init_mask)
        sample[0] = zt[0]
        ref_z[:T] = sample
        for n in range(rounds - 1):
            frames = vo.decode_first_stage(dsdt, dcfg, sample[-14:], eng.scale_factor)
            cc = co.recondition(to_t(c), frames, sample, lambda im: co.prediction_embedder(csdt, ccfg, im),
                                eng.scale_factor)
            ref_cross.append(cc["crossattn"])
            filled = torch.zeros_like(zt)
            filled[[0, 1, 2]] = sample[-3:]
            sample = fn(noises[n + 1].clone(), cc, filled, pred_mask)
            ref_z[(n + 1) * (T - 3) + 3:(n + 1) * (T - 3) + T] = sample[3:]
    rc = [rel_l2(a[..., :1024], b[..., :1024]) for a, b in zip(seen, ref_cross)]
    r = rel_l2(samples_z.cpu(), ref_z)
    print(f"rollout {rounds} rounds with CLIP re-conditioning: latents rel-L2 {r:.3e}, CLIP rows {[f'{x:.2e}' for x in rc]}")
    assert all(x < 5e-3 for x in rc) and r < 5e-3
