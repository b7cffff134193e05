"""The conditioner's CLIP image branch without a GPU: the CPU oracle (oracle/clip_oracle.py) against the fixtures made by
the real reference classes (oracle/make_golden_clip.py), the parameter inventory and state-dict loading of
vista_b200.clip, its option checks, and its host executor on CPU emulations of the new operators."""
import numpy as np
import pytest
import torch

from clip_fake_ops import patch_rows, patched_clip_ops
from helpers import golden, rel_l2
from oracle import clip_oracle as co
from oracle.make_golden_clip import CASES, clip_frames, clip_weights
from vista_b200 import spec, synth


def _case(name):
    g = golden(name)
    preset, seed, frames = CASES[name]
    cfg, sd = clip_weights(preset, seed)
    assert str(g["weights_crc"]) == synth.state_dict_checksum(sd)
    out = []
    for fname, n, H, W, aa in frames:
        assert list(g[f"{fname}_shape"]) == [n, H, W, int(aa)]
        x = clip_frames(seed, fname, n, H, W)
        assert str(g[f"{fname}_frames_crc"]) == synth.checksum([x])
        out.append((fname, torch.from_numpy(x), aa))
    return g, cfg, {k: torch.from_numpy(v) for k, v in sd.items()}, out


def test_oracle_matches_reference_clip_tiny():
    g, cfg, sd, frames = _case("clip_tiny")
    s = int(g["pre_stride"])
    for fname, x, aa in frames:
        pre = co.preprocess(x, aa)
        assert rel_l2(pre[:, :, ::s, ::s], torch.from_numpy(g[f"{fname}_pre"])) < 2e-5
        z = co.prediction_embedder(sd, cfg, x, antialias=aa)
        assert z.shape == g[f"{fname}_emb"].shape
        assert rel_l2(z, torch.from_numpy(g[f"{fname}_emb"])) < 2e-5, fname


@pytest.mark.slow
def test_oracle_matches_reference_clip_vith_14():
    g, cfg, sd, frames = _case("clip_vith_14")
    for fname, x, aa in frames:
        z = co.prediction_embedder(sd, cfg, x, antialias=aa)
        assert rel_l2(z, torch.from_numpy(g[f"{fname}_emb"])) < 2e-5


def test_param_inventory_and_load_state_dict():
    from vista_b200.clip import FrozenOpenCLIPImageEmbedder, FrozenOpenCLIPImagePredictionEmbedder
    cfg = spec.clip_preset("vit_h_14")
    specs = spec.clip_param_specs(cfg)
    n = sum(int(np.prod(s)) for s, _ in specs.values())
    assert 630e6 < n < 635e6                       # open_clip ViT-H-14 visual: 632 M parameters
    assert specs["conv1.weight"][0] == (1280, 3, 14, 14) and specs["positional_embedding"][0] == (257, 1280)
    assert specs["proj"][0] == (1280, 1024) and specs["transformer.resblocks.31.attn.in_proj_weight"][0] == (3840, 1280)
    tiny = spec.clip_preset("tiny")
    emb = FrozenOpenCLIPImagePredictionEmbedder(
        {"target": "vista_b200.clip.FrozenOpenCLIPImageEmbedder", "params": {"arch": tiny}}, n_cond_frames=1, n_copies=1)
    keys = set(emb.state_dict())
    want = {"open_clip.model.visual." + k for k in spec.clip_param_specs(tiny)}
    assert keys == want
    # a reference-shaped state dict: the visual tower plus what survives `del model.transformer` (modules.py:277)
    sd = {"open_clip.model.visual." + k: torch.from_numpy(v) for k, v in synth.synth_state_dict(spec.clip_param_specs(tiny), seed=3).items()}
    for k in spec.CLIP_TEXT_LEFTOVERS:
        sd["open_clip.model." + k] = torch.zeros(3)
    missing, unexpected = emb.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    assert torch.equal(emb.open_clip.model.visual.proj, sd["open_clip.model.visual.proj"])
    assert len(sd) == len(want) + len(spec.CLIP_TEXT_LEFTOVERS)      # the caller's dict is left as it was given


def test_load_open_clip_weights(tmp_path):
    from vista_b200.clip import FrozenOpenCLIPImageEmbedder, load_open_clip_weights
    tiny = spec.clip_preset("tiny")
    vis = {"visual." + k: torch.from_numpy(v) for k, v in synth.synth_state_dict(spec.clip_param_specs(tiny), seed=4).items()}
    ckpt = dict(vis)
    ckpt.update({"transformer.resblocks.0.attn.in_proj_weight": torch.zeros(2, 2), "token_embedding.weight": torch.zeros(2),
                 "logit_scale": torch.zeros(())})
    torch.save(ckpt, tmp_path / "open_clip_pytorch_model.bin")
    sd = load_open_clip_weights(str(tmp_path / "open_clip_pytorch_model.bin"))
    emb = FrozenOpenCLIPImageEmbedder(arch=tiny)
    missing, unexpected = emb.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    assert torch.equal(emb.model.visual.conv1.weight, vis["visual.conv1.weight"])


@pytest.mark.parametrize("kw", [dict(arch="ViT-L-14"), dict(output_tokens=True), dict(num_image_crops=2),
                                dict(ucg_rate=0.1), dict(unsqueeze_dim=True), dict(repeat_to_max_len=True)])
def test_unsupported_options_raise(kw):
    from vista_b200.clip import FrozenOpenCLIPImageEmbedder
    with pytest.raises(NotImplementedError):
        FrozenOpenCLIPImageEmbedder(**kw)


def test_no_cpu_fallback():
    from vista_b200.clip import FrozenOpenCLIPImageEmbedder
    emb = FrozenOpenCLIPImageEmbedder(arch=spec.clip_preset("tiny"), antialias=False)
    with pytest.raises(RuntimeError, match="CUDA"):
        emb(torch.zeros(1, 3, 64, 64))


def test_patch_rows_match_conv1():
    """The K order of the patch rows is the flattening of conv1.weight [width, 3, 14, 14]."""
    torch.manual_seed(0)
    pre = torch.randn(2, 3, 224, 224)
    w = torch.randn(8, 3, 14, 14)
    rows = patch_rows(pre, 640).reshape(2, 257, 640)
    ref = torch.nn.functional.conv2d(pre, w, stride=14).flatten(2).transpose(1, 2)
    got = rows[:, 1:, :588] @ w.reshape(8, 588).t()
    assert torch.allclose(got, ref, atol=1e-4) and torch.equal(rows[:, 0], torch.zeros(2, 640))


def test_executor_on_emulated_ops_matches_clip_tiny(monkeypatch):
    """vista_b200.clip's runtime (packing, buffer plumbing, token assembly through the GEMM row vector, strided ln_post)
    on CPU emulations of the kernels, against the reference fixture at the fp16 bar."""
    from vista_b200 import clip as clip_mod
    from vista_b200.clip import ClipRuntime, FrozenOpenCLIPImagePredictionEmbedder
    g, cfg, sd, frames = _case("clip_tiny")
    emb = FrozenOpenCLIPImagePredictionEmbedder(
        {"target": "vista_b200.clip.FrozenOpenCLIPImageEmbedder", "params": {"arch": cfg}}, n_cond_frames=1, n_copies=2)
    emb.load_state_dict({"open_clip.model.visual." + k: v for k, v in sd.items()})
    oc = emb.open_clip
    monkeypatch.setattr(clip_mod.FrozenOpenCLIPImageEmbedder, "runtime", lambda self, device: self.__dict__.setdefault(
        "_rt_cpu", ClipRuntime(self.b200_config, self.state_dict(), "cpu")))
    with patched_clip_ops():
        for fname, x, aa in frames:
            oc.antialias = aa
            z = emb(x)
            want = torch.from_numpy(g[f"{fname}_emb"])
            assert z.shape == (2 * want.shape[0],) + tuple(want.shape[1:])
            assert torch.equal(z[0::2], z[1::2])                       # n_copies repeats each image's row
            r = rel_l2(z[0::2], want)
            print(f"{fname}: emulated executor vs reference rel-L2 {r:.2e}")
            assert r < 5e-3
