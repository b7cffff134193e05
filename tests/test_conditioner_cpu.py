"""The native conditioner without a GPU: vista_b200.conditioner.GeneralConditioner (sinusoidal embedders, CLIP, cond-frame
encoder) built from configs/inference/vista_b200_native.yaml at tiny sizes, on CPU emulations of the kernels, against the
fixtures of the REAL reference conditioner (oracle/make_golden_cond.py); its routing rules; the checkpoint keys it loads;
and engine.rollout re-conditioned by it against the reference's own do_sample."""
import math
import os
import subprocess
import sys

import pytest
import torch
import yaml

import seam_fakes as sf
from cond_fake_ops import patched_cond_ops
from helpers import golden, golden_rel, rel_l2
from oracle import make_golden_cond as mgc
from vista_b200 import spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLIP_DIM = 1024


def native_engine(steps=2, cpu=True):
    """Engine from configs/inference/vista_b200_native.yaml at the tiny presets with the seam checkpoint and the conditioner
    weights of the fixtures (reference key names); ``cpu``: its native runtimes are built on the CPU, for emulated ops."""
    from vista_b200.diffusion import instantiate_from_config
    ucfg, dcfg, ecfg = cfgs = sf.presets()
    cfg = yaml.safe_load(open(os.path.join(ROOT, "configs", "inference", "vista_b200_native.yaml")))["model"]
    p = cfg["params"]
    p["network_config"]["params"].update(model_channels=ucfg.model_channels, channel_mult=list(ucfg.channel_mult),
                                         num_res_blocks=ucfg.num_res_blocks, attention_resolutions=list(ucfg.attention_resolutions))
    fs = p["first_stage_config"]["params"]
    fs["decoder_config"]["params"].update(ch=dcfg.ch, ch_mult=list(dcfg.ch_mult), num_res_blocks=dcfg.num_res_blocks)
    fs["encoder_config"]["params"].update(ch=ecfg.ch, ch_mult=list(ecfg.ch_mult), num_res_blocks=ecfg.num_res_blocks)
    cp = p["conditioner_config"]["params"]
    cp["emb_models"] = mgc.tiny_emb_models(cp["emb_models"], clip_arch=spec.clip_preset("tiny"))
    p["sampler_config"]["params"].update(num_steps=steps, device="cpu" if cpu else "cuda")
    p["sampler_config"]["params"]["guider_config"] = {"target": "vista_b200.diffusion.TrianglePredictionGuider",
                                                      "params": {"max_scale": 2.5, "num_frames": sf.T}}
    eng = instantiate_from_config(cfg)
    ck = dict(sf.checkpoint(cfgs))
    ck.update(mgc.conditioner_checkpoint())
    missing, unexpected = eng.load_state_dict(ck, strict=False)
    assert not missing and not unexpected, (missing[:3], unexpected[:3])
    if cpu:
        to_cpu(eng)
    return eng


def to_cpu(eng):
    """Instance-level overrides that build the engine's runtimes on the CPU (the emulated operators run there)."""
    from vista_b200 import clip as clip_mod
    from vista_b200 import vae as vae_mod
    eng.model._require_cuda = eng.model.diffusion_model._require_cuda = lambda device: None
    dec = eng.first_stage_model.decoder
    dec.runtime = lambda device: dec.__dict__.setdefault("_rt_cpu", vae_mod.DecoderRuntime(dec.b200_config, dec.state_dict(), "cpu"))
    oc = eng.conditioner.embedders[0].open_clip
    oc.runtime = lambda device: oc.__dict__.setdefault("_rt_cpu", clip_mod.ClipRuntime(oc.b200_config, oc.state_dict(), "cpu"))
    ae = eng.conditioner.embedders[3].encoder
    ae.runtime = lambda device: ae.__dict__.setdefault("_rt_cpu", vae_mod.EncoderRuntime(
        ae.encoder.b200_config, ae.encoder.state_dict(), "cpu",
        post=(ae.quant_conv.weight.detach().float().flatten(1), ae.quant_conv.bias.detach().float())))


def condition_case(eng, case):
    """engine.condition for one fixture case (the re-conditioning case with skip_encode set, as do_sample sets it)."""
    vd = mgc.recondition_value_dict() if case == "recond" else mgc.value_dict(case)
    skip = case == "recond"
    for e in eng.conditioner.embedders:
        if hasattr(e, "skip_encode"):
            e.skip_encode = skip
    try:
        return eng.condition(vd, mgc.T, mgc.UC_KEYS), vd
    finally:
        for e in eng.conditioner.embedders:
            if hasattr(e, "skip_encode"):
                e.skip_encode = False


def check_against_fixture(c, uc, g, case, vd, image_bar):
    """Every row equals row 0; sinusoid columns within 1e-6 abs, CLIP slot and concat within ``image_bar`` rel-L2, forced
    zeros exactly zero.  Returns the worst (CLIP, concat) rel-L2."""
    worst = [0.0, 0.0]
    for tag, d in (("c", c), ("uc", uc)):
        assert sorted(d) == sorted(k.split("_", 2)[2] for k in g.files if k.startswith(f"{case}_{tag}_")), (case, tag)
        for k, v in d.items():
            v = v.detach().float().cpu()
            ref = torch.from_numpy(g[f"{case}_{tag}_{k}"])
            assert v.shape[0] == mgc.T and tuple(v.shape[1:]) == tuple(ref.shape[1:]), (case, tag, k, v.shape, ref.shape)
            assert torch.equal(v, v[:1].expand_as(v)), (case, tag, k)
            v = v[:1]
            if k == "vector":
                assert (v - ref).abs().max() <= 1e-6, (case, tag, k, float((v - ref).abs().max()))
            elif k == "crossattn":
                assert (v[..., CLIP_DIM:] - ref[..., CLIP_DIM:]).abs().max() <= 1e-6, (case, tag)
                if tag == "uc":
                    assert not v[..., :CLIP_DIM].any()
                else:
                    r = rel_l2(v[..., :CLIP_DIM], ref[..., :CLIP_DIM])
                    worst[0] = max(worst[0], r)
                    assert r < image_bar, (case, tag, r)
            else:
                if tag == "uc":
                    assert not v.any()
                elif case == "recond":      # skip_encode: the latent passes through
                    assert torch.equal(v, vd["cond_frames"].float()), case
                else:
                    r = rel_l2(v, ref)
                    worst[1] = max(worst[1], r)
                    assert r < image_bar, (case, tag, r)
    return worst


@pytest.fixture
def no_graph(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)


def test_conditioner_on_emulated_ops_matches_reference():
    g = golden("cond_vista_tiny")
    assert int(g["rows"]) == mgc.T and list(g["uc_keys"]) == mgc.UC_KEYS
    eng = native_engine()
    with patched_cond_ops(), torch.no_grad():
        for case in mgc.CASES + ("recond",):
            (c, uc), vd = condition_case(eng, case)
            worst = check_against_fixture(c, uc, g, case, vd, 5e-3)
            print(f"{case}: CLIP rel-L2 {worst[0]:.2e}, concat rel-L2 {worst[1]:.2e}")
    # repeated rows: CLIP and the encoder ran on one row per conditioned call, never on the uc batch
    assert eng.conditioner.rows_embedded == {"cond_frames_without_noise": 6, "cond_frames": 5}


def _sin(v, outdim):
    """timestep_embedding (util.py:155-164) of every value, "(b d) d2 -> b (d d2)"."""
    half = outdim // 2
    f = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    a = v.float().reshape(-1, 1) * f
    e = torch.cat([torch.cos(a), torch.sin(a)], 1)
    if outdim % 2:
        e = torch.cat([e, torch.zeros(e.shape[0], 1)], 1)
    return e.reshape(v.shape[0], -1)


def _scalar_conditioner(models):
    from vista_b200.conditioner import GeneralConditioner
    return GeneralConditioner([{"input_key": k, "target": "vista_b200.conditioner.ConcatTimestepEmbedderND", "params": p}
                               for k, p in models])


def test_routing_rules():
    B = 3
    batch = {"fps_id": torch.tensor([9, 9, 4]), "cond_aug": torch.tensor([0.02, 0.0, 1.5]),
             "trajectory": torch.randn(B, 8) * 10, "command": torch.tensor([0, 2, 3])}
    with patched_cond_ops():
        cond = _scalar_conditioner([("fps_id", dict(outdim=256)), ("motion_bucket_id", dict(outdim=256)),
                                    ("cond_aug", dict(outdim=255)), ("command", dict(outdim=128, num_features=1, add_sequence_dim=True)),
                                    ("speed", dict(outdim=128, num_features=4, add_sequence_dim=True)),
                                    ("trajectory", dict(outdim=128, num_features=8, add_sequence_dim=True))])
        out = cond(batch)
        # a missing key without add_sequence_dim is left out (motion_bucket_id); an odd outdim has a zero last column
        assert torch.equal(out["vector"], torch.cat([_sin(batch["fps_id"], 256), _sin(batch["cond_aug"], 255)], 1))
        # a missing key with add_sequence_dim gives zeros (speed), rows from cond_aug; int64 input is cast (command)
        want = torch.cat([_sin(batch["command"], 128), torch.zeros(B, 512), _sin(batch["trajectory"], 128)], 1)[:, None]
        assert out["crossattn"].shape == (B, 1, 128 + 512 + 1024) and torch.equal(out["crossattn"], want)
        # forced zeros
        z = cond(batch, force_zero_embeddings=["trajectory", "fps_id"])
        assert not z["vector"][:, :256].any() and torch.equal(z["vector"][:, 256:], out["vector"][:, 256:])
        assert not z["crossattn"][..., 640:].any() and torch.equal(z["crossattn"][..., :640], out["crossattn"][..., :640])
        c, uc = cond.get_unconditional_conditioning(batch, force_uc_zero_embeddings=["command"])
        assert torch.equal(c["crossattn"], out["crossattn"]) and not uc["crossattn"][..., :128].any()
        # the 768 rule: a 768-wide vector embedding is added to an existing vector, not concatenated
        add = _scalar_conditioner([("fps_id", dict(outdim=768)), ("cond_aug", dict(outdim=768)), ("command", dict(outdim=256))])
        v = add(batch)["vector"]
        assert v.shape == (B, 768 + 256)
        assert torch.equal(v[:, :768], _sin(batch["fps_id"], 768) + _sin(batch["cond_aug"], 768))
        assert torch.equal(v[:, 768:], _sin(batch["command"], 256))
        # the embedder alone (modules.py:414-425): x.ndim == 1 -> x[:, None]
        from vista_b200.conditioner import ConcatTimestepEmbedderND
        e = ConcatTimestepEmbedderND(128, num_features=1, add_sequence_dim=True)
        assert torch.equal(e(batch["command"]), _sin(batch["command"], 128)[:, None])


@pytest.mark.parametrize("opt", [dict(ucg_rate=0.1), dict(legacy_ucg_value=0.0), dict(is_trainable=True),
                                 dict(input_keys=["fps_id"])])
def test_training_options_raise(opt):
    from vista_b200.conditioner import GeneralConditioner
    entry = {"input_key": "fps_id", "target": "vista_b200.conditioner.ConcatTimestepEmbedderND", "params": {"outdim": 256}}
    entry.update(opt)
    if "input_keys" in opt:
        del entry["input_key"]
    with pytest.raises(NotImplementedError):
        GeneralConditioner([entry])


def test_checkpoint_conditioner_keys_load():
    """`conditioner.embedders.0.open_clip.model.visual.*` and `conditioner.embedders.3.encoder.*` of a reference checkpoint
    fill the engine's conditioner (the CLIP text leftovers are accepted and dropped)."""
    eng = native_engine(cpu=False)
    ck = mgc.conditioner_checkpoint()
    for k in spec.CLIP_TEXT_LEFTOVERS:
        ck["conditioner.embedders.0.open_clip.model." + k] = torch.zeros(3)
    missing, unexpected = eng.load_state_dict(ck, strict=False)
    assert not unexpected, unexpected[:3]
    assert not [m for m in missing if m.startswith("_conditioner.")]
    sd = eng.state_dict()
    for k, v in mgc.conditioner_checkpoint().items():
        assert torch.equal(sd["_conditioner." + k[len("conditioner."):]], v), k


def test_engine_rollout_reconditioned_equals_the_real_do_sample(no_graph):
    """engine.rollout with conditioner_recondition against the unmodified sample_utils.do_sample on the all-reference engine
    holding the real conditioner: same encoded clip, sampler noise, trajectory action and uc_keys."""
    from vista_b200.rollout import conditioner_recondition
    g = golden("seam_rollout_cond")
    rounds, steps = int(g["rounds"]), int(g["steps"])
    eng = native_engine(steps)
    eng.en_and_decode_n_samples_a_time = 14
    vd = mgc.rollout_value_dict(sf)
    z = torch.from_numpy(g["z"])
    noises = [sf.noise("rollout_cond", i, z.shape) for i in range(rounds)]
    with patched_cond_ops(), torch.no_grad():
        c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
        frames, samples_z = eng.rollout(c, uc, z, rounds, noises=noises,
                                        recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS))
    assert all(not getattr(e, "skip_encode", False) for e in eng.conditioner.embedders)
    n = rounds * (sf.T - 3) + 3
    assert samples_z.shape == (n, 4, sf.H // 2, sf.W // 2) and frames.shape == (n, 3, sf.H, sf.W)
    rz, rx = golden_rel(samples_z, g, "lat_"), golden_rel(frames, g, "frames_")
    print(f"engine.rollout + conditioner_recondition vs the real do_sample: latents rel-L2 {rz}, frames rel-L2 {rx}")
    assert max(rz) < 5e-3 and max(rx) < 5e-3, (rz, rx)


def test_native_engine_conditions_without_the_reference_package():
    """A fresh interpreter turns an image and a trajectory into c / uc with the native-YAML engine and never imports vwm."""
    code = (
        "import sys, torch\n"
        "import test_conditioner_cpu as t\n"
        "from cond_fake_ops import patched_cond_ops\n"
        "from vista_b200 import fused\n"
        "fused.USE_GRAPH = False\n"
        "eng = t.native_engine()\n"
        "img = torch.rand(1, 3, 32, 64) * 2 - 1\n"
        "vd = {'fps_id': 9, 'motion_bucket_id': 127, 'cond_aug': 0.02, 'cond_frames_without_noise': img,\n"
        "      'cond_frames': img, 'trajectory': torch.arange(8.0)}\n"
        "with patched_cond_ops():\n"
        "    c, uc = eng.condition(vd, 25, t.mgc.UC_KEYS)\n"
        "assert c['crossattn'].shape == (25, 1, 3456) and c['vector'].shape == (25, 768), c['crossattn'].shape\n"
        "assert c['concat'].shape == (25, 4, 16, 32) and not uc['concat'].any()\n"
        "assert c['crossattn'][:, :, 1152:2176].abs().sum() > 0\n"
        "bad = sorted(m for m in sys.modules if m == 'vwm' or m.startswith('vwm.'))\n"
        "assert not bad, bad\n"
        "print('ok')\n")
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, ROOT]))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(args, cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
