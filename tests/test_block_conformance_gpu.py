"""Layer-level production conformance: the full-size engine of tools/bench_session.build_engine (seeded synthetic weights;
the oracle reads the same weights back from the engine's modules) run eagerly at 576 x 1024, T = 25, under the harness of
tests/block_shadow.py: every UNet, decoder and encoder layer, segment, conditioning vector and hand-off against the fp64
oracle on the input that layer really read.

Each test prints the census (per layer prefix: kind, shape, worst partition ratio), its wall time and its peak memory.
The wall time is dominated by the fp64 reference (the step is 154 TFLOP); the decoder's reference runs in pieces (per
frame, and in row bands for the temporal half: block_shadow.dec_video_res_block_pieces), so that every decoder layer of
the first chunk is checked at 576 x 1024."""
import time

import pytest
import torch

from block_shadow import BlockShadow

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
T, H, W = 25, 576, 1024
UC_KEYS = ["cond_frames", "cond_frames_without_noise", "command", "trajectory", "speed", "angle", "goal"]
ACTION = {"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}


@pytest.fixture(scope="module")
def eng():
    from tools.bench_session import build_engine
    from vista_b200 import lib
    lib.load()
    return build_engine(DEV)


@pytest.fixture(scope="module")
def problem(eng):
    from oracle.make_golden_clip import clip_frames
    from vista_b200 import synth
    frame = torch.from_numpy(clip_frames(12, "block_conformance", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "block_conformance.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    noise = torch.from_numpy(synth.normal(7, "block_conformance.noise", (T, 4, H // 8, W // 8))).to(DEV)
    with torch.no_grad():
        c, uc = eng.condition({**vd, **ACTION}, T, UC_KEYS)
    return vd, z, noise, c, uc


@pytest.fixture(autouse=True)
def eager(monkeypatch):
    from vista_b200 import fused
    monkeypatch.setattr(fused, "USE_GRAPH", False)


def weights(eng):
    from vista_b200 import spec
    unet = (spec.unet_preset("vista"), eng.model.diffusion_model.state_dict())
    dec = (spec.decoder_preset("vista"), eng.first_stage_model.decoder.state_dict())
    ae = eng.conditioner.embedders[3].encoder
    post = (ae.get_parameter("quant_conv.weight").detach().float().flatten(1), ae.get_parameter("quant_conv.bias").detach().float())
    enc = (ae.encoder.b200_config, ae.encoder.state_dict(), post)
    return unet, dec, enc


def block_run(name, fn, **kw):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    with torch.no_grad(), BlockShadow(**kw) as bs:
        fn()
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(DEV) / 2 ** 30
    print(f"\n[{name}] {torch.cuda.get_device_name(DEV)}: wall {wall:.1f} s, peak allocated {peak:.2f} GiB")
    print(bs.report())
    bs.assert_ok()
    return bs


@pytest.mark.parametrize("kind", ["vanilla", "action"])
def test_unet_step_layers(eng, problem, kind, monkeypatch):
    """One Euler step through the full-size UNet: the B = 50 CFG forward under VanillaCFG, and under action guidance
    also the T-row action-free forward (B = 25, its own conditioning and buffers)."""
    from test_production_conformance_gpu import sampler
    vd, z, noise, c, uc = problem
    monkeypatch.setattr(eng, "sampler", sampler(eng, "euler_vanilla" if kind == "vanilla" else "action", 1))
    unet, _, _ = weights(eng)
    bs = block_run(f"unet {kind}", lambda: eng.sample(c, uc=uc, N=T, shape=tuple(z.shape[1:]), noise=noise.clone(),
                                                      cond_frame=z), unet=unet)
    assert bs.n_forward["unet"] == (1 if kind == "vanilla" else 2)


def test_decoder_layers(eng, problem):
    """decode_first_stage_u8 of 25 latents: two 14-frame chunks; the layers of the first chunk, the hand-offs of both."""
    noise = problem[2]
    _, dec, _ = weights(eng)
    bs = block_run("decode", lambda: eng.decode_first_stage_u8(noise * 0.9), decoder=dec, decoder_layer_calls=1)
    assert bs.n_forward["dec"] == 2


def test_encoder_layers(eng, problem):
    """The conditioning encode of one 576 x 1024 frame through engine.condition.  The engine's quant_conv is the
    identity; here it is a seeded non-identity 1x1 convolution, so that the head check sees quant_conv folded into
    conv_out (the engine's own is restored afterwards)."""
    vd = problem[0]
    ae = eng.conditioner.embedders[3].encoder
    qw, qb = ae.get_parameter("quant_conv.weight"), ae.get_parameter("quant_conv.bias")
    saved = qw.detach().clone(), qb.detach().clone()
    g = torch.Generator().manual_seed(11)
    try:
        with torch.no_grad():
            qw.copy_((torch.eye(8) + 0.3 * torch.randn(8, 8, generator=g)).reshape(qw.shape))
            qb.copy_(0.1 * torch.randn(8, generator=g))
        ae._runtime = None
        _, _, enc = weights(eng)
        bs = block_run("encode", lambda: eng.condition({**vd, **ACTION}, T, UC_KEYS), encoder=enc)
    finally:
        with torch.no_grad():
            qw.copy_(saved[0])
            qb.copy_(saved[1])
        ae._runtime = None
    assert bs.n_forward["enc"] >= 1
