"""Host-side executors (vae.DecoderRuntime / EncoderRuntime) run on CPU tensors against an emulation of the C-ABI
operators (tests/fake_ops.py): checks the orchestration — buffer reuse, weight repacking, tap and gather conventions,
residual / blend wiring — against the REAL reference's fixtures without a GPU.  The decoder is the control (its GPU
parity is established): if the emulated decoder matches, the emulation is faithful, and the encoder executor, which has
not run on hardware yet, is checked by the same means."""
import pytest
import torch

from fake_ops import patched_ops
from helpers import decoder_weights, golden, rel_l2, to_t
from vista_b200 import spec, synth


def test_decoder_executor_on_emulated_ops_matches_reference():
    from vista_b200.vae import DecoderRuntime, decode_first_stage
    cfg, sd = decoder_weights("tiny")
    z = torch.from_numpy(synth.normal(9, "decfs.z", (25, cfg.z_channels, 8, 16), std=0.18215))
    with patched_ops(), torch.no_grad():
        rt = DecoderRuntime(cfg, to_t(sd), "cpu")
        out = decode_first_stage(rt, z)
    r = rel_l2(out, torch.from_numpy(golden("decode_first_stage_tiny")["out"]))
    assert r < 5e-3, r


@pytest.mark.parametrize("name,preset,h,w,n", [("encoder_tiny", "tiny", 32, 64, 5), ("encoder_small", "small", 64, 128, 3)])
def test_encoder_executor_on_emulated_ops_matches_reference(name, preset, h, w, n):
    from vista_b200.vae import EncoderRuntime, encode_first_stage
    g = golden(name)
    cfg = spec.encoder_preset(preset)
    sd = synth.synth_state_dict(spec.encoder_param_specs(cfg), seed=3)
    x = torch.from_numpy(synth.normal(11, "enc.x", (n, cfg.in_channels, h, w), std=0.5))
    noise = torch.from_numpy(synth.normal(12, "enc.noise", tuple(g["z"].shape), std=1.0))
    with patched_ops(), torch.no_grad():
        rt = EncoderRuntime(cfg, to_t(sd), "cpu")
        z = encode_first_stage(rt, x, n_samples=int(g["n_chunk"]), noise=noise)
    r = rel_l2(z, torch.from_numpy(g["z"]))
    assert r < 5e-3, r


def _unet_forward_emulated(preset, h, w, T, sigma=5.0):
    import numpy as np
    from helpers import unet_inputs, unet_weights
    from vista_b200 import ops
    from vista_b200.unet import UNetRuntime, padded_input_rows
    cfg, sd = unet_weights(preset)
    with patched_ops(), torch.no_grad():
        rt = UNetRuntime(cfg, to_t(sd), "cpu", num_frames=T)
        x, cc, mask2 = unet_inputs(7, cfg, h, w, T)
        B = 2 * T
        c_in = 1.0 / np.sqrt(sigma * sigma + 1.0)
        xin = torch.from_numpy(np.concatenate([x * np.float32(c_in), cc["concat"]], 1))
        tok = padded_input_rows(B * h * w, "cpu")             # the production layout: input conv as a tap-GEMM
        ops.nchw_to_tokens(xin.contiguous(), tok, B, 8, h, w)
        rt.set_conditioning(torch.from_numpy(cc["crossattn"]), torch.from_numpy(cc["vector"]))
        c_noise = torch.full((B,), 0.25 * float(np.log(sigma)))
        out = rt.forward(tok, c_noise, torch.from_numpy(mask2), h, w)
        res = torch.empty(B, cfg.out_channels, h, w)
        ops.tokens_to_nchw(out, res, B, cfg.out_channels, h, w)
    return res


def test_unet_executor_on_emulated_ops_matches_reference():
    """Control for the multi-rank emulation below: the single-rank UNet executor on emulated operators reproduces the
    real reference's forward (same fixture as the GPU test)."""
    out = _unet_forward_emulated("tiny", 8, 16, 25)
    ref = torch.from_numpy(golden("unet_tiny")["raw"])
    r = rel_l2(out, ref)
    assert r < 5e-3, r


# ---- multi-rank orchestration on emulated operators (gloo): the layouts the GPU budget cannot cover ----
def _sharded_worker(rank, world, port, cfg_split, q):
    import os
    import numpy as np
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_ops import patched_ops as patched
        from helpers import to_t as tt, unet_weights
        from vista_b200 import synth as sy
        from vista_b200.diffusion import B200Denoiser, Denoiser, EulerEDMSampler
        from vista_b200.modules import B200Wrapper, VideoUNet
        cfg, sd = unet_weights("tiny")
        unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                         num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                         channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                         context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                         use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                         use_linear_in_transformer=True, action_control=True)
        unet.load_state_dict(tt(sd), strict=True)
        T, h, w, steps = 25, 8, 16, 4
        c, uc = sy.synth_conditioning(7, T, h, w, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
        noise, z, mask = sy.synth_latents(7, T, h, w)
        td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
        den = Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=T)
        smp = EulerEDMSampler(num_steps=steps, device="cpu", s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, verbose=False,
                              discretization_config={"target": "vista_b200.diffusion.EDMDiscretization",
                                                     "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}},
                              guider_config={"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 2.5}})
        net = B200Wrapper(unet)
        net._require_cuda = lambda device: None            # the executors run on the emulated operators here
        net.enable_frame_sharding(cfg_split=cfg_split)
        with patched(), torch.no_grad():
            out = smp(B200Denoiser(den, net), torch.from_numpy(noise).clone(), td(c), uc=td(uc),
                      cond_frame=torch.from_numpy(z), cond_mask=torch.from_numpy(mask))
        rt = net._runtime
        st = next(iter(rt._loop_states.values()))
        q.put((rank, out.numpy(), st.tape is not None and len(st.tape) > 0, int(rt.t1 - rt.t0)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,cfg_split", [(4, True), (8, True), (4, False), (8, False)])
def test_sharded_sampler_on_emulated_ops(world, cfg_split):
    """One clip over 4 / 8 ranks (gloo, emulated operators): CFG halves x frame shards (sub-group collectives, pairwise
    exchange) and frames only, with the step recorded on the launch tape and replayed.  Every rank must end with the
    same latent, and it must match the REAL reference's 4-step sample (tests/golden/sampler_tiny_cfg.npz)."""
    import os
    import numpy as np
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() + 7 * world + int(cfg_split)) % 2000
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, cfg_split, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=240) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    ref = torch.from_numpy(golden("sampler_tiny_cfg")["sample"])
    frames = [r[3] for r in res]
    fw = world // 2 if cfg_split else world
    assert sorted(frames[:fw], reverse=True) == frames[:fw] and sum(frames[:fw]) == 25
    for rank, out, taped, _ in res:
        assert taped, "the step must have been recorded on the launch tape"
        assert np.array_equal(out, res[0][1]), f"rank {rank} holds a different latent"
        r = rel_l2(torch.from_numpy(out), ref)
        assert r < 5e-3, (rank, r)


def _pdecode_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_ops import patched_ops as patched
        from helpers import decoder_weights as dw, to_t as tt
        from vista_b200 import synth as sy
        from vista_b200.vae import DecoderRuntime, decode_first_stage, decode_first_stage_parallel
        cfg, sd = dw("tiny")
        z = torch.from_numpy(sy.normal(9, "decfs.z", (25, cfg.z_channels, 8, 16), std=0.18215))
        with patched(), torch.no_grad():
            rt = DecoderRuntime(cfg, tt(sd), "cpu")
            serial = decode_first_stage(rt, z)
            par = decode_first_stage_parallel(rt, z)
            small = decode_first_stage_parallel(rt, z, n_samples=8, overlap=2)      # 4 chunks over the ranks
            small_serial = decode_first_stage(rt, z, n_samples=8, overlap=2)
        q.put((rank, bool(torch.equal(serial, par)), bool(torch.equal(small, small_serial)), par.numpy()))
    finally:
        dist.destroy_process_group()


def test_parallel_decode_on_emulated_ops_three_ranks():
    """decode_first_stage_parallel with more ranks than chunks (3 ranks, 2 chunks) and with more chunks than ranks
    (4 chunks): bit-identical to the serial chunked decode on every rank, and equal to the reference fixture."""
    import os
    import torch.multiprocessing as mp
    world = 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 37500 + os.getpid() % 2000
    procs = [ctx.Process(target=_pdecode_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=240) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ref = torch.from_numpy(golden("decode_first_stage_tiny")["out"])
    for rank, same, same_small, out in res:
        assert same and same_small, rank
        assert rel_l2(torch.from_numpy(out), ref) < 5e-3


@pytest.mark.parametrize("name,steps,guider,n_cond", [("sampler_tiny_cfg", 4, "VanillaCFG", 1),
                                                     ("sampler_tiny_triangle", 3, "TrianglePredictionGuider", 3)])
def test_fused_and_generic_sampler_on_emulated_ops(name, steps, guider, n_cond, monkeypatch):
    """Single-rank sampler host logic on emulated operators: the fused loop (device-side step index, scale vector,
    conditioning-frame re-imposition) and the generic loop through B200Wrapper both reproduce the real reference's
    samples; same cases as tests/test_sampler_gpu.py."""
    from helpers import unet_weights
    from vista_b200 import fused as fused_mod
    from vista_b200.diffusion import B200Denoiser, Denoiser, EulerEDMSampler
    from vista_b200.modules import B200Wrapper, VideoUNet
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)          # no CUDA graphs on the emulated path
    cfg, sd = unet_weights("tiny")
    unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                     num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                     channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                     context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                     use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                     use_linear_in_transformer=True, action_control=True)
    unet.load_state_dict(to_t(sd), strict=True)
    net = B200Wrapper(unet)
    net._require_cuda = unet._require_cuda = lambda device: None
    den = Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=25)
    g = {"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 2.5}} if guider == "VanillaCFG" else \
        {"target": "vista_b200.diffusion.TrianglePredictionGuider", "params": {"max_scale": 2.5, "num_frames": 25}}
    smp = EulerEDMSampler(num_steps=steps, device="cpu", s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, verbose=False,
                          discretization_config={"target": "vista_b200.diffusion.EDMDiscretization",
                                                 "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}},
                          guider_config=g)
    c, uc = synth.synth_conditioning(7, 25, 8, 16, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
    noise, z, mask = synth.synth_latents(7, 25, 8, 16)
    mask[:n_cond] = 1.0
    td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    zt, mt = torch.from_numpy(z), torch.from_numpy(mask)
    ref = torch.from_numpy(golden(name)["sample"])
    with patched_ops(), torch.no_grad():
        fused = smp(B200Denoiser(den, net), torch.from_numpy(noise).clone(), td(c), uc=td(uc), cond_frame=zt, cond_mask=mt)
        generic = smp(lambda x, s, cc, m: den(net, x, s, cc, m), torch.from_numpy(noise).clone(), td(c), uc=td(uc),
                      cond_frame=zt, cond_mask=mt)
    assert rel_l2(fused, ref) < 5e-3 and rel_l2(generic, ref) < 5e-3
    assert torch.equal(fused[:n_cond], zt[:n_cond])              # conditioning frames re-imposed (sampling.py:122-123)


def _sdecode_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_ops import patched_ops as patched
        from helpers import decoder_weights as dw, to_t as tt
        from vista_b200 import synth as sy
        from vista_b200.sharded import ShardedDecoderRuntime, decode_first_stage_sharded
        from vista_b200.vae import DecoderRuntime, decode_first_stage
        cfg, sd = dw("tiny")
        z = torch.from_numpy(sy.normal(9, "decfs.z", (25, cfg.z_channels, 8, 16), std=0.18215))
        with patched(), torch.no_grad():
            serial = decode_first_stage(DecoderRuntime(cfg, tt(sd), "cpu"), z)
            sharded = decode_first_stage_sharded(ShardedDecoderRuntime(cfg, tt(sd), "cpu"), z)
        q.put((rank, serial.numpy(), sharded.numpy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_frame_sharded_decode_on_emulated_ops(world):
    """Experimental frame-sharded decode (sharded.ShardedDecoderRuntime): 14-frame chunks over 2 / 4 ranks (interior
    ranks, one- and multi-frame shards) reproduce the serial chunked decode up to the re-association of the temporal
    GroupNorm sums, on every rank, and match the reference fixture."""
    import os
    import numpy as np
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 39500 + (os.getpid() + 11 * world) % 2000
    procs = [ctx.Process(target=_sdecode_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=240) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ref = torch.from_numpy(golden("decode_first_stage_tiny")["out"])
    for rank, serial, sharded in res:
        assert np.array_equal(sharded, res[0][2]), "every rank must hold the same clip"
        r1 = rel_l2(torch.from_numpy(sharded), torch.from_numpy(serial))
        assert r1 < 2e-3, (rank, r1)
        assert rel_l2(torch.from_numpy(sharded), ref) < 5e-3


def test_multi_round_rollout_through_the_reference_closure_on_emulated_ops(monkeypatch):
    """BASELINE config 4 semantics (sample_utils.py:318-365): round 1 conditioned on frame 0, later rounds on the last
    three latents through cond_mask[[0,1,2]], TrianglePredictionGuider, results stitched into samples_z.  The sampler
    receives the reference's own closure shape around an engine-like object and must reach the fused loop; the result
    is compared with the same loop on the CPU oracle."""
    from helpers import rollout, unet_weights
    from oracle import vista_oracle as vo
    from vista_b200 import fused as fused_mod
    from vista_b200.diffusion import Denoiser, EulerEDMSampler
    from vista_b200.modules import B200Wrapper, VideoUNet
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    calls = {"fused": 0}
    real_fused = fused_mod.fused_sample
    monkeypatch.setattr(fused_mod, "fused_sample", lambda *a, **k: (calls.__setitem__("fused", calls["fused"] + 1), real_fused(*a, **k))[1])
    cfg, sd = unet_weights("tiny")
    unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                     num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                     channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                     context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                     use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                     use_linear_in_transformer=True, action_control=True)
    unet.load_state_dict(to_t(sd), strict=True)

    class Engine:
        pass
    model = Engine()
    model.model = B200Wrapper(unet)
    model.model._require_cuda = unet._require_cuda = lambda device: None
    model.denoiser = Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=25)

    def denoiser(x, sigma, cond, cond_mask):           # sample_utils.py:314-315, verbatim shape
        return model.denoiser(model.model, x, sigma, cond, cond_mask)
    T, h, w, steps, rounds = 25, 8, 16, 3, 2
    smp = EulerEDMSampler(num_steps=steps, device="cpu", s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, verbose=False,
                          discretization_config={"target": "vista_b200.diffusion.EDMDiscretization",
                                                 "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}},
                          guider_config={"target": "vista_b200.diffusion.TrianglePredictionGuider",
                                         "params": {"max_scale": 2.5, "num_frames": T}})
    c, uc = synth.synth_conditioning(7, T, h, w, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
    _, z, _ = synth.synth_latents(7, T, h, w)
    td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    zt = torch.from_numpy(z)
    noises = [torch.from_numpy(synth.normal(20 + i, "rollout.noise", (T, 4, h, w), std=1.0)) for i in range(rounds)]
    with patched_ops(), torch.no_grad():
        ours = rollout(lambda nz, cf, m: smp(denoiser, nz, cond=td(c), uc=td(uc), cond_frame=cf, cond_mask=m), zt, noises, T)
    assert calls["fused"] == rounds, "the reference's closure must reach the fused loop"
    sdt = to_t(sd)
    with torch.no_grad():
        ref = rollout(lambda nz, cf, m: vo.euler_edm_sample(sdt, cfg, nz, td(c), td(uc), cf, m, steps, T,
                                                            guider="TrianglePredictionGuider", scale=2.5), zt, noises, T)
    assert ours.shape == ref.shape == (rounds * (T - 3) + 3, 4, h, w)
    r = rel_l2(ours, ref)
    assert r < 5e-3, r


def test_engine_encode_sample_decode_on_emulated_ops(monkeypatch):
    """The DiffusionEngine surface end to end on emulated operators, built from configs/inference/vista_b200.yaml with
    tiny sizes and the B200 encoder plugged in: encode_first_stage(images) -> sample() ->
    decode_first_stage(), each stage against the CPU oracle, plus the reference checkpoint key layout."""
    import os
    import yaml
    from helpers import decoder_weights, unet_weights
    from oracle import vista_oracle as vo
    from vista_b200 import fused as fused_mod
    from vista_b200.diffusion import instantiate_from_config
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.safe_load(open(os.path.join(root, "configs", "inference", "vista_b200.yaml")))["model"]
    p = cfg["params"]
    p["network_config"]["params"].update(model_channels=64, channel_mult=[1, 2], num_res_blocks=1, attention_resolutions=[1, 2])
    fs = p["first_stage_config"]["params"]
    fs["decoder_config"]["params"].update(ch=64, ch_mult=[1, 2], num_res_blocks=1)
    fs["encoder_config"] = {"target": "vista_b200.vae.Encoder",
                            "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256, in_channels=3,
                                           out_ch=3, ch=64, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[], dropout=0.0)}
    p["sampler_config"]["params"]["num_steps"] = 3
    p["sampler_config"]["params"]["device"] = "cpu"
    p["replace_cond_frames"], p["fixed_cond_frames"] = True, [0]
    p["en_and_decode_n_samples_a_time"] = 14
    eng = instantiate_from_config(cfg)
    ucfg, usd = unet_weights("tiny")
    dcfg, dsd = decoder_weights("tiny")
    ecfg = spec.encoder_preset("tiny")
    esd = synth.synth_state_dict(spec.encoder_param_specs(ecfg), seed=3)
    sd = {"model.diffusion_model." + k: torch.from_numpy(v) for k, v in usd.items()}
    sd.update({"first_stage_model.decoder." + k: torch.from_numpy(v) for k, v in dsd.items()})
    sd.update({"first_stage_model.encoder." + k: torch.from_numpy(v) for k, v in esd.items()})
    missing, unexpected = eng.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    eng.model._require_cuda = eng.model.diffusion_model._require_cuda = lambda device: None
    from vista_b200 import vae as vae_mod                      # CPU executors for this test only
    monkeypatch.setattr(vae_mod.VideoDecoder, "runtime", lambda self, device: self.__dict__.setdefault(
        "_rt_cpu", vae_mod.DecoderRuntime(self.b200_config, self.state_dict(), "cpu")))
    monkeypatch.setattr(vae_mod.Encoder, "runtime", lambda self, device: self.__dict__.setdefault(
        "_rt_cpu", vae_mod.EncoderRuntime(self.b200_config, self.state_dict(), "cpu")))
    T, h, w = 25, 8, 16
    images = torch.from_numpy(synth.normal(31, "engine.images", (T, 3, 2 * h, 2 * w), std=0.5))
    enc_noise = torch.from_numpy(synth.normal(32, "engine.encnoise", (T, 4, h, w), std=1.0))
    c, uc = synth.synth_conditioning(7, T, h, w, trajectory=True, context_dim=ucfg.context_dim, adm=ucfg.adm_in_channels)
    noise, _, mask = synth.synth_latents(7, T, h, w)
    mask[:1] = 1.0
    td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    with patched_ops(), torch.no_grad():
        z = eng.encode_first_stage(images, noise=enc_noise)
        lat = eng.sample(td(c), cond_frame=z, uc=td(uc), N=T, shape=(4, h, w), noise=torch.from_numpy(noise))
        frames = eng.decode_first_stage(lat)
    with torch.no_grad():
        z_ref = vo.encode_first_stage(to_t(esd), ecfg, images, n_samples=14, noise=enc_noise)
        lat_ref = vo.euler_edm_sample(to_t(usd), ucfg, torch.from_numpy(noise), td(c), td(uc), z_ref, torch.from_numpy(mask), 3, T)
        frames_ref = vo.decode_first_stage(to_t(dsd), dcfg, lat_ref)
    assert rel_l2(z, z_ref) < 5e-3 and rel_l2(lat, lat_ref) < 5e-3 and rel_l2(frames, frames_ref) < 1e-2
    assert frames.shape == (T, 3, 2 * h, 2 * w)


def _tiny_engine(monkeypatch, steps=3, guider=None):
    """configs/inference/vista_b200.yaml at tiny sizes on CPU executors over the emulated operators."""
    import os
    import yaml
    from helpers import decoder_weights, unet_weights
    from vista_b200 import fused as fused_mod
    from vista_b200 import vae as vae_mod
    from vista_b200.diffusion import instantiate_from_config
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.safe_load(open(os.path.join(root, "configs", "inference", "vista_b200.yaml")))["model"]
    p = cfg["params"]
    p["network_config"]["params"].update(model_channels=64, channel_mult=[1, 2], num_res_blocks=1, attention_resolutions=[1, 2])
    p["first_stage_config"]["params"]["decoder_config"]["params"].update(ch=64, ch_mult=[1, 2], num_res_blocks=1)
    p["sampler_config"]["params"].update(num_steps=steps, device="cpu")
    if guider is not None:
        p["sampler_config"]["params"]["guider_config"] = guider
    p["replace_cond_frames"], p["fixed_cond_frames"] = True, [0]
    p["en_and_decode_n_samples_a_time"] = 14
    eng = instantiate_from_config(cfg)
    ucfg, usd = unet_weights("tiny")
    dcfg, dsd = decoder_weights("tiny")
    sd = {"model.diffusion_model." + k: torch.from_numpy(v) for k, v in usd.items()}
    sd.update({"first_stage_model.decoder." + k: torch.from_numpy(v) for k, v in dsd.items()})
    missing, unexpected = eng.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    eng.model._require_cuda = eng.model.diffusion_model._require_cuda = lambda device: None
    monkeypatch.setattr(vae_mod.VideoDecoder, "runtime", lambda self, device: self.__dict__.setdefault(
        "_rt_cpu", vae_mod.DecoderRuntime(self.b200_config, self.state_dict(), "cpu")))
    return eng, (ucfg, usd), (dcfg, dsd)


def _reference_rollout(sample_fn, c, z, noises, T, scale_factor, n_cond=3):
    """sample_utils.py:318-365 restated with the conditioner reduced to what the hot path sees: between rounds
    c["concat"] = sample[[-3]] / scale_factor (:343 through the skip_encode embedder, encoders/modules.py:470-471)."""
    init_mask, pred_mask = torch.zeros(T), torch.zeros(T)
    init_mask[0] = 1
    pred_mask[list(range(n_cond))] = 1
    rounds = len(noises)
    samples_z = torch.zeros((rounds * (T - n_cond) + n_cond,) + tuple(z.shape[1:]))
    sample = sample_fn(noises[0].clone(), c, z, init_mask)
    sample[0] = z[0]
    samples_z[:T] = sample
    for n in range(rounds - 1):
        c = dict(c)
        c["concat"] = (sample[[-n_cond]] / scale_factor).expand(c["concat"].shape[0], -1, -1, -1).contiguous()
        filled = torch.zeros_like(z)
        filled[list(range(n_cond))] = sample[-n_cond:]
        sample = sample_fn(noises[n + 1].clone(), c, filled, pred_mask)
        samples_z[(n + 1) * (T - n_cond) + n_cond:(n + 1) * (T - n_cond) + T] = sample[n_cond:]
    return samples_z


def test_engine_rollout_u8_and_ensemble_on_emulated_ops(monkeypatch):
    """SURVEY 8f rows 2-4 on emulated operators: engine.rollout (3 rounds, TrianglePredictionGuider, concat re-conditioning)
    against the same loop over the CPU oracle; the fused uint8 NHWC output against the reference's clamp / scale /
    truncate / rearrange of the fp32 frames; engine.sample_ensemble against reward_utils.py:318-337 over the oracle."""
    from oracle import vista_oracle as vo
    T, h, w, steps, rounds = 25, 8, 16, 2, 3
    guider = {"target": "vista_b200.diffusion.TrianglePredictionGuider", "params": {"max_scale": 2.5, "num_frames": T}}
    eng, (ucfg, usd), (dcfg, dsd) = _tiny_engine(monkeypatch, steps=steps, guider=guider)
    c, uc = synth.synth_conditioning(7, T, h, w, trajectory=True, context_dim=ucfg.context_dim, adm=ucfg.adm_in_channels)
    _, z, _ = synth.synth_latents(7, T, h, w)
    td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    zt = torch.from_numpy(z)
    noises = [torch.from_numpy(synth.normal(40 + i, "rollout.noise", (T, 4, h, w), std=1.0)) for i in range(rounds)]
    with patched_ops(), torch.no_grad():
        frames, samples_z = eng.rollout(td(c), td(uc), zt, rounds, noises=noises)
        frames8, samples_z8 = eng.rollout(td(c), td(uc), zt, rounds, noises=noises, u8=True)
    n_out = rounds * (T - 3) + 3
    assert samples_z.shape == (n_out, 4, h, w) and frames.shape == (n_out, 3, 2 * h, 2 * w)
    assert frames8.shape == (n_out, 2 * h, 2 * w, 3) and frames8.dtype == torch.uint8
    assert torch.equal(samples_z, samples_z8)
    # reference output path (sample_utils.py:374 then :96-126) applied to OUR fp32 frames: must be the same bytes
    want8 = (255.0 * frames).to(torch.uint8).permute(0, 2, 3, 1)
    assert torch.equal(frames8, want8)
    sdt = to_t(usd)
    with torch.no_grad():
        ref_z = _reference_rollout(lambda nz, cc, cf, m: vo.euler_edm_sample(sdt, ucfg, nz, cc, td(uc), cf, m, steps, T,
                                                                           guider="TrianglePredictionGuider", scale=2.5),
                                   td(c), zt, noises, T, eng.scale_factor)
        ref_x = vo.decode_first_stage(to_t(dsd), dcfg, ref_z)
        ref_frames = torch.clamp((ref_x + 1.0) / 2.0, 0.0, 1.0)
    assert rel_l2(samples_z, ref_z) < 5e-3, rel_l2(samples_z, ref_z)
    assert rel_l2(frames, ref_frames) < 1e-2
    ref8 = (255.0 * ref_frames).to(torch.uint8).permute(0, 2, 3, 1)
    assert (frames8.int() - ref8.int()).abs().max() <= 3 and (frames8 != ref8).float().mean() < 0.25

    # ensemble reward (VanillaCFG like reward_utils / sample.py's single-round default)
    eng2, (ucfg, usd), _ = _tiny_engine(monkeypatch, steps=steps)
    K = 3
    en = [torch.from_numpy(synth.normal(60 + i, "ens.noise", (T, 4, h, w), std=1.0)) for i in range(K)]
    with patched_ops(), torch.no_grad():
        reward, members = eng2.sample_ensemble(td(c), td(uc), zt, K, noises=en)
    mask = torch.zeros(T)
    mask[0] = 1
    with torch.no_grad():
        ref_members = []
        for i in range(K):
            s = vo.euler_edm_sample(sdt, ucfg, en[i].clone(), td(c), td(uc), zt, mask, steps, T)
            s[0] = zt[0]
            ref_members.append(s)
        u = torch.mean(torch.stack(ref_members), 0)
        diff = torch.zeros_like(u)
        for s in ref_members:
            diff.add_((s - u) ** 2)
        ref_reward = torch.exp(-(diff / (K - 1)).mean())
    assert all(rel_l2(a, b) < 5e-3 for a, b in zip(members, ref_members))
    assert abs(float(reward) - float(ref_reward)) < 2e-3 * max(1.0, abs(float(ref_reward))), (float(reward), float(ref_reward))


def _cond_embedder(device="cpu"):
    """vista_b200.conditioner.VideoPredictionEmbedderWithEncoder built from the reference's own YAML shape
    (vista.yaml:68-96 with the two `target:` strings changed), loaded through the reference checkpoint key layout."""
    from oracle.make_golden import cond_embedder_inputs
    from vista_b200.conditioner import VideoPredictionEmbedderWithEncoder
    cfg = spec.encoder_preset("tiny")
    sd = synth.synth_state_dict(spec.encoder_param_specs(cfg), seed=3)
    dd = dict(attn_type="vanilla-xformers", double_z=True, z_channels=cfg.z_channels, resolution=256, in_channels=cfg.in_channels,
              out_ch=3, ch=cfg.ch, ch_mult=list(cfg.ch_mult), num_res_blocks=cfg.num_res_blocks, attn_resolutions=[], dropout=0.0)
    emb = VideoPredictionEmbedderWithEncoder(
        n_cond_frames=1, n_copies=2, is_ae=True, scale_factor=0.5, disable_encoder_autocast=True, en_and_decode_n_samples_a_time=2,
        encoder_config={"target": "vista_b200.conditioner.AutoencoderKLModeOnly",
                        "params": {"embed_dim": cfg.z_channels, "monitor": "val/rec_loss", "ddconfig": dd,
                                   "loss_config": {"target": "torch.nn.Identity"}}})
    x, qw, qb = cond_embedder_inputs(cfg, 32, 64, 3)
    ck = {"encoder.encoder." + k: torch.from_numpy(v) for k, v in sd.items()}
    ck.update({"encoder.quant_conv.weight": torch.from_numpy(qw), "encoder.quant_conv.bias": torch.from_numpy(qb),
               "encoder.decoder.conv_in.weight": torch.zeros(1), "encoder.post_quant_conv.weight": torch.zeros(1)})
    missing, unexpected = emb.load_state_dict(ck, strict=False)          # sample_utils.py:72 loads with strict=False
    assert not missing and sorted(unexpected) == ["encoder.decoder.conv_in.weight", "encoder.post_quant_conv.weight"]
    return emb.to(device), torch.from_numpy(x).to(device)


def test_cond_frames_embedder_on_emulated_ops_matches_reference(monkeypatch):
    from helpers import golden
    from vista_b200 import conditioner as cmod
    from vista_b200 import vae as vae_mod
    emb, x = _cond_embedder()
    monkeypatch.setattr(cmod.AutoencoderKLModeOnly, "runtime", lambda self, device: self.__dict__.setdefault(
        "_rt_cpu", vae_mod.EncoderRuntime(self.encoder.b200_config, self.encoder.state_dict(), "cpu",
                                          post=(self.get_parameter("quant_conv.weight").detach().float().flatten(1),
                                                self.get_parameter("quant_conv.bias").detach().float()))))
    with patched_ops(), torch.no_grad():
        out = emb(x)
        emb.skip_encode = True
        assert emb(x) is x                         # latents pass through (encoders/modules.py:470-471)
    ref = torch.from_numpy(golden("cond_embedder_tiny")["out"])
    assert out.shape == ref.shape and rel_l2(out, ref) < 5e-3, rel_l2(out, ref)


def _ensemble_worker(rank, world, port, q):
    import os
    import types
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_ops import patched_ops as patched
        from helpers import to_t as tt, unet_weights
        from vista_b200 import fused as fused_mod
        from vista_b200 import synth as sy
        from vista_b200.diffusion import Denoiser, EulerEDMSampler
        from vista_b200.modules import B200Wrapper, VideoUNet
        from vista_b200.rollout import sample_ensemble
        fused_mod.USE_GRAPH = False
        cfg, sd = unet_weights("tiny")
        unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                         num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                         channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                         context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                         use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                         use_linear_in_transformer=True, action_control=True)
        unet.load_state_dict(tt(sd), strict=True)
        T, h, w, steps, K = 25, 8, 16, 2, 3
        net = B200Wrapper(unet)
        net._require_cuda = unet._require_cuda = lambda device: None
        eng = types.SimpleNamespace(
            model=net, denoiser=Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=T), num_frames=T,
            sampler=EulerEDMSampler(num_steps=steps, device="cpu", s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, verbose=False,
                                    discretization_config={"target": "vista_b200.diffusion.EDMDiscretization",
                                                           "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}},
                                    guider_config={"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 2.5}}))
        c, uc = sy.synth_conditioning(7, T, h, w, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
        _, z, _ = sy.synth_latents(7, T, h, w)
        td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
        noises = [torch.from_numpy(sy.normal(60 + i, "ens.noise", (T, 4, h, w), std=1.0)) for i in range(K)]
        with patched(), torch.no_grad():
            reward, members = sample_ensemble(eng, td(c), td(uc), torch.from_numpy(z), K, noises=noises, distributed=True)
            reward1, members1 = (sample_ensemble(eng, td(c), td(uc), torch.from_numpy(z), K, noises=noises) if rank == 0 else (reward, members))
        q.put((rank, float(reward), [m.numpy() for m in members], float(reward1), [m.numpy() for m in members1]))
    finally:
        dist.destroy_process_group()


def test_ensemble_members_dealt_over_two_ranks_on_emulated_ops():
    """reward path (reward_utils.py:318-337) as replicas: member k sampled by rank k % 2 and broadcast; both ranks end with the
    same members and reward, equal to the single-rank ensemble."""
    import os
    import numpy as np
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36500 + os.getpid() % 2000
    procs = [ctx.Process(target=_ensemble_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, r0, m0, r0s, m0s), (_, r1, m1, _, _) = res
    assert r0 == r1 and all(np.array_equal(a, b) for a, b in zip(m0, m1))
    assert r0 == r0s and all(np.array_equal(a, b) for a, b in zip(m0, m0s)), "distributed ensemble differs from the single-rank one"


def _peer_sharded_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    win = None
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_ops import patched_ops as patched
        from fake_peer import FakePeerWindow
        from helpers import to_t as tt, unet_weights
        from vista_b200 import fused as fused_mod
        from vista_b200 import synth as sy
        from vista_b200.diffusion import B200Denoiser, Denoiser, EulerEDMSampler
        from vista_b200.modules import B200Wrapper, VideoUNet
        fused_mod.USE_GRAPH = False                        # the emulated kernels are host code: no CUDA graph to capture
        cfg, sd = unet_weights("tiny")
        unet = VideoUNet(in_channels=cfg.in_channels, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                         num_res_blocks=cfg.num_res_blocks, attention_resolutions=list(cfg.attention_resolutions),
                         channel_mult=list(cfg.channel_mult), num_head_channels=64, num_classes="sequential",
                         context_dim=cfg.context_dim, adm_in_channels=cfg.adm_in_channels, extra_ff_mix_layer=True,
                         use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
                         use_linear_in_transformer=True, action_control=True)
        unet.load_state_dict(tt(sd), strict=True)
        T, h, w, steps = 25, 8, 16, 4
        c, uc = sy.synth_conditioning(7, T, h, w, trajectory=True, context_dim=cfg.context_dim, adm=cfg.adm_in_channels)
        noise, z, mask = sy.synth_latents(7, T, h, w)
        td = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
        den = Denoiser({"target": "vista_b200.diffusion.VScalingWithEDMcNoise"}, num_frames=T)
        smp = EulerEDMSampler(num_steps=steps, device="cpu", s_churn=0.0, s_tmin=0.0, s_tmax=999.0, s_noise=1.0, verbose=False,
                              discretization_config={"target": "vista_b200.diffusion.EDMDiscretization",
                                                     "params": {"sigma_min": 0.002, "sigma_max": 700.0, "rho": 7.0}},
                              guider_config={"target": "vista_b200.diffusion.VanillaCFG", "params": {"scale": 2.5}})
        net = B200Wrapper(unet)
        net._require_cuda = lambda device: None
        net.enable_frame_sharding(cfg_split=True)

        def peer_window(T_, h_, w_, mc, device):           # same size rule as modules.peer_window, windows in /dev/shm
            nonlocal win
            if win is None:
                fw = net._frame_world
                tp = -(-T_ // fw)
                ext, kv, nf = (tp + 2) * h_ * w_ * mc * 2, fw * tp * h_ * w_ * 2 * mc * 2, 2 * 2 * tp * h_ * w_ * 8 * 4
                win = FakePeerWindow(net.world_group, (4 * ext + kv + nf + (16 << 20)) if fw > 1 else (nf + (4 << 20)), str(port))
            return win
        net.peer_window = peer_window
        with patched(), torch.no_grad():
            out = smp(B200Denoiser(den, net), torch.from_numpy(noise).clone(), td(c), uc=td(uc),
                      cond_frame=torch.from_numpy(z), cond_mask=torch.from_numpy(mask))
            # a second sample on the same state: counters, flags and buffers carry over (what a graph replay relies on)
            out2 = smp(B200Denoiser(den, net), torch.from_numpy(noise).clone(), td(c), uc=td(uc),
                       cond_frame=torch.from_numpy(z), cond_mask=torch.from_numpy(mask))
        rt = net._runtime
        st = next(iter(rt._loop_states.values()))
        q.put((rank, out.numpy(), out2.numpy(), st.pair_peer is not None, getattr(rt, "win", None) is not None or net._frame_world == 1,
               int(rt.t1 - rt.t0)))
        dist.barrier()
    finally:
        if win is not None:
            win.close()
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_peer_memory_sharded_sampler_on_emulated_windows(world):
    """The NVLink peer-memory path of the sharded step with the windows emulated in /dev/shm (tests/fake_peer.py) and the
    three peer kernels restated over raw addresses: 2 ranks (CFG pair exchange only), 4 ranks (2 frame shards per half),
    8 ranks (4 frame shards per half: interior shards with two halo neighbours, 3 K|V peers) — the BASELINE config-5 layout.
    Validates the window layout / remote addresses / flag and counter protocol of vista_b200/sharded.py + fused.py: every rank
    must end with the same latent, equal to the REAL reference's 4-step sample within the fp16 tolerance, twice in a row."""
    import os
    import numpy as np
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 37500 + (os.getpid() + 11 * world) % 2000
    procs = [ctx.Process(target=_peer_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=600) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    ref = torch.from_numpy(golden("sampler_tiny_cfg")["sample"])
    fw = world // 2
    frames = [r[5] for r in res]
    assert sum(frames[:fw]) == 25 and frames[:fw] == frames[fw:]
    for rank, out, out2, pair_peer, has_win, _ in res:
        assert pair_peer and has_win, "the peer-memory path must have been taken"
        assert np.array_equal(out, res[0][1]), f"rank {rank} holds a different latent"
        assert np.array_equal(out, out2), "second sample on the same state differs"
        r = rel_l2(torch.from_numpy(out), ref)
        assert r < 5e-3, (rank, r)
