"""Conformance of the small kernels of the single-GPU path on the GPU: the case tables, references and bounds of
tests/test_conformance_small_cpu.py run on the kernels, with the twin of tests/fake_ops.py beside each on the same inputs
(where the case is small enough for the CPU), plus the production shapes and a profiler gate: every kernel the tiny native
engine launches on one GPU must be held by a conformance test."""
import re

import pytest
import torch

import clip_fake_ops
import fake_ops
from test_conformance_cpu import CPU, assert_conform
from test_conformance_small_cpu import (CONV_CASES, D80_CASES, D80_LARGE_QK, IM2COL_S2_CASES, KERNEL_TESTS,
                                        LAUNCHED_NOT_HELD, LAYOUT_CASES, NONFINITE_PAD, NUM_STEPS, REWARD_CASES,
                                        SAMPLER_CASES, SAMPLER_STEPS, TMIX_CASES, UPSAMPLE_CASES, blend_emb_combos,
                                        check_blend_emb, check_conv_case, check_conv_ignores_nonfinite_pad, check_d80,
                                        check_decode_sequence, check_im2col_s2, check_layout, check_reward,
                                        check_rollout_advance, check_sampler_step, check_session_round, check_temb,
                                        check_tmix_boundaries, check_tmix_case, check_trajectory, check_upsample2x,
                                        conv_case_id, conv_eps, conv_reference, identical_members, make_conv_inputs,
                                        randn, reward_members, run_trajectory, sampler_case_id, temb_cases,
                                        tmix_case_id, trajectory_inputs, trajectory_reference)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from vista_b200 import lib, ops as _ops
    lib.load()
    return _ops


def dev():
    return torch.device("cuda:0")


# ==================================================================================================================
# A. Sampler step
# ==================================================================================================================
@pytest.mark.parametrize("step", SAMPLER_STEPS)
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=sampler_case_id)
def test_sampler_step(ops, case, step):
    """prepare -> update at the first, a middle and the last step of the 50-step schedule (sigma' = 0), every argument
    variant: unet_in in the padded 64-column rows (NaN pad columns must survive), net_out rows of 8 with NaN in columns
    4..7, concat_u / concat_c given or NULL, no mask / the initial mask / the rollout mask, constant and triangle scales,
    token counts that are not a multiple of the block.  A wrong row stride, a concat column from the wrong half, c_skip
    or c_out from the wrong sigma, a scale from the wrong frame or a missed re-imposition is an O(1) error; the twin runs
    the same case on the CPU."""
    check_sampler_step(case, step, ops.sampler_prepare, ops.sampler_update, dev())
    if case[1] * case[2] <= 128:
        check_sampler_step(case, step, fake_ops.sampler_prepare, fake_ops.sampler_update, CPU)


def test_sampler_trajectory_and_graph_replay(ops):
    """50 prepare -> update steps at 25 x 72 x 128 (a fixed network output each step, the rollout mask, triangle scales)
    against the fp64 trajectory, within the per-step bound accumulated through the affine update.  Then the same 50
    steps replayed from one captured CUDA graph, as fused.py runs them: bit-equal to the eager launches, and step_idx
    (advanced on the device by step_inc_kernel) ends at 50."""
    d = trajectory_inputs(25, 72, 128, dev())
    ref, bound = trajectory_reference(d)
    x, idx = run_trajectory(d, ops.sampler_prepare, ops.sampler_update)
    torch.cuda.synchronize()
    assert int(idx[0]) == NUM_STEPS
    check_trajectory(x, ref, bound, "kernels")
    T, h, w = d["T"], d["h"], d["w"]
    xg = d["x"].clone()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.sampler_prepare(xg, d["cond_frame"], d["mask"], d["concat_u"], d["concat_c"], d["sigmas"], step, d["unet_in"],
                            d["c_noise"], T, h, w)
        ops.sampler_update(xg, d["net"], d["cond_frame"], d["mask"], d["scales"], d["sigmas"], step, NUM_STEPS, T, h, w)
    assert int(step[0]) == 0, "capture must not run the kernels"
    for _ in range(NUM_STEPS):
        g.replay()
    torch.cuda.synchronize()
    assert int(step[0]) == NUM_STEPS
    assert torch.equal(xg, x), "graph replay differs from the eager launches"


# ==================================================================================================================
# B. Thin direct convolution
# ==================================================================================================================
@pytest.mark.parametrize("case", CONV_CASES, ids=conv_case_id)
def test_conv3x3_small_cin_edges(ops, case):
    """Token counts that are not a multiple of the 32-token block, H = 1, W = 1, cout 1 / 100 / 256 / 257 / 512 (the
    per-thread output loop's second pass), a column-slice output between NaN sentinel columns, bias NULL; channels >= cin
    hold random values that must be ignored.  A tap at the wrong border, a second pass that skips or repeats a channel,
    or a store without the output stride is an O(1) error."""
    check_conv_case(case, ops.conv3x3_small_cin, dev())
    check_conv_case(case, fake_ops.conv3x3_small_cin, CPU)


def _border_rows(NB, H, W, device, n_random=4096):
    """Every border row / column of the first, middle and last image, the last 32-token block, and random tokens."""
    ar = torch.arange
    idx = lambda b, h, w: ((b * H + h) * W + w).reshape(-1)
    t = torch.tensor
    sets = [torch.randperm(NB * H * W, generator=torch.Generator().manual_seed(6))[:n_random]]
    for b in (0, NB // 2, NB - 1):
        sets += [idx(t(b), t(0), ar(W)), idx(t(b), t(H - 1), ar(W)), idx(t(b), ar(H), t(0)), idx(t(b), ar(H), t(W - 1))]
    M = NB * H * W
    sets.append(ar(M - 32 - M % 32, M))
    return torch.unique(torch.cat(sets)).to(device)


@pytest.mark.parametrize("name,NB,H,W,cin,cout,full", [("decoder conv_in", 14, 72, 128, 4, 512, True),
                                                      ("encoder conv_in", 1, 576, 1024, 3, 128, False),
                                                      ("unet conv_in", 50, 72, 128, 8, 320, False)])
def test_conv3x3_small_cin_production(ops, name, NB, H, W, cin, cout, full):
    """The three production geometries: the decoder's 4 -> 512 on a 14-frame chunk (every output), the encoder's 3 -> 128
    at 576 x 1024 and the UNet's 8 -> 320 on 50 frames, the last two on every border row and column of the first,
    middle and last image, the last block and 4096 random tokens."""
    x8, w, b, _, out = make_conv_inputs(NB, H, W, cin, cout, True, False, dev(), 700 + cin)
    ops.conv3x3_small_cin(x8, cin, w, b, out, NB, H, W)
    torch.cuda.synchronize()
    rows = None if full else _border_rows(NB, H, W, dev())
    ref, mag = conv_reference(x8, w, b, NB, H, W, rows=rows)
    assert_conform(out if full else out[rows], ref, mag, conv_eps(cin), "gemm", name)


@pytest.mark.parametrize("fill", NONFINITE_PAD)
def test_conv3x3_small_cin_ignores_nonfinite_pad_channels(ops, fill):
    """NaN / Inf in channels cin..7 (cin 1, 3 and 4): the output is bit-equal to the output with zeros there.  A kernel
    that stages those channels and multiplies them by zero weights returns NaN (NaN * 0 = NaN, Inf * 0 = NaN)."""
    for cin in (1, 3, 4):
        check_conv_ignores_nonfinite_pad(ops.conv3x3_small_cin, dev(), cin, fill)
        check_conv_ignores_nonfinite_pad(fake_ops.conv3x3_small_cin, CPU, cin, fill)


def test_conv3x3_small_cin_rejects_strided_input(ops):
    """The kernel reads x as rows of 8 halves: ops.conv3x3_small_cin refuses any other row stride (the padded 64-column
    input rows, a column slice) instead of misreading it, and a non-fp16 input."""
    from vista_b200.unet import padded_input_rows
    NB, H, W = 1, 4, 8
    w = randn((16, 4, 3, 3), 1, dev())
    out = torch.empty(NB * H * W, 16, dtype=torch.float16, device=dev())
    for x in (padded_input_rows(NB * H * W, dev()), torch.zeros(NB * H * W, 16, dtype=torch.float16, device=dev())[:, 8:]):
        assert x.stride(0) != 8
        with pytest.raises(AssertionError):
            ops.conv3x3_small_cin(x, 4, w, None, out, NB, H, W)
    with pytest.raises(AssertionError):
        ops.conv3x3_small_cin(torch.zeros(NB * H * W, 8, device=dev()), 4, w, None, out, NB, H, W)


# ==================================================================================================================
# C. Decoder output
# ==================================================================================================================
@pytest.mark.parametrize("case", TMIX_CASES, ids=tmix_case_id)
def test_time_mix_cases(ops, case):
    """T = 1 / 2 / 5 / 14, HW = 35, skipped and blended frames, bias NULL, fp32 kept from a frame on: both kernels against
    the fp64 mix (blend averaging included), the bytes within the fp32 bound of the fp64 output path and equal to the
    output path of the fp32 frames, nothing written outside its frames.  A mirrored tap, a dropped 0.5 or a rounding
    instead of a truncation is caught; the twin runs the same case."""
    check_tmix_case(case, ops.time_mix_small, ops.time_mix_small_u8, dev())
    check_tmix_case(case, fake_ops.time_mix_small, fake_ops.time_mix_small_u8, CPU)


def test_time_mix_boundaries(ops):
    """Frame values at and beyond +-1 and on every truncation boundary k / 255 (and their fp32 neighbours)."""
    check_tmix_boundaries(ops.time_mix_small, ops.time_mix_small_u8, dev())


def test_time_mix_decode_and_session_chunks(ops):
    """decode_first_stage(u8=True)'s chunk calls at T = 25 in order (40 x 72 frames), and RolloutSession's two chunks of a
    later round at 576 x 1024 (decoder rows of stride 8, NaN in columns 3..7): each call against the fp32 state the
    previous call left, with the fp32 frames below keep_f32_from untouched."""
    check_decode_sequence(ops.time_mix_small, ops.time_mix_small_u8, 40, 72, dev())
    check_session_round(ops.time_mix_small, ops.time_mix_small_u8, 576, 1024, dev())


# ==================================================================================================================
# D. Rollout glue
# ==================================================================================================================
@pytest.mark.parametrize("E", [37, 4 * 72 * 128])
def test_rollout_advance(ops, E):
    """n_cond 0 / 1 / 3 / T, src_frame0 0 / n_cond / T, destinations r (T - n) for rounds 0..3, z0 with and without
    filled, sentinels in every row of samples_z it must not write; 4 x 72 x 128 runs the grid-stride loop past the
    8-blocks-per-SM cap.  Exact."""
    check_rollout_advance(ops.rollout_advance, E, dev())
    if E == 37:
        check_rollout_advance(fake_ops.rollout_advance, E, CPU)


@pytest.mark.parametrize("K,n,offset", REWARD_CASES)
def test_ensemble_reward(ops, K, n, offset):
    """K 2 / 3 / 5 / 64, n 1 / 255 / 256 / 257 (below, at and past one block), the production n = 25 x 4 x 72 x 128 and one
    where every thread of the capped grid loops; members with a common offset of 30 standard deviations (the
    mean-subtraction cancellation).  Against the fp64 reward_utils arithmetic under the bound of reward_reference."""
    members = reward_members(K, n, offset, dev(), 1100 + K)
    out = ops.ensemble_reward(members)
    torch.cuda.synchronize()
    check_reward(out.cpu(), members, f"kernel K {K} n {n} offset {offset}")
    if K * n <= 10 ** 6:
        cm = [m.cpu() for m in members]
        check_reward(fake_ops.ensemble_reward(cm), cm, f"twin K {K} n {n} offset {offset}")


@pytest.mark.parametrize("K", [2, 3, 5, 64])
def test_ensemble_reward_identical_members(ops, K):
    """Identical members (values whose partial sums are exact): exactly [0, 1]."""
    out = ops.ensemble_reward(identical_members(K, 70000, dev()))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), torch.tensor([0.0, 1.0])), out


def test_ensemble_reward_back_to_back(ops):
    """Calls with different n (different grids) issued back to back on one workspace are bit-equal to the same calls
    made one at a time: the last block's ticket must be back at zero after every launch."""
    shapes = [(5, 25 * 4 * 72 * 128), (3, 257), (2, 1), (64, 4099), (5, 25 * 4 * 72 * 128)]
    sets = [reward_members(K, n, 0, dev(), 1300 + i) for i, (K, n) in enumerate(shapes)]
    alone = []
    for m in sets:
        alone.append(ops.ensemble_reward(m).clone())
        torch.cuda.synchronize()
    together = [ops.ensemble_reward(m) for m in sets]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(alone, together)):
        assert torch.equal(a, b), (shapes[i], a, b)


# ==================================================================================================================
# E. Embedding helpers and layout converters
# ==================================================================================================================
@pytest.mark.parametrize("name,t,dim", temb_cases(), ids=[c[0] for c in temb_cases()])
def test_timestep_embedding(ops, name, t, dim):
    """c_noise over the 50-step schedule at 320, frame indices 0..24 at 320 / 640 / 1280, into a strided output between
    NaN sentinels: swapped cos / sin halves or a frequency off by one index is an O(1) error."""
    check_temb(ops.timestep_embedding, name, t, dim, dev())
    check_temb(fake_ops.timestep_embedding, name, t, dim, CPU)


@pytest.mark.parametrize("combo", blend_emb_combos())
def test_blend_emb(ops, combo):
    """Every combination of the NULL arguments the ABI accepts (e_cond, label, mask, emb, silu_emb)."""
    check_blend_emb(ops.blend_emb, combo, dev())
    check_blend_emb(fake_ops.blend_emb, combo, CPU)


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_converters(ops, case):
    """nchw_to_tokens into token rows (50 x 4 x 72 x 128 into the 64-column padded layout: columns >= C untouched) and
    tokens_to_nchw from fp16 and fp32 rows, odd sizes.  Exact."""
    check_layout(ops.nchw_to_tokens, ops.tokens_to_nchw, case, dev())
    if case[0] * case[2] * case[3] <= 10 ** 4:
        check_layout(fake_ops.nchw_to_tokens, fake_ops.tokens_to_nchw, case, CPU)


@pytest.mark.parametrize("case", IM2COL_S2_CASES)
def test_im2col_s2(ops, case):
    """The UNet Downsample gather, odd H and W (the bottom / right padding row only for odd sizes), strided x.  Exact."""
    check_im2col_s2(ops.im2col_s2, case, dev())
    check_im2col_s2(fake_ops.im2col_s2, case, CPU)


@pytest.mark.parametrize("case", UPSAMPLE_CASES)
def test_upsample2x(ops, case):
    """Nearest 2x with row strides != C on both sides, sentinel columns untouched.  Exact."""
    check_upsample2x(ops.upsample2x, case, dev())
    check_upsample2x(fake_ops.upsample2x, case, CPU)


# ==================================================================================================================
# F. CLIP attention
# ==================================================================================================================
@pytest.mark.parametrize("batch,seq,heads", D80_CASES)
def test_attention_d80(ops, batch, seq, heads):
    """seq 1 / 2 / 63 / 64 / 65 / 128 / 129 / 257, 1 and 16 heads, 1 and 25 images; q / k / v column blocks of the fused
    in-projection output (padded row stride), out between NaN sentinel columns.  Held to the spatial attention's rule
    (P rounded unnormalised, the absolute term divided by the fp64 row sum): a key mask off by one admits a zero key, a
    wrong head or image offset mixes rows."""
    check_d80(ops.attention_d80, batch, seq, heads, dev())
    if batch * seq * heads <= 4096:
        check_d80(clip_fake_ops.attention_d80, batch, seq, heads, CPU, name="d80 twin")


def test_attention_d80_identical_keys_and_large_logits(ops):
    """Identical keys (every weight equal: a rescale applied twice or a missing normalisation breaks the mean of V), and
    logits of about +-30 (the running maximum must keep exp in range)."""
    check_d80(ops.attention_d80, 3, 257, 16, dev(), identical_keys=True, name="d80 identical keys")
    check_d80(ops.attention_d80, 3, 257, 16, dev(), qk_scale=D80_LARGE_QK, name="d80 large logits")


# ==================================================================================================================
# G. Every kernel the single-GPU path launches is held by a conformance test
# ==================================================================================================================
def test_launched_kernels_have_conformance_tests(monkeypatch):
    """Under torch.profiler, the tiny native engine's single-GPU path run eagerly: condition, a 2-step sample, the uint8
    decode, a 2-round rollout session, score() with 2 members, encode.  Every vb:: kernel it launches must be in
    KERNEL_TESTS (or be a NOT_HELD kernel checked indirectly), so a kernel added to or re-routed onto the path without a
    conformance test fails here."""
    from torch.profiler import ProfilerActivity, profile
    import seam_fakes as sf
    from oracle import make_golden_cond as mgc
    from test_session_cpu import inputs
    from test_session_gpu import gpu_engine
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    eng = gpu_engine(2)
    vd, z, noises = inputs(2, "conformance_gate")
    z = z.to(dev())
    with profile(activities=[ProfilerActivity.CUDA]) as prof, torch.no_grad():
        c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
        sample = eng.sample(c, cond_frame=z, uc=uc, N=sf.T, shape=tuple(z.shape[1:]), noise=noises[0])
        eng.decode_first_stage_u8(sample)
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        for nz in noises:
            sess.step(noise=nz)
        sess.score([None], ensemble_size=2, num_steps=2)
        eng.encode_first_stage(vd["cond_frames"].to(dev()).float(), sample=False)
        torch.cuda.synchronize()
    launched = set()
    for e in prof.events():
        m = re.search(r"\bvb::(\w+)", e.name)
        if m:
            launched.add(m.group(1))
    print(f"vb:: kernels launched: {sorted(launched)}")
    assert {"sampler_prepare_kernel", "time_mix_small_u8_kernel", "rollout_advance_kernel", "ensemble_reward_kernel",
            "conv3x3_small_cin_kernel", "attn_d80_kernel", "tapgemm_kernel"} <= launched, sorted(launched)
    unheld = launched - set(KERNEL_TESTS) - LAUNCHED_NOT_HELD
    assert not unheld, f"kernels launched without a conformance test: {sorted(unheld)}"
