"""The shadow harness of tests/shadow.py without a GPU: the tiny native engine on the CPU twins runs through condition, a
2M sample, an action-guided step, a decode, a session step and a score with every key held; the harness covers every
ops entry point that launches a kernel; its key follows the launcher's own choices; and a defect planted in a twin
(never in a kernel) fails the run with a message that names the op and the key."""
import pytest
import torch
import torch.nn.functional as F

import fake_ops
import seam_fakes as sf
import shadow
from action_fake_ops import patched_action_ops
from oracle import make_golden_cond as mgc
from test_action_cfg_cpu import A, action_sampler, triangle_cfg, with_guider
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs
from vista_b200 import ops


@pytest.fixture(scope="module")
def eng():
    e = native_engine(steps=3)
    e.en_and_decode_n_samples_a_time = 14
    return e


@pytest.fixture(autouse=True)
def eager(monkeypatch):
    from vista_b200 import fused
    monkeypatch.setattr(fused, "USE_GRAPH", False)


def test_every_key_passes_on_the_twins(eng, monkeypatch):
    vd, z, noises = inputs(2, "shadow")
    euler = eng.sampler                    # Euler under the triangle guider: the session's step and score
    with patched_action_ops(), torch.no_grad(), shadow.Shadow(random_rows=256) as sh:
        c, uc = eng.condition({**vd, **A}, sf.T, mgc.UC_KEYS)
        monkeypatch.setattr(eng, "sampler", with_guider(eng.sampler, "dpm", triangle_cfg(sf.T)))
        sample = eng.sample(c, uc=uc, N=sf.T, shape=tuple(z.shape[1:]), noise=noises[0].clone(), cond_frame=z)
        monkeypatch.setattr(eng, "sampler", action_sampler(eng, "euler", steps=1))
        eng.sample(c, uc=uc, N=sf.T, shape=tuple(z.shape[1:]), noise=noises[0].clone(), cond_frame=z)
        eng.decode_first_stage_u8(sample)
        monkeypatch.setattr(eng, "sampler", euler)
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
        sess.step(noise=noises[1])
        sess.score([None], ensemble_size=2, num_steps=1)
    print(sh.report())
    sh.assert_ok()
    fams = sh.families()
    want = {"gemm", "groupnorm", "groupnorm_from_partials", "groupnorm_apply", "layernorm", "attention_spatial",
            "attention_temporal", "attention_d80", "softmax_rows", "conv3x3_small_cin", "im2col_s2", "im2col_s2_asym",
            "upsample2x", "nchw_to_tokens", "tokens_to_nchw", "time_mix_small_u8", "sampler_prepare",
            "sampler_update_2m", "sampler_update_action", "sampler_update", "rollout_advance", "ensemble_reward",
            "timestep_embedding", "blend_emb", "sinusoid_embed", "clip_preprocess"}
    missing = {op for op in want if fams.get(op, (0, 0))[1] == 0}
    assert not missing, f"families with no checked key: {sorted(missing)}"
    assert fams["sampler_update_2m"][1] >= 2, "the 2M update's first- and second-order rows"


def test_checkers_and_exemptions_cover_every_kernel_entry_point():
    entry = shadow.kernel_entry_points()
    assert len(entry) >= 30, sorted(entry)
    assert not set(shadow.CHECKERS) & set(shadow.SHADOW_EXEMPT)
    assert entry == set(shadow.CHECKERS) | set(shadow.SHADOW_EXEMPT), \
        (sorted(entry - set(shadow.CHECKERS) - set(shadow.SHADOW_EXEMPT)), sorted(set(shadow.CHECKERS) - entry))


def test_an_unchecked_entry_point_fails_by_name(monkeypatch):
    monkeypatch.delitem(shadow.CHECKERS, "layernorm")
    with pytest.raises(AssertionError, match="ops.layernorm launches a kernel and has no checker"):
        with shadow.Shadow():
            ops.layernorm(torch.zeros(2, 8, dtype=torch.float16), torch.zeros(2, 8, dtype=torch.float16),
                          torch.ones(8), torch.zeros(8))


def test_an_uncalled_exempt_entry_point_fails_when_called():
    """An entry point exempted because nothing calls it is wrapped all the same: a new caller fails the run by name."""
    assert shadow.UNCALLED <= set(shadow.SHADOW_EXEMPT)
    with pytest.raises(AssertionError, match="ops.conv3x3_small_cout launches a kernel and is exempt only because"):
        with shadow.Shadow():
            ops.conv3x3_small_cout(None, None, None, None, 1, 1, 1)


def _gemm_args(geom=(16, 8, 1), N=96, act=0, stats=False, tile_n=None, taps=ops.TAPS_3X3):
    M = geom[0] * geom[1] * geom[2]
    a = torch.zeros(M, 64, dtype=torch.float16)
    return dict(a=a, w=torch.zeros(N, len(taps) * 64, dtype=torch.float16),
                out=torch.zeros(M, N // 2 if act == 2 else N), taps=taps, geom=geom, bias=None, rowvec=None, rv_div=1,
                rv_mod=1, res1=None, s_res1=1.0, res2=None, s_res2=1.0, s_acc=1.0, act=act, tile_n=tile_n, cin=None,
                stats=torch.zeros(-(-M // 128) * 4, N, 2) if stats else None, h_pad=0, upsample=False)


def differing_fields(k0, k1):
    assert len(k0) == len(k1), (k0, k1)
    names = shadow.GEMM_KEY_FIELDS + tuple(f"flag{i}" for i in range(len(k0) - len(shadow.GEMM_KEY_FIELDS)))
    return {n for n, a, b in zip(names, k0, k1) if a != b}


def test_key_follows_the_launcher():
    """The key's tile width and box fields hold what the launcher derives, and a pair of calls that differ only in a
    derived value (or in the tap offsets) differ only in that field."""
    f = shadow.gemm_field
    # the tile width: the default is pick_tile_n's; an explicit other width changes that field alone
    k0 = shadow._gemm_key(_gemm_args(N=96))
    assert f(k0, "tile_n") == ops.pick_tile_n(96)
    assert differing_fields(k0, shadow._gemm_key(_gemm_args(N=96, tile_n=64))) == {"tile_n"}
    assert k0 == shadow._gemm_key(_gemm_args(N=96, tile_n=ops.pick_tile_n(96)))
    # GEGLU: at N = 640 pick_tile_n picks 128 for GEGLU (a multiple of 64 dividing N), 224 otherwise
    geglu, plain = shadow._gemm_key(_gemm_args(N=640, act=2)), shadow._gemm_key(_gemm_args(N=640))
    assert f(geglu, "tile_n") == ops.pick_tile_n(640, True) == 128 and f(plain, "tile_n") == ops.pick_tile_n(640) == 224
    # the box: equal M, N and K at two geometries whose pick_box boxes differ; with fused statistics, stats_box's box
    g1, g2 = (32, 8, 2), (16, 16, 2)
    k1, k2 = shadow._gemm_key(_gemm_args(g1)), shadow._gemm_key(_gemm_args(g2))
    assert (f(k1, "rows"), f(k1, "N"), f(k1, "K")) == (f(k2, "rows"), f(k2, "N"), f(k2, "K"))
    assert f(k1, "box") == ops.pick_box(*g1) != f(k2, "box") == ops.pick_box(*g2)
    assert f(shadow._gemm_key(_gemm_args(g1, stats=True)), "box") == ops.stats_box(*g1) != ops.pick_box(*g1)
    # the tap offsets: three taps along W against three along frames / rows, same K
    along_w = [(0, -1), (0, 0), (0, 1)]
    assert differing_fields(shadow._gemm_key(_gemm_args(taps=along_w)),
                            shadow._gemm_key(_gemm_args(taps=ops.TAPS_T3))) == {"taps"}


# ==================================================================================================================
# Planted defects: each twin below is wrong in one way; the harness must fail naming the op and the key
# ==================================================================================================================
def run_planted(monkeypatch, op, defective, *args, **kwargs):
    monkeypatch.setattr(ops, op, defective)
    with shadow.Shadow(random_rows=64) as sh:
        getattr(ops, op)(*args, **kwargs)
    assert len(sh.failures) == 1, sh.failures
    (key, msg), = sh.failures.items()
    assert key[0] == op and msg.startswith(f"{op} key {key[1:]}"), msg
    with pytest.raises(AssertionError, match=op):
        sh.assert_ok()
    return msg


def rnd(*shape, seed=0, dtype=torch.float16, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dtype)


def test_planted_gemm_bias_dropped_on_last_n_tile(monkeypatch):
    N = 600
    tn = ops.pick_tile_n(N)
    n0 = (-(-N // tn) - 1) * tn

    def bad(a, w, out, **kw):
        fake_ops.gemm(a, w, out, **kw)
        out[:, n0:] = (out[:, n0:].float() - kw["bias"][n0:]).to(out.dtype)
        return out
    a, w, bias = rnd(300, 64, seed=1), rnd(N, 64, seed=2, scale=0.125), rnd(N, seed=3, dtype=torch.float32)
    run_planted(monkeypatch, "gemm", bad, a, w, torch.empty(300, N, dtype=torch.float16), bias=bias)


def test_planted_gemm_last_row_two_ulp(monkeypatch):
    def bad(a, w, out, **kw):
        fake_ops.gemm(a, w, out, **kw)
        out[-1] = (out[-1].view(torch.int16) + 2).view(torch.float16)
        return out
    a, w = rnd(300, 64, seed=4), rnd(96, 64, seed=5, scale=0.125)
    run_planted(monkeypatch, "gemm", bad, a, w, torch.empty(300, 96, dtype=torch.float16))


def test_planted_conv_border_column_wrong_tap(monkeypatch):
    NB, H, W, cin, cout = 2, 6, 9, 4, 32

    def bad(x8, cin, w, bias, out, NB, H, W):
        fake_ops.conv3x3_small_cin(x8, cin, w, bias, out, NB, H, W)
        img = x8[:, :cin].float().reshape(NB, H, W, cin).permute(0, 3, 1, 2)
        o = F.conv2d(F.pad(img, (1, 1, 1, 1), mode="replicate"), w, bias)          # the left tap reads column 0 again
        out.reshape(NB, H, W, -1)[:, :, 0] = o.permute(0, 2, 3, 1)[:, :, 0].to(out.dtype)
        return out
    x8 = rnd(NB * H * W, 8, seed=6)
    w, b = rnd(cout, cin, 3, 3, seed=7, dtype=torch.float32, scale=0.2), rnd(cout, seed=8, dtype=torch.float32)
    run_planted(monkeypatch, "conv3x3_small_cin", bad, x8, cin, w, b, torch.empty(NB * H * W, cout, dtype=torch.float16),
                NB, H, W)


def test_planted_groupnorm_stats_without_last_chunk(monkeypatch):
    from vista_b200 import lib
    frames, tpf, C, groups = 2, 300, 64, 32
    chunk = lib.load().b200v_groupnorm_chunk_for(frames, tpf)

    def bad(x, y, frames, tokens_per_frame, gamma, beta, eps, silu, stats=None, frames_per_stat=1, groups=32, ws=None):
        keep = (tokens_per_frame - 1) // chunk * chunk                      # the last chunk of every frame left out
        xs = x[:, :C].float().reshape(frames, tokens_per_frame, groups, C // groups)
        mean = xs[:, :keep].mean(dim=(1, 3), keepdim=True)
        var = xs[:, :keep].var(dim=(1, 3), unbiased=False, keepdim=True)
        o = ((xs - mean) * torch.rsqrt(var + eps)).reshape(-1, C) * gamma + beta
        y.copy_(F.silu(o).to(y.dtype) if silu else o.to(y.dtype))
        return y
    ramp = torch.linspace(0, 3, tpf).repeat(frames)[:, None]
    x = (rnd(frames * tpf, C, seed=9, dtype=torch.float32) + ramp).half()
    gamma, beta = torch.ones(C), torch.zeros(C)
    run_planted(monkeypatch, "groupnorm", bad, x, torch.empty_like(x), frames, tpf, gamma, beta, 1e-5, True)


def test_planted_spatial_attention_key_mask_one_past_seq(monkeypatch):
    frames, seq, heads = 3, 50, 2

    def bad(q, k, v, out, frames, seq, heads, impl=None):
        sp = lambda t: t.float().reshape(frames, seq, heads, 64).permute(0, 2, 1, 3)
        nxt = lambda t: torch.cat([t[1:, :, :1], torch.zeros_like(t[:1, :, :1])], 0)     # key seq: the next frame's first
        kk, vv = sp(k), sp(v)
        o = F.scaled_dot_product_attention(sp(q), torch.cat([kk, nxt(kk)], 2), torch.cat([vv, nxt(vv)], 2))
        out.copy_(o.permute(0, 2, 1, 3).reshape(frames * seq, heads * 64).to(out.dtype))
        return out
    qkv = rnd(frames * seq, 3 * heads * 64, seed=10)
    C = heads * 64
    run_planted(monkeypatch, "attention_spatial", bad, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:],
                torch.empty(frames * seq, C, dtype=torch.float16), frames, seq, heads)


def test_planted_time_mix_rounds_instead_of_truncating(monkeypatch):
    T, Hh, Ww = 3, 8, 16

    def bad(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0=0, skip_frames=0, keep_f32_from=-1):
        fake_ops.time_mix_small_u8(x, w, bias, out, out_u8, blend, T, HW, Cc, out_frame0, skip_frames, keep_f32_from)
        for t in range(skip_frames, T):
            f = out_frame0 + t
            out_u8[f] = torch.round(255.0 * ((out[f] + 1.0) / 2.0).clamp(0, 1)).to(torch.uint8).permute(1, 2, 0)
        return out_u8
    x = rnd(T * Hh * Ww, 8, seed=11, dtype=torch.float32, scale=0.8)
    w, b = rnd(3, 3, 3, seed=12, dtype=torch.float32, scale=0.5), rnd(3, seed=13, dtype=torch.float32, scale=0.1)
    out = torch.zeros(T, 3, Hh, Ww)
    out8 = torch.zeros(T, Hh, Ww, 3, dtype=torch.uint8)
    run_planted(monkeypatch, "time_mix_small_u8", bad, x, w, b, out, out8, None, T, Hh * Ww, 3)


def test_planted_fused_stats_shifted_by_one_tile(monkeypatch):
    geom, N = (16, 8, 4), 64
    M = geom[0] * geom[1] * geom[2]

    def bad(a, w, out, **kw):
        fake_ops.gemm(a, w, out, **kw)
        s = kw["stats"]
        s[4:] = s[:-4].clone()
        return out
    a, w = rnd(M, 64, seed=14), rnd(N, 9 * 64, seed=15, scale=1 / 24)
    stats = torch.zeros(M // 128 * 4, N, 2)
    run_planted(monkeypatch, "gemm", bad, a, w, torch.empty(M, N, dtype=torch.float16), taps=ops.TAPS_3X3, geom=geom,
                stats=stats)
