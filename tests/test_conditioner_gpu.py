"""The native conditioner on the H100: b200v_sinusoid_embed against the reference formula, GeneralConditioner from
configs/inference/vista_b200_native.yaml (tiny sizes) against the REAL reference conditioner's fixture, the exactness of
its work elimination, run-to-run determinism, and a re-conditioned rollout against the same loop on the CPU emulation."""
import pytest
import torch

import seam_fakes as sf
from cond_fake_ops import patched_cond_ops
from helpers import golden, rel_l2
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import _sin, check_against_fixture, condition_case, native_engine

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def eng():
    return native_engine(cpu=False).to(DEV)


def test_sinusoid_embed_matches_formula():
    from vista_b200 import ops
    from vista_b200.conditioner import _freq_table
    g = torch.Generator().manual_seed(0)
    rows = 37
    vals = (torch.rand(rows, 15, generator=g) * 2000 - 1000)
    vals[0, :3] = torch.tensor([1000.0, -1000.0, 127.0])
    freqs, offs = _freq_table([256, 128, 255], DEV)
    out = torch.full((rows, 256 + 8 * 128 + 2 * 255 + 4 * 128 + 3), float("nan"), device=DEV)
    slots = [(0, 1, 256, 0, False, offs[256]), (1, 8, 128, 256, False, offs[128]), (9, 2, 255, 1280, False, offs[255]),
             (0, 4, 128, 1790, True, 0)]
    ops.sinusoid_embed(vals.to(DEV).contiguous(), slots, freqs, out[:, :-3])
    torch.cuda.synchronize()
    got = out.cpu()
    want = torch.cat([_sin(vals[:, :1], 256), _sin(vals[:, 1:9], 128), _sin(vals[:, 9:11], 255), torch.zeros(rows, 512)], 1)
    err = float((got[:, :-3] - want).abs().max())
    print(f"b200v_sinusoid_embed vs the torch formula over [-1000, 1000]: max abs {err:.2e}")
    assert err <= 1e-6 and torch.isnan(got[:, -3:]).all()          # columns past the slots are not written


def test_native_conditioner_matches_reference(eng):
    g = golden("cond_vista_tiny")
    for case in mgc.CASES + ("recond",):
        (c, uc), vd = condition_case(eng, case)
        torch.cuda.synchronize()
        worst = check_against_fixture(c, uc, g, case, vd, 5e-3)
        print(f"{case}: CLIP slot rel-L2 {worst[0]:.2e}, concat rel-L2 {worst[1]:.2e}")


def test_work_elimination_is_exact(eng):
    """25 repeated rows: the conditioner embeds row 0 once; its c equals the embedders run on all 25 rows, bit for bit."""
    cond = eng.conditioner
    vd = mgc.value_dict("traj")
    cond.rows_embedded.clear()
    c, uc = eng.condition(vd, mgc.T, mgc.UC_KEYS)
    assert cond.rows_embedded == {"cond_frames_without_noise": 1, "cond_frames": 1}
    with torch.no_grad():
        clip_all = cond.embedders[0](vd["cond_frames_without_noise"].to(DEV).expand(mgc.T, -1, -1, -1).contiguous())
        enc_all = cond.embedders[3](vd["cond_frames"].to(DEV).expand(mgc.T, -1, -1, -1).contiguous())
        traj = cond.embedders[6](vd["trajectory"].to(DEV)[None].expand(mgc.T, -1).contiguous())
    torch.cuda.synchronize()
    assert torch.equal(c["crossattn"][..., :1024], clip_all)
    assert torch.equal(c["concat"], enc_all)
    assert torch.equal(c["crossattn"][..., 1152:2176], traj)
    assert not uc["crossattn"][..., :1024].any() and not uc["crossattn"][..., 1024:].any() and not uc["concat"].any()
    assert torch.equal(uc["vector"], c["vector"])


def test_two_runs_bit_identical(eng):
    for case in ("steer", "recond"):
        (c1, uc1), _ = condition_case(eng, case)
        (c2, uc2), _ = condition_case(eng, case)
        assert all(torch.equal(c1[k], c2[k]) and torch.equal(uc1[k], uc2[k]) for k in c1), case


def test_reconditioned_rollout_matches_cpu():
    """2 rounds x 3 steps with a trajectory action and conditioner_recondition: the H100 engine against the same loop on the
    CPU emulation of the kernels."""
    from vista_b200 import fused as fused_mod
    from vista_b200.rollout import conditioner_recondition
    rounds, steps = 2, 3
    vd = mgc.rollout_value_dict(sf)
    z = sf.noise("cond_gpu_z", 0, (sf.T, 4, sf.H // 2, sf.W // 2)) * 0.5
    noises = [sf.noise("cond_gpu", i, z.shape) for i in range(rounds)]

    def run(e, dev):
        e.en_and_decode_n_samples_a_time = 14
        c, uc = e.condition(vd, sf.T, mgc.UC_KEYS)
        return e.rollout(c, uc, z.to(dev), rounds, noises=noises, recondition=conditioner_recondition(e, vd, mgc.UC_KEYS))
    gpu_eng = native_engine(steps, cpu=False).to(DEV)
    fx, fz = run(gpu_eng, DEV)
    torch.cuda.synchronize()
    cpu_eng = native_engine(steps)
    saved = fused_mod.USE_GRAPH
    fused_mod.USE_GRAPH = False
    try:
        with patched_cond_ops(), torch.no_grad():
            rx, rz = run(cpu_eng, "cpu")
    finally:
        fused_mod.USE_GRAPH = saved
    ez, ex = rel_l2(fz.cpu(), rz), rel_l2(fx.cpu(), rx)
    print(f"re-conditioned rollout, H100 vs CPU emulation: latents rel-L2 {ez:.2e}, frames rel-L2 {ex:.2e}")
    assert ez < 5e-3 and ex < 5e-3, (ez, ex)
