"""engine.rollout_session on the H100 (tiny presets of configs/inference/vista_b200_native.yaml): byte-equal to
engine.rollout(..., u8=True) re-conditioned between rounds, with the same or a per-round action, in 2 N chunk decodes
instead of 3 N - 1; the seam_rollout_cond inputs against the same session on the CPU emulation and against the reference's
do_sample; two sessions from the same seed bit-identical, and equal to the batch rollout drawing its own noise."""
import pytest
import torch

import seam_fakes as sf
from cond_fake_ops import patched_cond_ops
from helpers import golden, golden_rel, rel_l2
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine
from test_session_cpu import ACTIONS, counting_decodes, inputs, per_round_recondition, run_session

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def gpu_engine(steps=3):
    e = native_engine(steps, cpu=False).to(DEV)
    e.en_and_decode_n_samples_a_time = 14
    return e


@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


@pytest.mark.parametrize("rounds", [1, 2, 3])
def test_session_equals_batch_rollout(eng, rounds, monkeypatch):
    from vista_b200.rollout import conditioner_recondition
    vd, z, noises = inputs(rounds)
    z = z.to(DEV)
    calls = counting_decodes(monkeypatch)
    frames, sz, steps = run_session(eng, vd, z, noises, [None] * rounds)
    session_decodes, calls[0] = calls[0], 0
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, rounds, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                               u8=True)
    torch.cuda.synchronize()
    assert [s.shape for s in steps] == [(sf.T - 3, sf.H, sf.W, 3)] * rounds and frames.is_cuda
    assert torch.equal(frames, want) and torch.equal(sz, want_z)
    assert (session_decodes, calls[0]) == (2 * rounds, 3 * rounds - 1)


def test_session_matches_cpu_and_the_real_do_sample():
    """The seam_rollout_cond inputs (2 rounds, trajectory action): the H100 session against the same session on the CPU
    emulation of the kernels, and against the unmodified do_sample's fixture."""
    from vista_b200 import fused as fused_mod
    g = golden("seam_rollout_cond")
    rounds, steps = int(g["rounds"]), int(g["steps"])
    vd = mgc.rollout_value_dict(sf)
    action = {"trajectory": vd.pop("trajectory")}
    z = torch.from_numpy(g["z"])
    noises = [sf.noise("rollout_cond", i, z.shape) for i in range(rounds)]
    actions = [action] + [None] * (rounds - 1)
    fx, fz, _ = run_session(gpu_engine(steps), vd, z.to(DEV), noises, actions)
    torch.cuda.synchronize()
    cpu_eng = native_engine(steps)
    cpu_eng.en_and_decode_n_samples_a_time = 14
    saved = fused_mod.USE_GRAPH
    fused_mod.USE_GRAPH = False
    try:
        with patched_cond_ops():
            rx, rz, _ = run_session(cpu_eng, vd, z, noises, actions)
    finally:
        fused_mod.USE_GRAPH = saved
    ez, ex = rel_l2(fz.cpu(), rz), rel_l2(fx.cpu().float(), rx.float())
    print(f"rollout_session, H100 vs CPU emulation: latents rel-L2 {ez:.2e}, uint8 frames rel-L2 {ex:.2e}")
    assert ez < 5e-3 and ex < 5e-3, (ez, ex)
    gz, gx = golden_rel(fz, g, "lat_"), golden_rel((fx.permute(0, 3, 1, 2).float() + 0.5) / 255.0, g, "frames_")
    print(f"rollout_session on the H100 vs the real do_sample: latents rel-L2 {gz}, frames rel-L2 {gx}")
    assert max(gz) < 5e-3 and max(gx) < 5e-3, (gz, gx)


def test_per_round_actions(eng):
    rounds = len(ACTIONS)
    vd, z, noises = inputs(rounds, "session_actions")
    z = z.to(DEV)
    del vd["trajectory"]
    vds, action = [], {}
    for a in ACTIONS:
        action = action if a is None else a
        vds.append({**vd, **action})
    frames, sz, steps = run_session(eng, vd, z, noises, ACTIONS)
    c, uc = eng.condition(vds[0], sf.T, mgc.UC_KEYS)
    want, want_z = eng.rollout(c, uc, z, rounds, noises=noises, recondition=per_round_recondition(eng, vds), u8=True)
    other = [ACTIONS[0], {"speed": torch.tensor([5.41, 5.62, 5.80, 6.03]), "angle": torch.tensor([-0.02, -0.01, 0, 0.01])}]
    _, _, steps2 = run_session(eng, vd, z, noises[:2], other)
    torch.cuda.synchronize()
    assert torch.equal(frames, want) and torch.equal(sz, want_z)
    assert torch.equal(steps2[0], steps[0])
    assert not torch.equal(steps2[1], steps[1])


def test_seeded_sessions_bit_identical(eng):
    """Without injected noise: two sessions from the same seed agree bit for bit, and with engine.rollout from that seed
    (the noise is drawn in the same order)."""
    from vista_b200.rollout import conditioner_recondition
    rounds = 2
    vd, z, _ = inputs(rounds, "session_seed")
    z = z.to(DEV)
    runs = []
    for _ in range(2):
        torch.manual_seed(77)
        runs.append(run_session(eng, vd, z, [None] * rounds, [None] * rounds)[:2])
    c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
    torch.manual_seed(77)
    want, want_z = eng.rollout(c, uc, z, rounds, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS), u8=True)
    torch.cuda.synchronize()
    for frames, sz in runs:
        assert torch.equal(frames, want) and torch.equal(sz, want_z)
