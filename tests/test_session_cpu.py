"""engine.rollout_session without a GPU: the native-YAML engine at tiny sizes on CPU emulations of the kernels (as in
tests/test_conditioner_cpu.py).  A session stepped N rounds is byte for byte engine.rollout(..., u8=True) with the
conditioner re-run between rounds, with the same or a per-round action; it matches the reference's own do_sample; it
decodes 2 N chunks where the batch rollout decodes 3 N - 1; and the geometries it cannot line up with the rounds raise."""
import pytest
import torch

import seam_fakes as sf
from cond_fake_ops import patched_cond_ops
from helpers import golden, golden_rel
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine

ACTIONS = [{"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}, {"command": torch.tensor(2)},
           None]


@pytest.fixture(scope="module")
def eng():
    e = native_engine()
    e.en_and_decode_n_samples_a_time = 14
    return e


@pytest.fixture(autouse=True)
def no_graph(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)


def inputs(rounds, tag="session"):
    z = sf.noise(f"{tag}_z", 0, (sf.T, 4, sf.H // 2, sf.W // 2)) * 0.5
    return mgc.rollout_value_dict(sf), z, [sf.noise(tag, i, z.shape) for i in range(rounds)]


def counting_decodes(monkeypatch):
    """Counts DecoderRuntime.forward calls: one per decoded chunk."""
    from vista_b200 import vae as vae_mod
    calls = [0]
    forward = vae_mod.DecoderRuntime.forward

    def counted(self, *a, **k):
        calls[0] += 1
        return forward(self, *a, **k)
    monkeypatch.setattr(vae_mod.DecoderRuntime, "forward", counted)
    return calls


def run_session(eng, vd, z, noises, actions):
    """-> (the frames of every step and close() concatenated, samples_z, [the frames of each step])."""
    sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
    steps = [sess.step(a, noise=nz) for a, nz in zip(actions, noises)]
    return torch.cat(steps + [sess.close()]), sess.samples_z, steps


def per_round_recondition(eng, vds):
    """engine.rollout's recondition= hook that swaps in round n's value dict (the session's per-round action)."""
    from vista_b200.rollout import conditioner_recondition

    def recondition(round_idx, sample, decode_tail):
        return conditioner_recondition(eng, vds[round_idx], mgc.UC_KEYS)(round_idx, sample, decode_tail)
    return recondition


@pytest.mark.parametrize("rounds", [1, 2, 3])
def test_session_equals_batch_rollout(eng, rounds, monkeypatch):
    from vista_b200.rollout import conditioner_recondition
    vd, z, noises = inputs(rounds)
    calls = counting_decodes(monkeypatch)
    with patched_cond_ops(), torch.no_grad():
        frames, sz, steps = run_session(eng, vd, z, noises, [None] * rounds)
        session_decodes, calls[0] = calls[0], 0
        c, uc = eng.condition(vd, sf.T, mgc.UC_KEYS)
        want, want_z = eng.rollout(c, uc, z, rounds, noises=noises, recondition=conditioner_recondition(eng, vd, mgc.UC_KEYS),
                                   u8=True)
    assert [s.shape for s in steps] == [(sf.T - 3, sf.H, sf.W, 3)] * rounds and frames.dtype == torch.uint8
    assert torch.equal(frames, want) and torch.equal(sz, want_z)
    assert (session_decodes, calls[0]) == (2 * rounds, 3 * rounds - 1)
    assert all(not getattr(e, "skip_encode", False) for e in eng.conditioner.embedders)


def test_session_matches_the_real_do_sample(eng):
    """The seam_rollout_cond fixture: the unmodified do_sample, 2 rounds with a trajectory action, on the all-reference
    engine.  The session gets the trajectory as its action.  Its uint8 frames are compared at the centres of their
    truncation intervals ((k + 0.5) / 255)."""
    g = golden("seam_rollout_cond")
    rounds, steps = int(g["rounds"]), int(g["steps"])
    e = native_engine(steps)
    e.en_and_decode_n_samples_a_time = 14
    vd = mgc.rollout_value_dict(sf)
    action = {"trajectory": vd.pop("trajectory")}
    z = torch.from_numpy(g["z"])
    noises = [sf.noise("rollout_cond", i, z.shape) for i in range(rounds)]
    with patched_cond_ops():
        frames, sz, _ = run_session(e, vd, z, noises, [action] + [None] * (rounds - 1))
    x = (frames.permute(0, 3, 1, 2).float() + 0.5) / 255.0
    rz, rx = golden_rel(sz, g, "lat_"), golden_rel(x, g, "frames_")
    print(f"rollout_session vs the real do_sample: latents rel-L2 {rz}, frames rel-L2 {rx}")
    assert max(rz) < 5e-3 and max(rx) < 5e-3, (rz, rx)


def test_per_round_actions(eng):
    """A different action every round equals engine.rollout re-conditioned with the same per-round value dicts; round 0
    does not depend on later actions, and a different action in round 1 changes round 1's frames."""
    rounds = len(ACTIONS)
    vd, z, noises = inputs(rounds, "session_actions")
    del vd["trajectory"]
    vds, action = [], {}
    for a in ACTIONS:
        action = action if a is None else a
        vds.append({**vd, **action})
    with patched_cond_ops(), torch.no_grad():
        frames, sz, steps = run_session(eng, vd, z, noises, ACTIONS)
        c, uc = eng.condition(vds[0], sf.T, mgc.UC_KEYS)
        want, want_z = eng.rollout(c, uc, z, rounds, noises=noises, recondition=per_round_recondition(eng, vds), u8=True)
        other = [ACTIONS[0], {"speed": torch.tensor([5.41, 5.62, 5.80, 6.03]), "angle": torch.tensor([-0.02, -0.01, 0, 0.01])}]
        _, _, steps2 = run_session(eng, vd, z, noises[:2], other)
    assert torch.equal(frames, want) and torch.equal(sz, want_z)
    assert torch.equal(steps2[0], steps[0])
    assert not torch.equal(steps2[1], steps[1])


def test_unsupported_geometry_raises(eng, monkeypatch):
    vd, z, _ = inputs(1)
    with pytest.raises(NotImplementedError, match="line up"):
        eng.rollout_session(vd, z, n_cond=2)
    with pytest.raises(NotImplementedError, match="line up"):
        eng.rollout_session(vd, z[:21])
    monkeypatch.setattr(eng, "en_and_decode_n_samples_a_time", 10)
    with pytest.raises(NotImplementedError, match="line up"):
        eng.rollout_session(vd, z)
    monkeypatch.setattr(eng, "en_and_decode_n_samples_a_time", 14)
    monkeypatch.setattr(eng.model, "frame_sharded", True, raising=False)
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        eng.rollout_session(vd, z)
    monkeypatch.setattr(eng.model, "frame_sharded", False)
    monkeypatch.setattr(eng, "_conditioner", None)
    with pytest.raises(NotImplementedError, match="conditioner"):
        eng.rollout_session(vd, z)


def test_session_misuse_raises(eng):
    vd, z, noises = inputs(1)
    sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)
    with pytest.raises(RuntimeError, match="before the first step"):
        sess.close()
    with pytest.raises(ValueError, match="action keys"):
        sess.step({"fps_id": 3}, noise=noises[0])
    with patched_cond_ops():
        sess.step(noise=noises[0])
    assert sess.close().shape == (3, sf.H, sf.W, 3)
    with pytest.raises(RuntimeError, match="after close"):
        sess.step(noise=noises[0])
