"""RolloutSession.score and RolloutSession.fork without a GPU: the native-YAML engine at tiny sizes on CPU emulations of the
kernels (as in tests/test_session_cpu.py).  In round 0, score is engine.sample_ensemble on the same conditioning.  In a
later round, a member equals the round latent that step() then samples with the same action and noise.  Scoring leaves
the session as it was, with injected or with seeded noise.  The reward is exp(-mean variance) of the members.  A fork
steps like the original and independently of it, and misuse raises.  tests/test_score_gpu.py runs the same checks on
the H100."""
import copy

import pytest
import torch

import seam_fakes as sf
from cond_fake_ops import patched_cond_ops
from oracle import make_golden_cond as mgc
from test_conditioner_cpu import native_engine
from test_session_cpu import inputs

# the session's value dict carries a trajectory; these candidates replace it, or add a command
A = {"trajectory": torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])}
B = {"trajectory": torch.tensor([-0.35, 2.41, -1.02, 4.66, -1.93, 6.74, -3.05, 8.62])}
C = {"command": torch.tensor(2)}
STRIDE = sf.T - 3           # latent frames a round adds after the first


@pytest.fixture(scope="module")
def eng():
    e = native_engine()
    e.en_and_decode_n_samples_a_time = 14
    return e


@pytest.fixture(autouse=True)
def emulated(monkeypatch):
    from vista_b200 import fused as fused_mod
    monkeypatch.setattr(fused_mod, "USE_GRAPH", False)
    with patched_cond_ops():
        yield


def session(eng, vd, z):
    return eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS)


def vanilla(eng, steps):
    """The engine's sampler with reward.py's guider (VanillaCFG) and ``steps`` steps."""
    from vista_b200.diffusion import VanillaCFG
    s = copy.copy(eng.sampler)
    s.guider, s.num_steps = VanillaCFG(2.5), steps
    return s


def fp64_reward(members):
    """exp(-mean unbiased variance) over the ensemble axis of one candidate's (E, T, 4, h, w) members, in fp64."""
    return float(torch.exp(-members.double().var(dim=0, correction=1).mean()))


def check_round0_equals_sample_ensemble(eng, dev, monkeypatch):
    vd, z, ns = inputs(3, "score_round0")
    z = z.to(dev)
    smp = vanilla(eng, 3)
    sess = session(eng, vd, z)
    rewards, members = sess.score([A], ensemble_size=3, num_steps=3, noises=ns, sampler=smp)
    monkeypatch.setattr(eng, "sampler", smp)
    reward, want = eng.sample_ensemble(*eng.condition({**vd, **A}, sf.T, mgc.UC_KEYS), z, 3, noises=ns)
    assert rewards.shape == (1,) and rewards.dtype == torch.float32 and rewards.device == z.device
    assert members.shape == (1, 3) + tuple(z.shape) and members.dtype == torch.float32
    assert torch.equal(members[0], torch.stack(want)) and torch.equal(rewards[0], reward)
    assert sess.rounds == 0 and sess.samples_z.shape[0] == 0


def check_later_round_equals_step(eng, dev, rounds_before):
    """After ``rounds_before`` steps with A: candidate B's member 0 is the round latent step(B, noise=n0) samples; the
    candidate None is the session's current action (A); every member keeps the conditioning frames."""
    r = rounds_before
    vd, z, ns = inputs(r + 2, f"score_round{r}")
    z = z.to(dev)
    sess = session(eng, vd, z)
    for i in range(r):
        sess.step(A if i == 0 else None, noise=ns[i])
    filled = sess.samples_z[-3:].clone()
    rewards, members = sess.score([B, None], ensemble_size=2, num_steps=eng.sampler.num_steps, noises=ns[r:])
    again, _ = sess.score([A], ensemble_size=2, num_steps=eng.sampler.num_steps, noises=ns[r:])
    sess.step(B, noise=ns[r])
    lat = sess.samples_z[r * STRIDE:r * STRIDE + sf.T]
    assert torch.equal(members[0, 0], lat)
    assert not torch.equal(members[1, 0], lat)
    assert torch.equal(again[0], rewards[1])
    assert torch.equal(members[:, :, :3], filled.expand_as(members[:, :, :3]))
    for k in range(2):
        assert abs(float(rewards[k]) - fp64_reward(members[k].cpu())) <= 1e-5 * fp64_reward(members[k].cpu())


def check_scoring_leaves_the_session_untouched(eng, dev, seeded):
    """A session that scores before every step and before close() against one that never scores: same frames, tail
    and latents — with injected step noise, or (``seeded``) with both sessions drawing their own from the same seed."""
    actions = [A, C]
    vd, z, ns = inputs(len(actions), "score_untouched")
    z = z.to(dev)
    noises = [None] * len(actions) if seeded else ns

    def run(scoring):
        if seeded:
            torch.manual_seed(77)
        sess = session(eng, vd, z)
        frames = []
        for a, nz in zip(actions, noises):
            if scoring:
                sess.score([B, None], ensemble_size=2, num_steps=2)
            frames.append(sess.step(a, noise=nz))
        if scoring:
            sess.score([A], ensemble_size=2, num_steps=2, seed=3)
        return torch.cat(frames + [sess.close()]), sess.samples_z

    f0, z0 = run(False)
    f1, z1 = run(True)
    assert torch.equal(f0, f1) and torch.equal(z0, z1)


def check_score_deterministic(eng, dev):
    vd, z, _ = inputs(0, "score_seed")
    z = z.to(dev)
    sess = session(eng, vd, z)
    r1, m1 = sess.score([A, B], ensemble_size=2, num_steps=2, seed=5)
    r2, m2 = sess.score([A, B], ensemble_size=2, num_steps=2, seed=5)
    _, m3 = sess.score([A], ensemble_size=2, num_steps=2, seed=6)
    assert torch.equal(r1, r2) and torch.equal(m1, m2)
    assert not torch.equal(m1[0], m3[0])
    assert float(r1[0]) != float(r1[1])
    for k in range(2):
        want = fp64_reward(m1[k].cpu())
        print(f"candidate {k}: reward {float(r1[k]):.6f}, fp64 recomputation {want:.6f}")
        assert abs(float(r1[k]) - want) <= 1e-5 * want


def check_fork(eng, dev):
    """A fresh session stepped A, B, C against a session forked after round 1: the fork's rounds 2 and 3 are the fresh
    ones; the original, stepped after the fork has moved on, still samples them; a fork stepped with another action
    leaves the original's next round as it was."""
    vd, z, ns = inputs(3, "score_fork")
    z = z.to(dev)
    fresh = session(eng, vd, z)
    want = [fresh.step(a, noise=nz) for a, nz in zip((A, B, C), ns)]
    want_tail, want_z = fresh.close(), fresh.samples_z
    sess = session(eng, vd, z)
    assert torch.equal(sess.step(A, noise=ns[0]), want[0])
    fork = sess.fork()
    assert fork.rounds == 1 and fork.engine is sess.engine
    assert torch.equal(fork.step(B, noise=ns[1]), want[1]) and torch.equal(fork.step(C, noise=ns[2]), want[2])
    assert torch.equal(fork.close(), want_tail) and torch.equal(fork.samples_z, want_z)
    assert sess.rounds == 1
    assert torch.equal(sess.step(B, noise=ns[1]), want[1])
    other = sess.fork()
    assert not torch.equal(other.step(A, noise=ns[2]), want[2])
    assert torch.equal(sess.step(C, noise=ns[2]), want[2])
    assert torch.equal(sess.close(), want_tail) and torch.equal(sess.samples_z, want_z)


def check_misuse_raises(eng, dev, monkeypatch):
    vd, z, ns = inputs(2, "score_misuse")
    z = z.to(dev)
    sess = session(eng, vd, z)

    def no_sampling(*a, **k):
        raise AssertionError("score sampled before rejecting its arguments")
    with monkeypatch.context() as m:
        m.setattr(eng, "sampler", no_sampling)
        for bad in (dict(ensemble_size=1), dict(ensemble_size=65), dict(noises=ns),
                    dict(ensemble_size=2, noises=[ns[0], ns[1][:, :2]])):
            with pytest.raises(ValueError, match="ensemble_size|noises"):
                sess.score([A], **bad)
        with pytest.raises(ValueError, match="action keys"):
            sess.score([A, {"fps_id": 3}], ensemble_size=2)
        for empty in ([], A):
            with pytest.raises(ValueError, match="non-empty list"):
                sess.score(empty, ensemble_size=2)
    sess.step(A, noise=ns[0])
    sess.close()
    with pytest.raises(RuntimeError, match="after close"):
        sess.score([A], ensemble_size=2)


def test_round0_equals_sample_ensemble(eng, monkeypatch):
    check_round0_equals_sample_ensemble(eng, torch.device("cpu"), monkeypatch)


@pytest.mark.parametrize("rounds_before", [1, 2])
def test_later_round_equals_step(eng, rounds_before):
    check_later_round_equals_step(eng, torch.device("cpu"), rounds_before)


@pytest.mark.parametrize("seeded", [False, True])
def test_scoring_leaves_the_session_untouched(eng, seeded):
    check_scoring_leaves_the_session_untouched(eng, torch.device("cpu"), seeded)


def test_score_deterministic(eng):
    check_score_deterministic(eng, torch.device("cpu"))


def test_fork(eng):
    check_fork(eng, torch.device("cpu"))


def test_misuse_raises(eng, monkeypatch):
    check_misuse_raises(eng, torch.device("cpu"), monkeypatch)
