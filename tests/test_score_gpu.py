"""RolloutSession.score and RolloutSession.fork on the H100: the checks of tests/test_score_cpu.py on the tiny presets of
configs/inference/vista_b200_native.yaml, with the fused sampler replayed from CUDA graphs.  At Vista's 576 x 1024 with
the native YAML, a round-1 score followed by a step completes, repeats bit for bit and fits on the 80 GB card."""
import pytest
import torch

import test_score_cpu as tsc
from test_fullres_gpu import _bench_session
from test_session_gpu import gpu_engine
from vista_b200 import synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GIB = 2 ** 30


@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


def test_round0_equals_sample_ensemble(eng, monkeypatch):
    tsc.check_round0_equals_sample_ensemble(eng, DEV, monkeypatch)


@pytest.mark.parametrize("rounds_before", [1, 2])
def test_later_round_equals_step(eng, rounds_before):
    tsc.check_later_round_equals_step(eng, DEV, rounds_before)


@pytest.mark.parametrize("seeded", [False, True])
def test_scoring_leaves_the_session_untouched(eng, seeded):
    tsc.check_scoring_leaves_the_session_untouched(eng, DEV, seeded)


def test_score_deterministic(eng):
    tsc.check_score_deterministic(eng, DEV)


def test_fork(eng):
    tsc.check_fork(eng, DEV)


def test_misuse_raises(eng, monkeypatch):
    tsc.check_misuse_raises(eng, DEV, monkeypatch)


def test_score_at_576x1024_repeats_and_fits():
    """The native YAML engine at Vista's resolution: after one round of 2 steps, two candidates x 2 members x 2 steps
    scored twice, then the next round stepped.  The two scores agree bit for bit, and the peak allocation over the run
    stays within 72 GiB."""
    from oracle.make_golden_clip import clip_frames
    bs = _bench_session()
    eng = bs.build_engine(DEV)
    eng.sampler.num_steps = 2
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)        # the run's peak, with the weights and executors resident
    T, H, W = eng.num_frames, 576, 1024
    frame = torch.from_numpy(clip_frames(12, "score_fullres", 1, H, W)).to(DEV)
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": frame, "cond_frames": frame}
    z = torch.from_numpy(synth.normal(7, "score_fullres.z", (T, 4, H // 8, W // 8), std=0.9)).to(DEV)
    candidates = [{"trajectory": bs.TRAJECTORY}, {"trajectory": bs.TRAJECTORY * 0.5}]
    torch.manual_seed(5)
    sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=bs.UC_KEYS)
    sess.step(candidates[0])
    r1, m1 = sess.score(candidates, ensemble_size=2, num_steps=2, seed=1)
    r2, m2 = sess.score(candidates, ensemble_size=2, num_steps=2, seed=1)
    frames = sess.step(candidates[1])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV)
    print(f"576 x 1024 score at round 1 (K = 2, E = 2, 2 steps), then a step: rewards {r1.tolist()}, "
          f"peak allocated {peak / GIB:.2f} GiB")
    assert m1.shape == (2, 2, T, 4, H // 8, W // 8) and frames.shape == (T - 3, H, W, 3)
    assert torch.isfinite(m1).all() and torch.equal(m1, m2) and torch.equal(r1, r2)
    assert peak <= 72 * GIB
