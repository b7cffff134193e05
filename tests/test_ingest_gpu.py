"""Camera frames in, on the H100: ``engine.frames_from_u8`` (csrc/ingest/ingest.cu) is ``torch.equal`` to sample.py's load_img
body run with PIL and torchvision, for every geometry of tests/test_ingest_cpu.py, from host and device tensors, at T = 1
and for 25 nuScenes-sized frames; and ``engine.rollout_session_from_frames`` is the session sample.py's recipe builds by
hand, with a latent clip that is zero outside the conditioning frames."""
import os

import numpy as np
import pytest
import torch

import seam_fakes as sf
from oracle import make_golden_cond as mgc
from test_ingest_cpu import GEOMETRIES, geometry_id, load_img_body, random_frames
from test_session_gpu import gpu_engine

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAJECTORY = torch.tensor([0.12, 2.85, 0.31, 5.62, 0.55, 8.31, 0.94, 10.97])


@pytest.fixture(scope="module")
def eng():
    return gpu_engine()


def _source(rgb: np.ndarray, where: str) -> torch.Tensor:
    t = torch.from_numpy(rgb)
    if where == "host":
        return t
    # a device view with padded rows and frames, so the kernel reads through its strides
    T, H, W, _ = t.shape
    buf = torch.zeros(T, H + 3, W + 5, 3, dtype=torch.uint8, device=DEV)
    view = buf[:, 2:2 + H, 1:1 + W]
    view.copy_(t)
    return view


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("geom", GEOMETRIES, ids=geometry_id)
def test_frames_from_u8_equals_load_img(eng, geom, where):
    (ws, hs), (W, H) = geom
    rgb = random_frames(1, hs, ws, seed=ws + 3 * hs)
    want = torch.stack([load_img_body(f, H, W) for f in rgb])
    got = eng.frames_from_u8(_source(rgb, where), height=H, width=W)
    assert got.device.type == "cuda" and got.dtype == torch.float32 and got.shape == (1, 3, H, W)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("where", ["host", "device"])
def test_frames_from_u8_25_nuscenes_frames(eng, where):
    rgb = random_frames(25, 900, 1600, seed=11)
    want = torch.stack([load_img_body(f, 576, 1024) for f in rgb])
    src = _source(rgb, where)
    a = eng.frames_from_u8(src)
    b = eng.frames_from_u8(src)
    assert a.shape == (25, 3, 576, 1024)
    assert torch.equal(a, b)                                        # two calls bit-identical
    assert torch.equal(a.cpu(), want)


def test_frames_from_u8_rejects_malformed_input(eng):
    good = torch.zeros(2, 90, 160, 3, dtype=torch.uint8)
    for bad, kw in ((good.float(), {}), (good[..., :2], {}), (torch.zeros(2, 90, 160, 4, dtype=torch.uint8), {}),
                    (good, dict(height=60, width=100)), (good, dict(height=36, width=64)), (good[0], {})):
        with pytest.raises(ValueError):
            eng.frames_from_u8(bad, **kw)
    with pytest.raises(ValueError):
        eng.rollout_session_from_frames(good, n_conds=3, height=sf.H, width=sf.W)
    with pytest.raises(ValueError):
        eng.rollout_session_from_frames(good, action={"steer": torch.tensor(0.1)}, height=sf.H, width=sf.W)


def _hand_built(eng, rgb, n_conds, cond_aug, action, cond_aug_noise, encode_noise, H, W, uc_keys):
    """sample.py:222-253 and the head of do_sample on load_img's tensors, written out: the session the caller would build."""
    img = torch.stack([load_img_body(f, H, W) for f in rgb[:n_conds]]).to(DEV)
    vd = {}
    for key in {e.input_key for e in eng.conditioner.embedders}:          # init_embedder_options, sample_utils.py:83-93
        if key in ("fps_id", "fps"):
            vd["fps"] = 10
            vd["fps_id"] = 9
        elif key == "motion_bucket_id":
            vd["motion_bucket_id"] = 127
    cond_img = img[0][None]
    vd["cond_frames_without_noise"] = cond_img
    vd["cond_aug"] = cond_aug
    vd["cond_frames"] = cond_img + cond_aug * cond_aug_noise.to(DEV)
    vd.update(action)
    zc = eng.encode_first_stage(img, noise=encode_noise[:n_conds].to(DEV))
    z = torch.zeros((eng.num_frames,) + tuple(zc.shape[1:]), device=DEV)
    z[:n_conds] = zc
    return eng.rollout_session(vd, z, force_uc_zero_embeddings=uc_keys, initial_cond_indices=list(range(n_conds)))


def _run(sess, noises):
    steps = [sess.step(None, noise=nz) for nz in noises]
    return torch.cat(steps + [sess.close()]), sess.samples_z.clone()


def test_session_from_frames_equals_hand_built(eng):
    rgb = random_frames(2, 90, 160, seed=5)
    h, w = sf.H // 2, sf.W // 2
    cond_aug_noise = torch.randn(1, 3, sf.H, sf.W, generator=torch.Generator().manual_seed(6))
    encode_noise = torch.randn(2, 4, h, w, generator=torch.Generator().manual_seed(7))
    noises = [sf.noise("ingest", i, (sf.T, 4, h, w)) for i in range(2)]
    action = {"trajectory": TRAJECTORY}
    sess = eng.rollout_session_from_frames(torch.from_numpy(rgb), n_conds=1, cond_aug=0.02, action=action,
                                           force_uc_zero_embeddings=mgc.UC_KEYS, height=sf.H, width=sf.W,
                                           cond_aug_noise=cond_aug_noise, encode_noise=encode_noise)
    fx, fz = _run(sess, noises)
    want = _hand_built(eng, rgb, 1, 0.02, action, cond_aug_noise, encode_noise, sf.H, sf.W, mgc.UC_KEYS)
    wx, wz = _run(want, noises)
    torch.cuda.synchronize()
    assert fx.dtype == torch.uint8 and fx.shape == (2 * (sf.T - 3) + 3, sf.H, sf.W, 3)
    assert torch.equal(fx, wx) and torch.equal(fz, wz)


@pytest.mark.parametrize("n_conds", [1, 3])
def test_zero_latents_outside_conditioning_frames(eng, n_conds):
    """A session reads its latent clip only on the conditioning frames: the full 25-frame encode and the same latents
    zeroed outside [0, n_conds) give the same frames, latents and rewards."""
    img = eng.frames_from_u8(torch.from_numpy(random_frames(sf.T, 90, 160, seed=8)), height=sf.H, width=sf.W)
    z_full = eng.encode_first_stage(img, noise=torch.randn(sf.T, 4, sf.H // 2, sf.W // 2, device=DEV,
                                                           generator=torch.Generator(DEV).manual_seed(9)))
    z_zero = torch.zeros_like(z_full)
    z_zero[:n_conds] = z_full[:n_conds]
    assert z_full[n_conds:].abs().amax() > 0
    vd = {"fps_id": 9, "motion_bucket_id": 127, "cond_aug": 0.0, "cond_frames_without_noise": img[0:1],
          "cond_frames": img[0:1], "trajectory": TRAJECTORY}
    noises = [sf.noise("ingest_zero", i, z_full.shape) for i in range(2)]
    out = []
    for z in (z_full, z_zero):
        sess = eng.rollout_session(vd, z, force_uc_zero_embeddings=mgc.UC_KEYS, initial_cond_indices=list(range(n_conds)))
        r0, _ = sess.score([None, {"command": torch.tensor(2)}], ensemble_size=2, num_steps=2, seed=3)
        sess.step(None, noise=noises[0])
        r1, _ = sess.score([None], ensemble_size=2, num_steps=2, seed=4)
        fx = torch.cat([sess.step(None, noise=noises[1]), sess.close()])
        out.append((fx, sess.samples_z.clone(), r0, r1))
    torch.cuda.synchronize()
    (fa, za, r0a, r1a), (fb, zb, r0b, r1b) = out
    assert torch.equal(fa, fb) and torch.equal(za, zb)
    assert torch.equal(r0a, r0b) and torch.equal(r1a, r1b)


def _bench_session():
    import importlib.util
    spec_ = importlib.util.spec_from_file_location("bench_session", os.path.join(ROOT, "tools", "bench_session.py"))
    mod = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(mod)
    return mod


def test_session_from_frames_full_size():
    """1600 x 900 frames at 576 x 1024 on the full-size native engine (2 EDM steps): one step equals the hand-built
    session's."""
    bs = _bench_session()
    big = bs.build_engine(DEV)
    big.sampler.num_steps = 2
    rgb = random_frames(2, 900, 1600, seed=12)
    cond_aug_noise = torch.randn(1, 3, 576, 1024, generator=torch.Generator().manual_seed(13))
    encode_noise = torch.randn(1, 4, 72, 128, generator=torch.Generator().manual_seed(14))
    noise = torch.randn(big.num_frames, 4, 72, 128, generator=torch.Generator().manual_seed(15))
    action = {"trajectory": bs.TRAJECTORY}
    sess = big.rollout_session_from_frames(torch.from_numpy(rgb), n_conds=1, cond_aug=0.02, action=action,
                                           force_uc_zero_embeddings=bs.UC_KEYS, cond_aug_noise=cond_aug_noise,
                                           encode_noise=encode_noise)
    got = sess.step(None, noise=noise)
    want_sess = _hand_built(big, rgb, 1, 0.02, action, cond_aug_noise, encode_noise, 576, 1024, bs.UC_KEYS)
    want = want_sess.step(None, noise=noise)
    torch.cuda.synchronize()
    assert got.shape == (big.num_frames - 3, 576, 1024, 3)
    assert torch.equal(got, want) and torch.equal(sess.samples_z, want_sess.samples_z)
