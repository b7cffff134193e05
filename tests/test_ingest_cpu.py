"""Camera frames in, without a GPU: the host half of ``engine.frames_from_u8`` (vista_b200/ingest.py).  ``lanczos_tables``
with a numpy restatement of the kernel's two integer passes is byte-equal to PIL's LANCZOS resize; ``crop_box`` is
load_img's crop; and the whole restatement (crop, resize, / 255, * 2 - 1) is ``torch.equal`` to load_img's body run with
the real PIL and torchvision.  It also holds INGEST_KERNEL_TESTS, the conformance tests of the kernels under
vista_b200/csrc/ingest/, and checks that every kernel anywhere under vista_b200/csrc/ is held by a test."""
import os
import re

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision import transforms

import seam_fakes as sf
from vista_b200 import ingest

# (source width, height) -> (target width, height)
GEOMETRIES = [
    ((1600, 900), (1024, 576)),          # nuScenes
    ((1920, 1080), (1024, 576)),
    ((640, 480), (1024, 576)),           # row crop + upscale
    ((900, 1600), (1024, 576)),          # portrait: row crop
    ((1024, 576), (1024, 576)),          # no pass
    ((1025, 577), (1024, 576)),
    ((1600, 900), (576, 320)),
    ((1600, 900), (sf.W, sf.H)),         # the tiny presets' frame
    ((1601, 900), (1024, 576)),          # column crop with an odd margin: the extra column is on the right
    ((1024, 700), (1024, 576)),          # vertical pass only
]


def geometry_id(g):
    (ws, hs), (w, h) = g
    return f"{ws}x{hs}-{w}x{h}"


def random_frames(n, hs, ws, seed=0):
    return np.random.default_rng(seed).integers(0, 256, size=(n, hs, ws, 3), dtype=np.uint8)


def load_img_body(rgb: np.ndarray, target_height: int, target_width: int) -> torch.Tensor:
    """sample.py:174-201 (load_img) after the file is decoded to RGB, with the real PIL and torchvision."""
    image = Image.fromarray(rgb)
    ori_w, ori_h = image.size
    if ori_w / ori_h > target_width / target_height:
        tmp_w = int(target_width / target_height * ori_h)
        left = (ori_w - tmp_w) // 2
        right = (ori_w + tmp_w) // 2
        image = image.crop((left, 0, right, ori_h))
    elif ori_w / ori_h < target_width / target_height:
        tmp_h = int(target_height / target_width * ori_w)
        top = (ori_h - tmp_h) // 2
        bottom = (ori_h + tmp_h) // 2
        image = image.crop((0, top, ori_w, bottom))
    image = image.resize((target_width, target_height), resample=Image.LANCZOS)
    image = transforms.Compose([
        transforms.ToTensor(),
        transforms.Lambda(lambda x: x * 2.0 - 1.0)
    ])(image)
    return image


def load_img_box(ori_w, ori_h, target_width, target_height):
    """The crop box load_img computes (sample.py:185-194), with the un-cropped case as the whole frame."""
    if ori_w / ori_h > target_width / target_height:
        tmp_w = int(target_width / target_height * ori_h)
        return (ori_w - tmp_w) // 2, 0, (ori_w + tmp_w) // 2, ori_h
    if ori_w / ori_h < target_width / target_height:
        tmp_h = int(target_height / target_width * ori_w)
        return 0, (ori_h - tmp_h) // 2, ori_w, (ori_h + tmp_h) // 2
    return 0, 0, ori_w, ori_h


def _pass(img: np.ndarray, tab: ingest.Tables, axis: int) -> np.ndarray:
    """One integer pass of the kernel along ``axis`` of an (H, W, 3) uint8 image: 1 << 21 + sum src * w, >> 22, clamp."""
    out_n = tab.bounds.shape[0]
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((out_n,) + src.shape[1:], 1 << (ingest.PRECISION_BITS - 1), np.int64)
    for k in range(tab.ksize):
        live = k < tab.bounds[:, 1]
        idx = np.where(live, tab.bounds[:, 0] + k, 0)
        w = np.where(live, tab.weights[:, k], 0).astype(np.int64)
        acc += src[idx] * w.reshape((-1,) + (1,) * (src.ndim - 1))
    assert acc.max() < 2 ** 31 and acc.min() >= -2 ** 31          # the kernel accumulates in int32
    return np.moveaxis(np.clip(acc >> ingest.PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def resize_restated(img: np.ndarray, W: int, H: int) -> np.ndarray:
    """The kernel's resize in numpy: the horizontal pass over the rows the vertical pass reads, then the vertical pass;
    a pass whose size is unchanged is skipped."""
    h, w, _ = img.shape
    y0, y1 = 0, h
    ytab = ingest.lanczos_tables(h, H) if h != H else None
    if ytab is not None:
        y0, y1 = int(ytab.bounds[0, 0]), int(ytab.bounds[-1, 0] + ytab.bounds[-1, 1])
    mid = _pass(img[y0:y1], ingest.lanczos_tables(w, W), 1) if w != W else img[y0:y1]
    if ytab is None:
        return mid
    shifted = ingest.Tables(ytab.bounds - np.array([y0, 0], np.int32), ytab.weights, ytab.ksize)
    return _pass(mid, shifted, 0)


def host_restated(rgb: np.ndarray, H: int, W: int) -> torch.Tensor:
    """crop_box + resize_restated + ToTensor's / 255 + * 2 - 1."""
    left, top, right, bottom = ingest.crop_box(rgb.shape[1], rgb.shape[0], W, H)
    u8 = resize_restated(rgb[top:bottom, left:right], W, H)
    return torch.from_numpy(np.ascontiguousarray(u8)).permute(2, 0, 1).to(torch.float32).div(255) * 2.0 - 1.0


@pytest.mark.parametrize("geom", GEOMETRIES, ids=geometry_id)
def test_tables_and_integer_passes_equal_pil(geom):
    (ws, hs), (W, H) = geom
    rgb = random_frames(1, hs, ws, seed=ws * 7 + hs)[0]
    left, top, right, bottom = ingest.crop_box(ws, hs, W, H)
    want = np.asarray(Image.fromarray(rgb).crop((left, top, right, bottom)).resize((W, H), resample=Image.LANCZOS))
    got = resize_restated(rgb[top:bottom, left:right], W, H)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_tables_shape_and_normalisation():
    for n_in, n_out in ((1600, 1024), (506, 576), (900, 32), (7, 7), (1, 5)):
        t = ingest.lanczos_tables(n_in, n_out)
        assert t.bounds.shape == (n_out, 2) and t.weights.shape == (n_out, t.ksize)
        assert (t.bounds[:, 0] >= 0).all() and (t.bounds.sum(1) <= n_in).all() and (t.bounds[:, 1] <= t.ksize).all()
        sums = t.weights.astype(np.int64).sum(1)
        assert (np.abs(sums - (1 << 22)) <= t.ksize).all()          # each weight rounded once
        for i, (_, n) in enumerate(t.bounds):
            assert not t.weights[i, n:].any()
    assert ingest.lanczos_tables(1600, 1024) is ingest.lanczos_tables(1600, 1024)     # cached per geometry
    with pytest.raises(ValueError):
        ingest.lanczos_tables(0, 4)


def test_crop_box_is_load_imgs():
    margins = set()
    for ws in list(range(1590, 1611)) + [97, 333, 640, 900, 1025, 1280, 1920]:
        for hs in (61, 187, 480, 577, 899, 900, 901, 1080, 1600):
            for W, H in ((1024, 576), (576, 320), (sf.W, sf.H), (200, 57)):
                box = ingest.crop_box(ws, hs, W, H)
                assert box == load_img_box(ws, hs, W, H), (ws, hs, W, H)
                left, top, right, bottom = box
                if ws / hs > W / H:
                    margins.add(("column", (ws - int(W / H * hs)) % 2))
                elif ws / hs < W / H:
                    margins.add(("row", (hs - int(H / W * ws)) % 2))
    # odd and even margins on both axes: an odd one leaves its extra pixel on the right / at the bottom
    assert margins == {("column", 0), ("column", 1), ("row", 0), ("row", 1)}


@pytest.mark.parametrize("geom", GEOMETRIES, ids=geometry_id)
def test_host_restatement_equals_load_img(geom):
    (ws, hs), (W, H) = geom
    rgb = random_frames(1, hs, ws, seed=hs * 5 + ws)[0]
    want = load_img_body(rgb, H, W)
    got = host_restated(rgb, H, W)
    assert got.dtype == torch.float32 and torch.equal(got, want)


def test_embedder_options_are_sample_utils():
    # sample_utils.py:83-93
    assert ingest.embedder_options({"fps_id", "motion_bucket_id", "cond_aug", "cond_frames"}) == \
        {"fps": 10, "fps_id": 9, "motion_bucket_id": 127}
    assert ingest.embedder_options({"cond_frames"}) == {}


def test_check_frames_rejects_malformed_input():
    good = torch.zeros(2, 9, 16, 3, dtype=torch.uint8)
    ingest.check_frames(good, 8, 16, min_frames=2)
    for bad, H, W in ((good.float(), 8, 16), (good[..., :2], 8, 16), (good[0], 8, 16), (good, 12, 16), (good, 8, 20),
                      (good, 0, 16), (good[:, :0], 8, 16), (good.numpy(), 8, 16)):
        with pytest.raises(ValueError):
            ingest.check_frames(bad, H, W)
    with pytest.raises(ValueError):
        ingest.check_frames(good, 8, 16, min_frames=3)


# The ingest kernels (csrc/ingest/) and the tests that hold them: the same rule KERNEL_TESTS of
# tests/test_conformance_small_cpu.py applies to the kernels at the top of csrc/.
INGEST_KERNEL_TESTS = {
    "resize_h_kernel": ["test_ingest_gpu.py::test_frames_from_u8_equals_load_img",
                        "test_ingest_gpu.py::test_frames_from_u8_25_nuscenes_frames"],
    "resize_v_kernel": ["test_ingest_gpu.py::test_frames_from_u8_equals_load_img",
                        "test_ingest_gpu.py::test_frames_from_u8_25_nuscenes_frames"],
}
_KERNEL = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(")


def kernels_under(directory):
    """Names of every __global__ function in the .cu / .cuh files under ``directory``, subdirectories included."""
    names = set()
    for d, _, files in os.walk(directory):
        for f in sorted(files):
            if f.endswith((".cu", ".cuh")):
                names.update(_KERNEL.findall(open(os.path.join(d, f)).read()))
    return names


def test_every_kernel_under_csrc_has_a_conformance_test():
    """Every kernel under vista_b200/csrc/ is held by a conformance test (KERNEL_TESTS, INGEST_KERNEL_TESTS) or left out
    with a reason (NOT_HELD); the ingest entries name kernels of csrc/ingest/ and test functions that exist."""
    from test_conformance_small_cpu import KERNEL_TESTS, NOT_HELD, _test_functions
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    csrc = os.path.join(root, "vista_b200", "csrc")
    ingest_kernels = kernels_under(os.path.join(csrc, "ingest"))
    assert set(INGEST_KERNEL_TESTS) == ingest_kernels, (sorted(INGEST_KERNEL_TESTS), sorted(ingest_kernels))
    held = set(KERNEL_TESTS) | set(NOT_HELD) | set(INGEST_KERNEL_TESTS)
    assert not kernels_under(csrc) - held, f"kernels without a conformance test: {sorted(kernels_under(csrc) - held)}"
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    for k, ids in INGEST_KERNEL_TESTS.items():
        for tid in ids:
            f, fn = tid.split("::")
            assert fn in _test_functions(os.path.join(tests_dir, f)), f"{k}: {tid} does not exist"
