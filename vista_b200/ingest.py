"""Camera frames in: sample.py's ``load_img`` (sample.py:174-201) on decoded uint8 RGB frames, on the GPU.

``load_img`` centre-crops a frame to the target aspect ratio, resizes it with ``Image.resize((W, H), LANCZOS)`` and applies
``ToTensor()`` and ``x * 2 - 1``.  Pillow's 8-bit resampler (Resample.c) is integer arithmetic once its coefficient
tables exist, so ``lanczos_tables`` restates the table construction in double on the host and the kernel
(csrc/ingest/ingest.cu, ``ops.frames_u8_resize``) only multiplies and adds integers: its bytes are Pillow's, and the fp32 result
is torchvision's ``to_tensor`` followed by ``* 2 - 1``, bit for bit.  Decoding (JPEG / PNG) stays with the caller: a
device decoder's IDCT is not libjpeg's.
"""
from __future__ import annotations

import functools
import math
from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import ops

PRECISION_BITS = 22          # Resample.c: fixed-point fraction bits of the 8-bit passes
LANCZOS_SUPPORT = 3.0


class Tables(NamedTuple):
    """One axis of the resampler: output index i reads inputs [bounds[i, 0], bounds[i, 0] + bounds[i, 1]) with the first
    bounds[i, 1] weights of row i (int32, 2^22 = 1.0, zero padded to ksize)."""
    bounds: np.ndarray       # (out, 2) int32: xmin, n
    weights: np.ndarray      # (out, ksize) int32
    ksize: int


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    # truncated sinc (Resample.c lanczos_filter); math.sin is the C library's sin, as in Pillow
    if -3.0 <= x < 3.0:
        return _sinc(x) * _sinc(x / 3.0)
    return 0.0


@functools.lru_cache(maxsize=None)
def lanczos_tables(in_size: int, out_size: int) -> Tables:
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc (Resample.c) for LANCZOS from ``in_size`` to ``out_size``
    samples along one axis, the whole input as the box."""
    if in_size <= 0 or out_size <= 0:
        raise ValueError(f"lanczos_tables: sizes must be positive, got {in_size} -> {out_size}")
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = LANCZOS_SUPPORT * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), np.int32)
    weights = np.zeros((out_size, ksize), np.int32)
    one = float(1 << PRECISION_BITS)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        bounds[xx] = (xmin, xmax)
        weights[xx, :xmax] = [int(-0.5 + w * one) if w < 0 else int(0.5 + w * one) for w in k]
    bounds.setflags(write=False)
    weights.setflags(write=False)
    return Tables(bounds, weights, ksize)


def crop_box(ori_w: int, ori_h: int, W: int, H: int) -> Tuple[int, int, int, int]:
    """(left, top, right, bottom) of load_img's centre crop (sample.py:185-194), its arithmetic verbatim: a float compare
    of the aspect ratios, the target width / height truncated, and an odd margin's extra pixel on the right / bottom."""
    if ori_w / ori_h > W / H:
        tmp_w = int(W / H * ori_h)
        return (ori_w - tmp_w) // 2, 0, (ori_w + tmp_w) // 2, ori_h
    if ori_w / ori_h < W / H:
        tmp_h = int(H / W * ori_w)
        return 0, (ori_h - tmp_h) // 2, ori_w, (ori_h + tmp_h) // 2
    return 0, 0, ori_w, ori_h


_device_tables: Dict[Tuple[int, int, torch.device], Tuple[torch.Tensor, torch.Tensor, int]] = {}


def device_tables(in_size: int, out_size: int, device) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """``lanczos_tables`` on ``device`` (bounds, weights, ksize), uploaded once per geometry and device."""
    key = (in_size, out_size, torch.device(device))
    t = _device_tables.get(key)
    if t is None:
        tab = lanczos_tables(in_size, out_size)
        t = _device_tables[key] = (torch.from_numpy(tab.bounds.copy()).to(device),
                                   torch.from_numpy(tab.weights.copy()).to(device), tab.ksize)
    return t


def frames_u8_resize(frames: torch.Tensor, height: int, width: int) -> torch.Tensor:
    """load_img's crop, LANCZOS resize, ToTensor and ``* 2 - 1`` on uint8 RGB frames (T, Hs, Ws, 3) on a CUDA device
    -> fp32 (T, 3, height, width) on that device.  Each pixel's three bytes must be adjacent; rows and frames may be
    strided.  The crop is read in place, and only the rows the vertical pass reads are resized horizontally."""
    T, Hs, Ws, _ = frames.shape
    dev = frames.device
    if frames.stride(3) != 1 or frames.stride(2) != 3:
        frames = frames.contiguous()
    left, top, right, bottom = crop_box(Ws, Hs, width, height)
    cw, ch = right - left, bottom - top
    xt = device_tables(cw, width, dev) if cw != width else None        # Pillow skips a pass whose size is unchanged
    yt = None
    y_first, y_rows = 0, ch
    if ch != height:
        yt = device_tables(ch, height, dev)
        b = lanczos_tables(ch, height).bounds
        y_first, y_rows = int(b[0, 0]), int(b[-1, 0] + b[-1, 1] - b[0, 0])   # Pillow's ybox_first / ybox_last
    scratch = torch.empty(T * y_rows * width * 3, dtype=torch.uint8, device=dev) if xt is not None else None
    out = torch.empty(T, 3, height, width, dtype=torch.float32, device=dev)
    return ops.frames_u8_resize(frames, (left, top, cw, ch), out, xt, yt, y_first, y_rows, scratch)


def embedder_options(keys) -> Dict:
    """sample_utils.init_embedder_options (sample_utils.py:83-93): fps 10, fps_id 9 and motion_bucket_id 127 for the
    conditioner's input keys that ask for them."""
    value_dict = {}
    for key in keys:
        if key in ("fps_id", "fps"):
            value_dict["fps"] = 10
            value_dict["fps_id"] = 9
        elif key == "motion_bucket_id":
            value_dict["motion_bucket_id"] = 127
    return value_dict


def check_frames(frames, height: int, width: int, min_frames: Optional[int] = None):
    """ValueError unless ``frames`` is a uint8 (T, Hs, Ws, 3) tensor and the target size is a positive multiple of 8."""
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
        raise ValueError(f"frames must be a uint8 tensor, got {getattr(frames, 'dtype', type(frames))}")
    if frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError(f"frames must be (T, H, W, 3) RGB, got shape {tuple(frames.shape)}")
    if min(frames.shape[:3]) <= 0:
        raise ValueError(f"frames must not be empty, got shape {tuple(frames.shape)}")
    if min_frames is not None and frames.shape[0] < min_frames:
        raise ValueError(f"{min_frames} frames needed, got {frames.shape[0]}")
    for name, v in (("height", height), ("width", width)):
        if not isinstance(v, int) or v <= 0 or v % 8:
            raise ValueError(f"{name} must be a positive multiple of 8 (the encoder's stride), got {v}")
