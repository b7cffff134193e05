"""Loader / builder of the C-ABI shared library ``libvista_b200.so`` (include/vista_b200.h).

The library is built in-tree with nvcc for sm_90a (H100) (``build()``) and loaded with ctypes.
There is no fallback of any kind: if the library is missing or a call fails, a RuntimeError
is raised (SURVEY.md §8b "Error convention").
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
from typing import List, Optional

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libvista_b200.so")
SOURCES = ["host.cu", "gemm_tc.cu", "gemm_tn_32_256.cu", "gemm_tn_64_224.cu", "gemm_tn_96_192.cu", "gemm_tn_128_160.cu",
           "attn_tc.cu", "misc.cu", "glue.cu", "peer.cu", "clip.cu", "cond.cu", "ingest/ingest.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(d, f) for d, _, files in os.walk(CSRC) for f in files] + [os.path.join(ROOT, "include", "vista_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu of csrc/ for sm_90a and link libvista_b200.so in-tree."""
    if not force and not _stale():
        return LIB_PATH
    nvcc = _nvcc()
    objdir = os.path.join(PKG_DIR, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        os.makedirs(os.path.dirname(obj), exist_ok=True)
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out:
            print(out)
    cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    return LIB_PATH


# ----------------------------------------------------------------------------------------------
# ctypes binding
# ----------------------------------------------------------------------------------------------
class GemmDesc(C.Structure):
    """Mirror of ``b200v_gemm_desc`` (include/vista_b200.h)."""
    _fields_ = [
        ("a", C.c_void_p), ("lda", C.c_int64), ("tokens", C.c_int64), ("a_mode", C.c_int32),
        ("W", C.c_int32), ("H", C.c_int32), ("NB", C.c_int32),
        ("box_w", C.c_int32), ("box_h", C.c_int32), ("box_b", C.c_int32),
        ("cin", C.c_int32), ("ntaps", C.c_int32), ("dh", C.c_int32 * 9), ("dw", C.c_int32 * 9),
        ("b", C.c_void_p), ("N", C.c_int32), ("tile_n", C.c_int32), ("bf16", C.c_int32),
        ("out", C.c_void_p), ("ldo", C.c_int64), ("out_f32", C.c_int32), ("act", C.c_int32),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("ld_rowvec", C.c_int64),
        ("rv_div", C.c_int32), ("rv_mod", C.c_int32),
        ("res1", C.c_void_p), ("ld_res1", C.c_int64), ("s_res1", C.c_float),
        ("res2", C.c_void_p), ("ld_res2", C.c_int64), ("s_res2", C.c_float),
        ("s_acc", C.c_float),
        ("stats", C.c_void_p), ("stats_ld", C.c_int64), ("stats_col0", C.c_int32), ("h_pad", C.c_int32),
    ]


SINUSOID_MAX_SLOTS = 16


class SinusoidSlot(C.Structure):
    """Mirror of ``b200v_sinusoid_slot`` (include/vista_b200.h)."""
    _fields_ = [("value_col", C.c_int32), ("num_features", C.c_int32), ("outdim", C.c_int32), ("dst_col", C.c_int32),
                ("zero", C.c_int32), ("freq_off", C.c_int32)]


class SinusoidTable(C.Structure):
    """Mirror of ``b200v_sinusoid_table``."""
    _fields_ = [("n_slots", C.c_int32), ("slot", SinusoidSlot * SINUSOID_MAX_SLOTS)]


_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float

# name -> argtypes; every function returns int (0 = ok).  Must list every symbol of the header.
SIGNATURES = {
    "b200v_version": [],
    "b200v_device_info": [_P, _P, _P],
    "b200v_gemm": [C.POINTER(GemmDesc), _P],
    "b200v_attention_spatial_v3": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _P],
    "b200v_attention_spatial_v7": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _P],
    "b200v_attention_temporal": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _I32, _P],
    "b200v_groupnorm_from_partials": [_P, _I64, _I32, _I32, _I32, _I32, _I32, _F, _P, _P, _P],
    "b200v_groupnorm_chunk": [],
    "b200v_groupnorm_chunk_for": [C.c_int32, C.c_int32],
    "b200v_groupnorm_sums": [_P, _I64, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P],
    "b200v_groupnorm_finalize": [_P, _I32, C.c_double, _F, _P, _P],
    "b200v_attention_temporal_sharded": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _I32, _I32, _P, _P],
    "b200v_groupnorm_stats": [_P, _I64, _I32, _I32, _I32, _I32, _I32, _F, _P, _P, _P, _P],
    "b200v_groupnorm_apply": [_P, _I64, _P, _I64, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _I32, _P],
    "b200v_layernorm": [_P, _I64, _P, _I64, _I64, _I32, _P, _P, _F, _P, _I64, _I32, _I32, _P],
    "b200v_conv3x3_small_cin": [_P, _I32, _P, _P, _P, _I64, _I32, _I32, _I32, _I32, _P],
    "b200v_conv3x3_small_cout": [_P, _I64, _I32, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_im2col_s2": [_P, _I64, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_im2col_s2_asym": [_P, _I64, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_upsample2x": [_P, _I64, _P, _I64, _I32, _I32, _I32, _I32, _P],
    "b200v_timestep_embedding": [_P, _I32, _I32, _F, _P, _I64, _P],
    "b200v_blend_emb": [_P, _P, _P, _P, _P, _P, _I32, _I32, _P],
    "b200v_sampler_prepare": [_P, _P, _P, _P, _P, _P, _P, _P, _I64, _P, _I32, _I32, _I32, _P],
    "b200v_sampler_update": [_P, _P, _I64, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_sampler_update_2m": [_P, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_sampler_update_action": [_P, _P, _I64, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_sampler_update_cond": [_P, _P, _I64, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_softmax_rows": [_P, _I64, _P, _I64, _I64, _I32, _P],
    "b200v_time_mix_small": [_P, _I64, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _P],
    "b200v_time_mix_small_u8": [_P, _I64, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    "b200v_rollout_advance": [_P, _P, _P, _P, _I32, _I64, _I32, _I32, _I32, _P],
    "b200v_ensemble_reward_scratch": [],
    "b200v_ensemble_reward": [_P, _I32, _I64, _P, _P, _P, _P],
    "b200v_peer_alloc": [_I64, C.POINTER(C.c_void_p), _P],
    "b200v_peer_open": [_P, C.POINTER(C.c_void_p)],
    "b200v_peer_close": [_P],
    "b200v_peer_free": [_P],
    "b200v_peer_allreduce_max": [],
    "b200v_peer_allreduce_f64": [_P, _I32, _P, _I64, _I64, _I32, _I32, _P, _P],
    "b200v_peer_put": [_P, _I64, _I64, _I64, _P, _I64, _P, _I32, _P, _P, _P],
    "b200v_peer_wait": [_P, _I32, _P, _P],
    "b200v_clip_preprocess": [_P, _I32, _I32, _I32, _I32, _P, _I64, _I32, _P],
    "b200v_attention_d80": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _P],
    "b200v_nchw_to_tokens": [_P, _P, _I64, _I32, _I32, _I32, _I32, _P],
    "b200v_tokens_to_nchw": [_P, _I32, _I64, _P, _I32, _I32, _I32, _I32, _P],
    "b200v_sinusoid_embed": [_P, _I64, _I32, C.POINTER(SinusoidTable), _P, _P, _I64, _P],
    "b200v_frames_u8_resize": [_P, _I64, _I64, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _I32, _P, _P,
                               _I32, _I32, _I32, _P, _P, _P],
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """dlopen the in-tree library (must have been built); binds all signatures."""
    global _lib
    if _lib is not None:
        return _lib if _tape is None else _Recorder(_lib)
    if os.path.isfile(LIB_PATH) and _stale() and os.environ.get("VISTA_B200_NO_AUTOBUILD") != "1":
        try:                      # sources newer than the library (an edit without a rebuild): rebuild before dlopen
            build()
        except Exception as e:    # no nvcc on this host: the symbol check below reports what is missing
            sys.stderr.write(f"vista_b200: stale library and rebuild failed: {e}\n")
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no fallback path)")
    lib = C.CDLL(LIB_PATH)
    lib.b200v_last_error.restype = C.c_char_p
    lib.b200v_last_error.argtypes = []
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = C.c_int
        fn.argtypes = argtypes
    _lib = lib
    return lib


# ---------------------------------------------------------------------------------------------------------------
# Launch tape.  The executor issues the same C-ABI calls with the same arguments every sampler step (all buffers are
# persistent), so one recorded step can be replayed without the Python logic above it: `begin_tape()` makes `load()`
# hand out a recording proxy, `end_tape()` returns [(callable, args)]; host-side operations that must stay in order
# with the kernels (torch.distributed collectives, tensor copies) are added with `tape_host()`.  Used where a CUDA
# graph is not (the frame-sharded step with its NCCL calls); the same stability rules as for graph capture apply.
# ---------------------------------------------------------------------------------------------------------------
_tape: Optional[list] = None
_NO_TAPE = {"b200v_peer_alloc", "b200v_peer_open", "b200v_peer_close", "b200v_peer_free", "b200v_peer_allreduce_max", "b200v_ensemble_reward_scratch", "b200v_groupnorm_chunk", "b200v_groupnorm_chunk_for", "b200v_version", "b200v_device_info", "b200v_last_error"}


class _Recorder:
    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name in _NO_TAPE:
            return fn

        def call(*args):
            if _tape is not None:
                _tape.append((fn, args))
            return fn(*args)
        return call


def begin_tape():
    global _tape
    _tape = []


def end_tape() -> list:
    global _tape
    t, _tape = _tape, None
    return t


def taping() -> bool:
    return _tape is not None


HOST_PROFILE = None     # (begin(family, detail, flops, bytes), end()): brackets host-side operations with CUDA events (bench.py)


def tape_host(fn, detail: str = "host"):
    """Run a host-side operation now and, while a tape is being recorded, put it on the tape."""
    if _tape is not None:
        _tape.append((fn, ()))
    if HOST_PROFILE is not None:
        HOST_PROFILE[0]("nccl+host", detail, 0.0, 0.0)
        r = fn()
        HOST_PROFILE[1]()
        return r
    return fn()


def replay(tape: list):
    for fn, args in tape:
        rc = fn(*args)
        if type(rc) is int and rc != 0:
            check(rc, "replayed call")


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().b200v_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"vista_b200 C-ABI call {what} failed (rc={rc}): {msg}")


def exported_symbols() -> List[str]:
    return ["b200v_last_error"] + list(SIGNATURES)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
