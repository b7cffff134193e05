"""CPU emulation of the CLIP tower's operators (b200v_clip_preprocess, b200v_attention_d80, the erf-GELU epilogue of
b200v_gemm), on top of tests/fake_ops.py, for testing vista_b200.clip's host executor without a GPU.  Same rounding points
as the kernels: fp16 operands and outputs, fp32 arithmetic in between."""
import contextlib

import torch
import torch.nn.functional as F

import fake_ops
from oracle import clip_oracle


def gemm(a, w, out, *, act=0, **kw):
    if act != 3:
        return fake_ops.gemm(a, w, out, act=act, **kw)
    tmp = torch.empty(out.shape, dtype=torch.float32)
    fake_ops.gemm(a, w, tmp, act=0, **kw)
    out.copy_(F.gelu(tmp).to(out.dtype))
    return out


def attention_d80(q, k, v, out, batch, seq, heads):
    def sp(t):
        return t[:, :heads * 80].float().reshape(batch, seq, heads, 80).permute(0, 2, 1, 3)
    o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v))
    out.copy_(o.permute(0, 2, 1, 3).reshape(batch * seq, heads * 80).to(out.dtype))
    return out


def patch_rows(pre: torch.Tensor, k_pad: int) -> torch.Tensor:
    """(n,3,224,224) -> [n*257, k_pad] patch rows in the layout b200v_clip_preprocess writes (zero class-token row)."""
    n = pre.shape[0]
    p = pre.reshape(n, 3, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(n, 256, 588)
    rows = torch.zeros(n, 257, k_pad, dtype=pre.dtype)
    rows[:, 1:, :588] = p
    return rows.reshape(n * 257, k_pad)


def clip_preprocess(x, out, antialias=True):
    out.copy_(patch_rows(clip_oracle.preprocess(x.float(), antialias), out.shape[1]).to(out.dtype))
    return out


@contextlib.contextmanager
def patched_clip_ops():
    """fake_ops.patched_ops() plus the CLIP operators, swapped into vista_b200.ops for the duration of the block."""
    from vista_b200 import ops
    new = {"gemm": gemm, "attention_d80": attention_d80, "clip_preprocess": clip_preprocess}
    with fake_ops.patched_ops():
        saved = {k: getattr(ops, k) for k in new}
        try:
            for k, v in new.items():
                setattr(ops, k, v)
            yield
        finally:
            for k, v in saved.items():
                setattr(ops, k, v)
