"""CPU emulation of b200v_sinusoid_embed, on top of tests/clip_fake_ops.py, for testing vista_b200.conditioner's host logic
without a GPU: the same fp32 product of value and host-computed frequency, then torch's cos / sin."""
import contextlib

import torch

from clip_fake_ops import patched_clip_ops


def sinusoid_embed(values, slots, freqs, out):
    rows = out.shape[0]
    for vc, nf, od, dc, zero, fo in slots:
        half = od // 2
        dst = out[:, dc:dc + nf * od]
        if zero:
            dst.zero_()
            continue
        a = values[:, vc:vc + nf].reshape(rows * nf, 1) * freqs[fo:fo + half].reshape(1, half)
        e = torch.cat([torch.cos(a), torch.sin(a)] + ([torch.zeros(rows * nf, 1)] if od % 2 else []), dim=1)
        dst.copy_(e.reshape(rows, nf * od))
    return out


@contextlib.contextmanager
def patched_cond_ops():
    """patched_clip_ops() plus the sinusoid kernel, swapped into vista_b200.ops for the duration of the block."""
    from vista_b200 import ops
    with patched_clip_ops():
        saved = ops.sinusoid_embed
        try:
            ops.sinusoid_embed = sinusoid_embed
            yield
        finally:
            ops.sinusoid_embed = saved
