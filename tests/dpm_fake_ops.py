"""CPU emulation of b200v_sampler_update_2m, on top of tests/cond_fake_ops.py (and so of fake_ops.patched_ops()), for
testing the DPM-Solver++(2M) sampler's fused loop without a GPU: the same denoised value as fake_ops.sampler_update,
then the 2M step from the coefficient row of the current step.  D_prev is read only on a second-order row (e != 0)."""
import contextlib

from cond_fake_ops import patched_cond_ops
from fake_ops import _f


def sampler_update_2m(x, net_out, cond_frame, mask, scales, coefs, d_prev, sigmas, step_idx, num_steps, T, h, w):
    step = int(step_idx[0])
    sigma = float(sigmas[step])
    c_skip, c_out = 1.0 / (sigma * sigma + 1.0), -sigma * (sigma * sigma + 1.0) ** -0.5
    hw = h * w
    nu = _f(net_out[: T * hw, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    nc = _f(net_out[T * hw:, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    du, dc = nu * c_out + x * c_skip, nc * c_out + x * c_skip
    den = du + _f(scales).reshape(T, 1, 1, 1) * (dc - du)
    a, b, c, e = (float(v) for v in coefs[step])
    dd = c * den if e == 0.0 else c * den - e * d_prev
    xn = a * x - b * dd
    if step + 1 == num_steps and mask is not None and cond_frame is not None:
        m = _f(mask).reshape(T, 1, 1, 1)
        xn = xn * (1.0 - m) + cond_frame * m
    d_prev.copy_(den)
    x.copy_(xn)
    step_idx += 1


@contextlib.contextmanager
def patched_dpm_ops():
    """patched_cond_ops() plus the 2M update, swapped into vista_b200.ops for the duration of the block."""
    from vista_b200 import lib, ops
    with patched_cond_ops():
        saved = ops.sampler_update_2m
        try:
            ops.sampler_update_2m = lambda *a, **k: lib.tape_host(lambda: sampler_update_2m(*a, **k))
            yield
        finally:
            ops.sampler_update_2m = saved
