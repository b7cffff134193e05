"""CPU emulation of b200v_sampler_update_cond, on top of tests/action_fake_ops.py (and so of fake_ops.patched_ops()), for
testing interval guidance's fused loop without a GPU: D = D_c from the T rows of net_c, in the kernel's order, then the
Euler step (coefs and d_prev None) or the 2M step (both given, D written to d_prev), as
action_fake_ops.sampler_update_action takes them."""
import contextlib

from action_fake_ops import patched_action_ops
from fake_ops import _f


def sampler_update_cond(x, net_c, cond_frame, mask, coefs, d_prev, sigmas, step_idx, num_steps, T, h, w):
    assert (coefs is None) == (d_prev is None), "coefs and d_prev are both None (Euler) or both given (2M)"
    step = int(step_idx[0])
    sigma, sigma_next = float(sigmas[step]), float(sigmas[step + 1])
    c_skip, c_out = 1.0 / (sigma * sigma + 1.0), -sigma * (sigma * sigma + 1.0) ** -0.5
    nc = _f(net_c[: T * h * w, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    den = nc * c_out + x * c_skip
    if coefs is None:
        xn = x + (x - den) / sigma * (sigma_next - sigma)
    else:
        a, b, c, e = (float(v) for v in coefs[step])
        dd = c * den if e == 0.0 else c * den - e * d_prev
        xn = a * x - b * dd
        d_prev.copy_(den)
    if step + 1 == num_steps and mask is not None and cond_frame is not None:
        m = _f(mask).reshape(T, 1, 1, 1)
        xn = xn * (1.0 - m) + cond_frame * m
    x.copy_(xn)
    step_idx += 1


@contextlib.contextmanager
def patched_interval_ops():
    """patched_action_ops() plus the unguided update, swapped into vista_b200.ops for the duration of the block."""
    from vista_b200 import lib, ops
    with patched_action_ops():
        saved = ops._sampler_update_cond
        try:
            ops._sampler_update_cond = lambda *a, **k: lib.tape_host(lambda: sampler_update_cond(*a, **k))
            yield
        finally:
            ops._sampler_update_cond = saved
