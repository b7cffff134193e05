"""CPU emulation of b200v_sampler_update_action, on top of tests/dpm_fake_ops.py (and so of fake_ops.patched_ops()), for
testing action guidance's fused loop without a GPU: the three denoised values D_u, D_img, D_c from rows t and T + t of
net_out and row t of net_img, D = D_u + s_img (D_img - D_u) + s_act (D_c - D_img) in the kernel's order, then the Euler
step (coefs and d_prev None) or the 2M step (both given), as fake_ops.sampler_update and dpm_fake_ops.sampler_update_2m
take them."""
import contextlib

from dpm_fake_ops import patched_dpm_ops
from fake_ops import _f


def sampler_update_action(x, net_out, net_img, cond_frame, mask, scales, action_scales, coefs, d_prev, sigmas, step_idx,
                          num_steps, T, h, w):
    assert (coefs is None) == (d_prev is None), "coefs and d_prev are both None (Euler) or both given (2M)"
    step = int(step_idx[0])
    sigma, sigma_next = float(sigmas[step]), float(sigmas[step + 1])
    c_skip, c_out = 1.0 / (sigma * sigma + 1.0), -sigma * (sigma * sigma + 1.0) ** -0.5
    hw = h * w
    nch = lambda t: _f(t[:, :4]).reshape(T, h, w, 4).permute(0, 3, 1, 2)
    nu, nc, ni = nch(net_out[: T * hw]), nch(net_out[T * hw: 2 * T * hw]), nch(net_img[: T * hw])
    du, dc, di = nu * c_out + x * c_skip, nc * c_out + x * c_skip, ni * c_out + x * c_skip
    den = du + _f(scales).reshape(T, 1, 1, 1) * (di - du)
    den = den + _f(action_scales).reshape(T, 1, 1, 1) * (dc - di)
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
def patched_action_ops():
    """patched_dpm_ops() plus the action-guided update, swapped into vista_b200.ops for the duration of the block."""
    from vista_b200 import lib, ops
    with patched_dpm_ops():
        saved = ops.sampler_update_action
        try:
            ops.sampler_update_action = lambda *a, **k: lib.tape_host(lambda: sampler_update_action(*a, **k))
            yield
        finally:
            ops.sampler_update_action = saved
