"""TEST INFRASTRUCTURE: the DPM-Solver++(2M) counterpart of oracle.vista_oracle.euler_edm_sample, in plain torch on the
CPU.  It restates k-diffusion's sample_dpmpp_2m (Lu et al. 2022, arXiv 2211.01095, Algorithm 2) in its own terms
(t = -ln sigma, h = t' - t, r = h_prev / h) rather than through vista_b200.diffusion.dpmpp2m_coefficients, so that the
coefficient table is checked too.  The conditioning frames are re-imposed before every step and after the loop, as in
Vista's sampling.py:105-106,122-123."""
import math

import torch

from oracle import vista_oracle as vo


def dpmpp2m_sample(sd, cfg, noise, c, uc, cond_frame, cond_mask, num_steps, num_frames=25, guider="VanillaCFG",
                   scale=2.5):
    sigmas = vo.edm_sigmas(num_steps)
    s = [float(v) for v in sigmas]
    x = noise.clone() * torch.sqrt(1.0 + sigmas[0] ** 2)
    scales = vo.guider_scales(guider, num_frames, scale)[:, None, None, None]
    keep = (1 - cond_mask)[:, None, None, None]
    put = cond_mask[:, None, None, None]
    replace = bool(cond_mask.any())
    cc = {k: torch.cat((uc[k], c[k]), 0) for k in ("vector", "crossattn", "concat")}
    old, h_last = None, None
    for i in range(num_steps):
        if replace:
            x = x * keep + cond_frame * put
        sig = x.new_ones([x.shape[0]]) * sigmas[i]
        den = vo.denoise(sd, cfg, torch.cat([x] * 2), torch.cat([sig] * 2), cc, torch.cat([cond_mask] * 2), num_frames)
        x_u, x_c = den.chunk(2)
        den = x_u + scales * (x_c - x_u)
        if s[i + 1] == 0.0:
            x = den
        else:
            h = -math.log(s[i + 1]) + math.log(s[i])
            dd = den if old is None else (1 + 1 / (2 * h_last / h)) * den - (1 / (2 * h_last / h)) * old
            x = (s[i + 1] / s[i]) * x - math.expm1(-h) * dd
            h_last = h
        old = den
    if replace:
        x = x * keep + cond_frame * put
    return x
