"""Diffusion mechanics with the reference's public surface (names, constructor arguments, call
signatures, error behaviour) — so that ``sample_utils.do_sample`` / ``DiffusionEngine.sample`` style
callers work unchanged — plus the fused B200 loop.

Mirrors (paths relative to the reference root):
  EDMDiscretization ........ vwm/modules/diffusionmodules/discretizer.py:15-37
  VScalingWithEDMcNoise & co vwm/modules/diffusionmodules/denoiser_scaling.py
  Denoiser ................. vwm/modules/diffusionmodules/denoiser.py:10-35
  VanillaCFG / Identity / Linear / TrianglePredictionGuider ... guiders.py
  ActionCFG ................ a separate guidance scale for the action (not in Vista; InstructPix2Pix's two-scale CFG)
  IntervalCFG .............. guidance on a sigma interval only (not in Vista; Kynkäänniemi et al. 2024)
  cache_schedule ........... which steps run the whole UNet under feature caching (not in Vista; Ma et al. 2024)
  EulerEDMSampler .......... vwm/modules/diffusionmodules/sampling.py:15-124
  DPMPP2MSampler ........... sgm's sampling.py DPMPP2MSampler (Vista does not ship it), on the same loop
  instantiate_from_config .. vwm/util.py:154-173

The generic path keeps the reference's step algebra in torch (a dozen tiny fp32 ops per step on a
(25,4,h,w) latent); the network call is where the time goes and that is the B200 executor.  When the
network is a ``B200Wrapper`` the sampler switches to the fused loop (``fused_sample``): two small CUDA
kernels per step around the UNet, no host synchronisation, no per-step tensor allocation.
"""
from __future__ import annotations

import importlib
import math
from typing import Dict, List, Optional, Union

import torch
import torch.nn as nn


# ----------------------------------------------------------------------------------------------
# config plumbing
# ----------------------------------------------------------------------------------------------
def get_obj_from_str(string: str):
    module, cls = string.rsplit(".", 1)
    return getattr(importlib.import_module(module, package=None), cls)


def instantiate_from_config(config):
    if "target" not in config:
        if config in ("__is_first_stage__", "__is_unconditional__"):
            return None
        raise KeyError("Expected key `target` to instantiate")
    return get_obj_from_str(config["target"])(**config.get("params", dict()))


def append_dims(x: torch.Tensor, target_dims: int) -> torch.Tensor:
    d = target_dims - x.ndim
    if d < 0:
        raise ValueError(f"Input has {x.ndim} dims but target_dims is {target_dims}, which is less")
    return x[(...,) + (None,) * d]


# ----------------------------------------------------------------------------------------------
# discretisation / scalings
# ----------------------------------------------------------------------------------------------
class EDMDiscretization:
    def __init__(self, sigma_min: float = 0.002, sigma_max: float = 80.0, rho: float = 7.0):
        self.sigma_min, self.sigma_max, self.rho = sigma_min, sigma_max, rho

    def get_sigmas(self, n: int, device="cpu") -> torch.Tensor:
        ramp = torch.linspace(0, 1, n, device=device)
        min_inv_rho = self.sigma_min ** (1 / self.rho)
        max_inv_rho = self.sigma_max ** (1 / self.rho)
        return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** self.rho

    def __call__(self, n: int, do_append_zero: bool = True, device="cpu", flip: bool = False) -> torch.Tensor:
        sigmas = self.get_sigmas(n, device=device)
        if do_append_zero:
            sigmas = torch.cat((sigmas, sigmas.new_zeros([1])))
        return sigmas if not flip else torch.flip(sigmas, (0,))


class EDMScaling:
    def __init__(self, sigma_data: float = 0.5):
        self.sigma_data = sigma_data

    def __call__(self, sigma):
        c_skip = self.sigma_data ** 2 / (sigma ** 2 + self.sigma_data ** 2)
        c_out = sigma * self.sigma_data / (sigma ** 2 + self.sigma_data ** 2) ** 0.5
        c_in = 1 / (sigma ** 2 + self.sigma_data ** 2) ** 0.5
        return c_skip, c_out, c_in, 0.25 * sigma.log()


class EpsScaling:
    def __call__(self, sigma):
        return torch.ones_like(sigma), -sigma, 1 / (sigma ** 2 + 1.0) ** 0.5, sigma.clone()


class VScaling:
    def __call__(self, sigma):
        return 1.0 / (sigma ** 2 + 1.0), -sigma / (sigma ** 2 + 1.0) ** 0.5, 1.0 / (sigma ** 2 + 1.0) ** 0.5, sigma.clone()


class VScalingWithEDMcNoise:
    def __call__(self, sigma):
        c_skip = 1.0 / (sigma ** 2 + 1.0)
        c_out = -sigma / (sigma ** 2 + 1.0) ** 0.5
        c_in = 1.0 / (sigma ** 2 + 1.0) ** 0.5
        c_noise = 0.25 * sigma.log()
        return c_skip, c_out, c_in, c_noise


class Denoiser(nn.Module):
    def __init__(self, scaling_config: Dict, num_frames: int = 25):
        super().__init__()
        self.scaling = instantiate_from_config(scaling_config)
        self.num_frames = num_frames

    def possibly_quantize_sigma(self, sigma):
        return sigma

    def possibly_quantize_c_noise(self, c_noise):
        return c_noise

    def forward(self, network: nn.Module, noised_input: torch.Tensor, sigma: torch.Tensor, cond: Dict,
                cond_mask: torch.Tensor):
        sigma = self.possibly_quantize_sigma(sigma)
        sigma_shape = sigma.shape
        sigma = append_dims(sigma, noised_input.ndim)
        c_skip, c_out, c_in, c_noise = self.scaling(sigma)
        c_noise = self.possibly_quantize_c_noise(c_noise.reshape(sigma_shape))
        return network(noised_input * c_in, c_noise, cond, cond_mask, self.num_frames) * c_out + noised_input * c_skip


# ----------------------------------------------------------------------------------------------
# guiders
# ----------------------------------------------------------------------------------------------
class Guider:
    additional_cond_keys: List[str] = []

    def scale_vector(self, num_frames: int) -> torch.Tensor:
        """Per-frame guidance scale (fused path)."""
        raise NotImplementedError

    def _merge(self, c, uc):
        c_out = dict()
        for k in c:
            if k in ["vector", "crossattn", "concat"] + list(self.additional_cond_keys):
                c_out[k] = torch.cat((uc[k], c[k]), 0)
            else:
                assert c[k] == uc[k]
                c_out[k] = c[k]
        return c_out


class VanillaCFG(Guider):
    def __init__(self, scale: float):
        self.scale = scale

    def __call__(self, x, sigma):
        x_u, x_c = x.chunk(2)
        return x_u + self.scale * (x_c - x_u)

    def prepare_inputs(self, x, s, c, cond_mask, uc):
        return torch.cat([x] * 2), torch.cat([s] * 2), self._merge(c, uc), torch.cat([cond_mask] * 2)

    def scale_vector(self, num_frames):
        return torch.full((num_frames,), float(self.scale))


class IdentityGuider(Guider):
    def __call__(self, x, sigma):
        return x

    def prepare_inputs(self, x, s, c, cond_mask, uc):
        return x, s, {k: c[k] for k in c}, cond_mask


class LinearPredictionGuider(Guider):
    def __init__(self, num_frames: int = 25, max_scale: float = 2.5, min_scale: float = 1.0,
                 additional_cond_keys: Optional[Union[List[str], str]] = None):
        self.min_scale, self.max_scale, self.num_frames = min_scale, max_scale, num_frames
        self.scale = torch.linspace(min_scale, max_scale, num_frames).unsqueeze(0)
        keys = additional_cond_keys or list()
        self.additional_cond_keys = [keys] if isinstance(keys, str) else list(keys)

    def __call__(self, x, sigma):
        x_u, x_c = x.chunk(2)
        T = self.num_frames
        shp = x_u.shape
        x_u = x_u.reshape(shp[0] // T, T, *shp[1:])
        x_c = x_c.reshape(shp[0] // T, T, *shp[1:])
        scale = append_dims(self.scale.expand(x_u.shape[0], T), x_u.ndim).to(x_u.device)
        return (x_u + scale * (x_c - x_u)).reshape(shp)

    def prepare_inputs(self, x, s, c, cond_mask, uc):
        return torch.cat([x] * 2), torch.cat([s] * 2), self._merge(c, uc), torch.cat([cond_mask] * 2)

    def scale_vector(self, num_frames):
        assert num_frames == self.num_frames
        return self.scale[0].clone()


class TrianglePredictionGuider(LinearPredictionGuider):
    def __init__(self, num_frames: int = 25, max_scale: float = 2.5, min_scale: float = 1.0, period=1.0,
                 period_fusing: str = "max", additional_cond_keys=None):
        super().__init__(num_frames, max_scale, min_scale, additional_cond_keys)
        values = torch.linspace(0, 1, num_frames)
        periods = [period] if isinstance(period, float) else list(period)
        scales = [self.triangle_wave(values, p) for p in periods]
        if period_fusing == "mean":
            scale = sum(scales) / len(periods)
        elif period_fusing == "multiply":
            scale = torch.prod(torch.stack(scales), dim=0)
        elif period_fusing == "max":
            scale = torch.max(torch.stack(scales), dim=0).values
        else:
            raise NotImplementedError
        self.scale = (scale * (max_scale - min_scale) + min_scale).unsqueeze(0)

    @staticmethod
    def triangle_wave(values, period):
        return 2 * (values / period - torch.floor(values / period + 0.5)).abs()


class ActionCFG(Guider):
    """Classifier-free guidance with a separate scale for the driving action (Brooks et al. 2023, InstructPix2Pix,
    arXiv 2211.09800, eq. 3; Liu et al. 2022, Composable Diffusion):

        D = D_u + s_img (D_img - D_u) + s_act (D_c - D_img)

    D_u and D_c are the denoiser on ``uc`` and ``c``; D_img is the denoiser on ``c`` with every action slot zeroed
    (``action_free``), which Vista's action training puts in distribution (each action embedder is dropped on its own,
    ucg_rate 0.15).  ``guider_config`` is the image guider (VanillaCFG, Linear- or TrianglePredictionGuider): it gives
    the per-frame s_img and applies the image term; ``action_scale`` is s_act for every frame.  With s_act == s_img this
    is the image guider alone; with no action in ``c``, D_c == D_img.  One more network evaluation per step on the
    conditional rows."""

    def __init__(self, action_scale: float, guider_config: Dict, context_dim: int = 1024):
        self.action_scale = float(action_scale)
        self.image_guider = instantiate_from_config(guider_config)
        if isinstance(self.image_guider, IntervalCFG):
            raise ValueError("IntervalCFG must be the outermost guider: wrap ActionCFG in it, not the other way round")
        self.context_dim = context_dim
        self.additional_cond_keys = list(self.image_guider.additional_cond_keys)

    def action_free(self, c: Dict) -> Dict:
        """``c`` with its action slots zeroed: every action key is a crossattn slot in the columns after the CLIP
        embedding's ``context_dim``, and a zeroed or missing action key is a zero slot (encoders/modules.py:128-130).
        The other keys are shared, not copied."""
        out = dict(c)
        ctx = c["crossattn"].clone()
        ctx[..., self.context_dim:] = 0.0
        out["crossattn"] = ctx
        return out

    def __call__(self, x, sigma):
        x_u, x_img, x_c = x.chunk(3)
        return self.image_guider(torch.cat((x_u, x_img)), sigma) + self.action_scale * (x_c - x_img)

    def prepare_inputs(self, x, s, c, cond_mask, uc):
        """Three batches (uc, action-free c, c): crossattn from those three, every other merged key from (uc, c, c)."""
        c_img = self.action_free(c)
        c_out = dict()
        for k in c:
            if k == "crossattn":
                c_out[k] = torch.cat((uc[k], c_img[k], c[k]), 0)
            elif k in ["vector", "concat"] + list(self.additional_cond_keys):
                c_out[k] = torch.cat((uc[k], c[k], c[k]), 0)
            else:
                assert c[k] == uc[k]
                c_out[k] = c[k]
        return torch.cat([x] * 3), torch.cat([s] * 3), c_out, torch.cat([cond_mask] * 3)

    def scale_vector(self, num_frames):
        return self.image_guider.scale_vector(num_frames)

    def action_scale_vector(self, num_frames):
        """Per-frame s_act (fused path): ``action_scale`` on every frame."""
        return torch.full((num_frames,), self.action_scale)


class IntervalCFG(Guider):
    """Limited-interval guidance (Kynkäänniemi et al. 2024, arXiv 2404.07724): the wrapped guider on the steps whose
    sigma lies in (sigma_lo, sigma_hi], guidance weight 1 on every other step.  At weight 1 each guider it may wrap
    (VanillaCFG, Linear- or TrianglePredictionGuider, ActionCFG) gives D = D_c, so an unguided step evaluates the
    network on the T conditional rows only, half the rows of a CFG step.

    Whether a step is guided is decided per call from its sigma (the value of the fp32 sigma table the sampler reads):
    ``prepare_inputs`` is the wrapped guider's inside the interval and passes ``(x, s, c, cond_mask)`` through outside
    it; ``__call__`` is the wrapped guider inside and the identity outside.  It must be the outermost guider."""

    GUIDERS = (VanillaCFG, LinearPredictionGuider, ActionCFG)

    def __init__(self, sigma_lo: float, sigma_hi: float, guider_config: Dict):
        self.sigma_lo, self.sigma_hi = float(sigma_lo), float(sigma_hi)
        if not self.sigma_lo < self.sigma_hi:
            raise ValueError(f"IntervalCFG: sigma_lo ({sigma_lo}) must be below sigma_hi ({sigma_hi})")
        self.guider = instantiate_from_config(guider_config)
        inner = self.guider.image_guider if isinstance(self.guider, ActionCFG) else self.guider
        if not isinstance(self.guider, self.GUIDERS) or not isinstance(inner, (VanillaCFG, LinearPredictionGuider)):
            raise ValueError(f"IntervalCFG wraps VanillaCFG, LinearPredictionGuider, TrianglePredictionGuider or ActionCFG "
                             f"over one of the first three; got {type(self.guider).__name__}")
        self.additional_cond_keys = list(self.guider.additional_cond_keys)

    def guided(self, sigma) -> bool:
        """Whether the step at ``sigma`` (a number, or the step's per-row sigma tensor) is guided."""
        s = float(sigma.reshape(-1)[0]) if isinstance(sigma, torch.Tensor) else float(sigma)
        return self.sigma_lo < s <= self.sigma_hi

    def __call__(self, x, sigma):
        return self.guider(x, sigma) if self.guided(sigma) else x

    def prepare_inputs(self, x, s, c, cond_mask, uc):
        if self.guided(s):
            return self.guider.prepare_inputs(x, s, c, cond_mask, uc)
        return x, s, {k: c[k] for k in c}, cond_mask

    def scale_vector(self, num_frames):
        return self.guider.scale_vector(num_frames)


# ----------------------------------------------------------------------------------------------
# feature caching
# ----------------------------------------------------------------------------------------------
def _check_cache_args(cache_interval, cache_branch):
    for name, v, lo in (("cache_interval", cache_interval, 1), ("cache_branch", cache_branch, 0)):
        if isinstance(v, bool) or not isinstance(v, int) or v < lo:
            raise ValueError(f"{name} must be an int >= {lo}; got {v!r}")


def cache_schedule(kinds, interval: int) -> List[bool]:
    """Feature caching (Ma et al. 2024, DeepCache, arXiv 2312.00858): which steps run the whole UNet (True) and which
    reuse the deep feature of the last full step and run only the outermost blocks (False).  ``kinds[i]`` is step i's
    kind of network call (guided or not, under IntervalCFG or IdentityGuider); a step is full if it is the first, if its
    kind differs from step i-1's, or if ``interval`` steps have passed since the last full step.  A cached step reads the
    feature its own kind's rows left, so a kind change always starts with a full step."""
    _check_cache_args(interval, 0)
    full, last = [], 0
    for i, k in enumerate(kinds):
        f = i == 0 or k != kinds[i - 1] or i - last >= interval
        if f:
            last = i
        full.append(f)
    return full


# ----------------------------------------------------------------------------------------------
# sampler
# ----------------------------------------------------------------------------------------------
class B200Denoiser:
    """Callable handed to the sampler by our engine: same ``(x, sigma, c, cond_mask)`` signature as the
    reference's lambda (sample_utils.py:314-315), but it also exposes the pieces so that the sampler can
    run the fused loop."""

    def __init__(self, denoiser: Denoiser, network: nn.Module):
        self.denoiser, self.network = denoiser, network

    def __call__(self, x, sigma, c, cond_mask):
        return self.denoiser(self.network, x, sigma, c, cond_mask)


def _unwrap_reference_closure(fn):
    """The reference's callers hand the sampler a local closure, ``def denoiser(x, sigma, cond, cond_mask): return
    model.denoiser(model.model, x, sigma, cond, cond_mask)`` (sample_utils.py:314-315, diffusion.py:324-325), which
    hides the engine.  When that engine's network is a B200Wrapper and its denoiser is ours, recover the pair so that an
    UNMODIFIED ``do_sample`` / ``DiffusionEngine.sample`` runs the fused loop; anything else is returned untouched."""
    if isinstance(fn, B200Denoiser) or not callable(fn):
        return fn
    cells = getattr(fn, "__closure__", None) or ()
    from .modules import B200Wrapper
    for cell in cells:
        try:
            obj = cell.cell_contents
        except ValueError:          # empty cell
            continue
        net, den = getattr(obj, "model", None), getattr(obj, "denoiser", None)
        if isinstance(net, B200Wrapper) and isinstance(den, Denoiser):
            return B200Denoiser(den, net)
    return fn


class BaseDiffusionSampler:
    """``cache_interval`` / ``cache_branch``: feature caching on the fused loop (``cache_schedule``).  With an interval
    k > 1 a full UNet step runs at most every k steps, and the steps between run input blocks 0..b and output blocks
    n-1-b..n-1 on the deep feature of the last full step, b = ``cache_branch``.  1 (the default) runs every step whole.
    Only the fused loop caches: the torch loop, ``s_churn > 0`` and a frame-sharded engine raise NotImplementedError."""

    def __init__(self, discretization_config, num_steps: Optional[int] = None, guider_config=None,
                 verbose: bool = False, device: str = "cuda", cache_interval: int = 1, cache_branch: int = 0):
        _check_cache_args(cache_interval, cache_branch)
        self.num_steps = num_steps
        self.discretization = instantiate_from_config(discretization_config)
        self.guider = instantiate_from_config(guider_config)
        self.verbose = verbose
        self.device = device
        self.cache_interval, self.cache_branch = cache_interval, cache_branch

    def _refuse_cache(self, why: str):
        if self.cache_interval > 1:
            raise NotImplementedError(f"{type(self).__name__}: cache_interval > 1 runs on the fused loop only, not {why}")

    def prepare_sampling_loop(self, x, cond, uc=None, num_steps=None):
        sigmas = self.discretization(self.num_steps if num_steps is None else num_steps, device=self.device)
        uc = cond if uc is None else uc
        x *= torch.sqrt(1.0 + sigmas[0] ** 2)        # in place on the caller's tensor, as the reference does
        num_sigmas = len(sigmas)
        s_in = x.new_ones([x.shape[0]])
        return x, s_in, sigmas, num_sigmas, cond, uc

    def denoise(self, x, denoiser, sigma, cond, cond_mask, uc):
        denoised = denoiser(*self.guider.prepare_inputs(x, sigma, cond, cond_mask, uc))
        return self.guider(denoised, sigma)

    def get_sigma_gen(self, num_sigmas):
        gen = range(num_sigmas - 1)
        if self.verbose:
            from tqdm import tqdm
            gen = tqdm(gen, total=num_sigmas, desc=f"Sampling with {self.__class__.__name__} for {num_sigmas} steps")
        return gen


class EulerEDMSampler(BaseDiffusionSampler):
    def __init__(self, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.s_churn, self.s_tmin, self.s_tmax, self.s_noise = s_churn, s_tmin, s_tmax, s_noise

    def euler_step(self, x, d, dt):
        return x + dt * d

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, cond_mask=None, uc=None, gamma=0.0):
        sigma_hat = sigma * (gamma + 1.0)
        if gamma > 0:
            eps = torch.randn_like(x) * self.s_noise
            x = x + eps * append_dims(sigma_hat ** 2 - sigma ** 2, x.ndim) ** 0.5
        denoised = self.denoise(x, denoiser, sigma_hat, cond, cond_mask, uc)
        d = (x - denoised) / append_dims(sigma_hat, x.ndim)
        dt = append_dims(next_sigma - sigma_hat, x.ndim)
        return self.euler_step(x, d, dt)

    def __call__(self, denoiser, x, cond, uc=None, cond_frame=None, cond_mask=None, num_steps=None):
        denoiser = _unwrap_reference_closure(denoiser)
        if self.s_churn > 0.0:
            self._refuse_cache("with s_churn > 0")
        if isinstance(denoiser, B200Denoiser) and self.s_churn == 0.0 and self._fusable(denoiser, cond, uc):
            from .fused import fused_sample
            return fused_sample(self, denoiser, x, cond, uc, cond_frame, cond_mask, num_steps)
        self._refuse_cache("on the torch loop")
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        replace_cond_frames = cond_mask is not None and bool(cond_mask.any())
        for i in self.get_sigma_gen(num_sigmas):
            if replace_cond_frames:
                x = x * append_dims(1 - cond_mask, x.ndim) + cond_frame * append_dims(cond_mask, cond_frame.ndim)
            gamma = (min(self.s_churn / (num_sigmas - 1), 2 ** 0.5 - 1)
                     if self.s_tmin <= sigmas[i] <= self.s_tmax else 0.0)
            x = self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, cond_mask, uc, gamma)
        if replace_cond_frames:
            x = x * append_dims(1 - cond_mask, x.ndim) + cond_frame * append_dims(cond_mask, cond_frame.ndim)
        return x

    def _fusable(self, denoiser: "B200Denoiser", cond, uc) -> bool:
        from .modules import B200Wrapper
        guider = self.guider.guider if isinstance(self.guider, IntervalCFG) else self.guider
        guider = guider.image_guider if isinstance(guider, ActionCFG) else guider
        return (isinstance(denoiser.network, B200Wrapper) and isinstance(denoiser.denoiser.scaling, VScalingWithEDMcNoise)
                and (isinstance(guider, (VanillaCFG, LinearPredictionGuider)) or type(self.guider) is IdentityGuider)
                and all(k in cond for k in ("crossattn", "vector", "concat")))


def dpmpp2m_coefficients(sigmas: torch.Tensor) -> torch.Tensor:
    """(n, 4) float64 rows {a, b, c, e} of the DPM-Solver++(2M) step x = a x - b (c D - e D_prev) from the n + 1 sigmas
    (Lu et al. 2022, arXiv 2211.01095, Algorithm 2; k-diffusion's sample_dpmpp_2m): with h_i = ln(s_i / s_i+1),
    a = s_i+1 / s_i, b = expm1(-h_i); c = 1 + 1/(2 r), e = 1/(2 r), r = h_i-1 / h_i, except on the first step and on a
    step to sigma = 0, which are first order (c = 1, e = 0; to sigma = 0 that is x = D).  Computed in double from the
    sigma table the loop reads, so the fused kernel, its CPU twin and the torch loop apply the same coefficients."""
    s = [float(v) for v in sigmas.detach().double().cpu()]
    rows, h_prev = [], None
    for i in range(len(s) - 1):
        if s[i + 1] == 0.0:
            rows.append((0.0, -1.0, 1.0, 0.0))
            h_prev = None
            continue
        h = math.log(s[i] / s[i + 1])
        if h_prev is None:
            c, e = 1.0, 0.0
        else:
            e = h / (2.0 * h_prev)          # 1 / (2 r)
            c = 1.0 + e
        rows.append((s[i + 1] / s[i], math.expm1(-h), c, e))
        h_prev = h
    return torch.tensor(rows, dtype=torch.float64).reshape(-1, 4)


class DPMPP2MSampler(BaseDiffusionSampler):
    """DPM-Solver++(2M) (sgm's ``DPMPP2MSampler``): a second-order multistep solver of the sampling ODE at one network
    evaluation per step, like Euler.  Same call as ``EulerEDMSampler``; the conditioning frames are re-imposed before
    every step and after the loop (sampling.py:105-106,122-123), and the fused CUDA-graph loop runs under the same
    conditions as Euler's."""

    def __call__(self, denoiser, x, cond, uc=None, cond_frame=None, cond_mask=None, num_steps=None):
        denoiser = _unwrap_reference_closure(denoiser)
        if isinstance(denoiser, B200Denoiser) and self._fusable(denoiser, cond, uc):
            from .fused import fused_sample
            return fused_sample(self, denoiser, x, cond, uc, cond_frame, cond_mask, num_steps)
        self._refuse_cache("on the torch loop")
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        coefs = dpmpp2m_coefficients(sigmas).tolist()
        replace_cond_frames = cond_mask is not None and bool(cond_mask.any())
        old_denoised = None
        for i in self.get_sigma_gen(num_sigmas):
            if replace_cond_frames:
                x = x * append_dims(1 - cond_mask, x.ndim) + cond_frame * append_dims(cond_mask, cond_frame.ndim)
            denoised = self.denoise(x, denoiser, s_in * sigmas[i], cond, cond_mask, uc)
            a, b, c, e = coefs[i]
            d = c * denoised if e == 0.0 else c * denoised - e * old_denoised
            x = a * x - b * d
            old_denoised = denoised
        if replace_cond_frames:
            x = x * append_dims(1 - cond_mask, x.ndim) + cond_frame * append_dims(cond_mask, cond_frame.ndim)
        return x

    _fusable = EulerEDMSampler._fusable
