"""Trajectory-level conformance, one level above tests/block_shadow.py: a whole sample through ``engine.sample`` as the
product runs it, recorded after every sampler step, against the oracle's trajectory on the same conditioning, latent and
noise.

The launch harness (tests/shadow.py) and the layer harness (tests/block_shadow.py) hold one step to fp64, each piece on
its own inputs and within c x rho of it.  A small *systematic* bias inside that bound (a residual scaled by one fp16
rounding too many, a time-mixer weight off by one fp16 ulp) passes both, and adds up over the 40-odd layers of a step
and the 25 or 50 steps of a sample.  This harness measures that: ours against a high-precision oracle at the steps of
``REPORT_STEPS``, per frame at the last step, and against the reference's own inference precision (the same oracle under
fp16 autocast, the "yardstick") for scale.

Pieces:
  * ``run_ours``: ``engine.sample`` with ``fused._run_steps`` replaced by a copy that clones the loop state after every
    step (same launches, same replay order, same graph keys), in graph or eager mode;
  * ``run_reference``: the oracle's Euler sampler (``euler_edm_sample``) for VanillaCFG / TrianglePredictionGuider, and
    vista_b200.diffusion's torch loop (the sampler object itself, handed a plain function around ``vo.denoise``) for
    DPM-Solver++(2M) and ActionCFG, in a given dtype, optionally under autocast;
  * ``case_bound`` / ``check_final``: rel-L2 <= 5e-3 over the clip and <= 1e-2 per frame, or 4x the yardstick's error
    when the yardstick itself is above 5e-3 (the ratio of DESIGN §2: 5e-3 against the reference's own 1.2e-3);
  * planted systematic defects (``planted``), test-local, for the sensitivity checks.

Imports nothing that needs a GPU."""
import contextlib
import math
import time
from typing import Dict, List, NamedTuple, Optional

import torch

from oracle import vista_oracle as vo

BOUND = 5e-3                # rel-L2 of a sampler trajectory against the fp32 reference (DESIGN §2)
FRAME_BOUND = 1e-2          # per frame at the last step: one bad frame cannot hide in the clip average
YARDSTICK_FACTOR = 4.0      # 5e-3 against the reference's own 1.2e-3 (SURVEY Appendix C)
SENSITIVITY = 2.0           # a planted defect counts as caught when it misses the bound by this factor
REPORT_STEPS = (1, 5, 10, 25)
U16 = 2.0 ** -11            # unit roundoff of fp16


class Problem(NamedTuple):
    """One sample's inputs: conditioning dicts, the latent clip whose first ``n_cond`` frames are the conditioning
    frames, and the sampler noise."""
    c: Dict
    uc: Dict
    z: torch.Tensor
    noise: torch.Tensor
    n_cond: int

    def mask(self) -> torch.Tensor:
        m = torch.zeros(self.z.shape[0], dtype=torch.float32, device=self.z.device)
        m[:self.n_cond] = 1.0
        return m


def rel_l2(a, b) -> float:
    a, b = a.double().flatten(), b.double().flatten().to(a.device)
    return float((a - b).norm() / (b.norm() + 1e-30))


def frame_errors(out, ref) -> List[float]:
    return [rel_l2(out[f], ref[f]) for f in range(out.shape[0])]


def impose(x, problem: Problem):
    """The conditioning frames re-imposed (sampling.py:105-106): the state the next step hands to the denoiser."""
    m = problem.mask().to(x.device, x.dtype)[:, None, None, None]
    return x * (1 - m) + problem.z.to(x.device, x.dtype) * m


# ==================================================================================================================
# Our arm
# ==================================================================================================================
@contextlib.contextmanager
def recorded_steps(states: List[torch.Tensor]):
    """``fused._run_steps`` replaced by a copy of itself that appends a clone of the loop state after every step: the
    same eager first step, the same ``runner`` (so the same graph keys and replays), one extra device copy per step."""
    from vista_b200 import fused

    def run_steps(st, rt, n, multistep=False, action=False):
        if n < 3:
            for _ in range(n):
                st.one_step(rt, n, multistep, action)
                states.append(st.x.clone())
            return
        st.one_step(rt, n, multistep, action)
        states.append(st.x.clone())
        step = st.runner(rt, n, multistep, action)
        for _ in range(n - 1):
            step()
            states.append(st.x.clone())
    real = fused._run_steps
    fused._run_steps = run_steps
    try:
        yield
    finally:
        fused._run_steps = real


@contextlib.contextmanager
def engine_setting(eng, sampler, n_cond: int, graph: bool):
    """``eng`` sampling with ``sampler``, the first ``n_cond`` frames fixed (``replace_cond_frames``), and the fused loop
    replayed from CUDA graphs (``graph``, the product's path) or launched eagerly."""
    from vista_b200 import fused
    saved = (eng.sampler, eng.replace_cond_frames, eng.fixed_cond_frames, fused.USE_GRAPH)
    eng.sampler, eng.replace_cond_frames, eng.fixed_cond_frames = sampler, n_cond > 0, list(range(n_cond))
    fused.USE_GRAPH = graph
    try:
        yield
    finally:
        eng.sampler, eng.replace_cond_frames, eng.fixed_cond_frames, fused.USE_GRAPH = saved


def run_ours(eng, sampler, problem: Problem, graph: bool, record: bool = True):
    """``eng.sample`` as the product calls it -> (states after steps 1..n, final latent); ``record=False`` runs the
    unmodified loop (states empty)."""
    p = problem
    states: List[torch.Tensor] = []
    with engine_setting(eng, sampler, p.n_cond, graph), torch.no_grad(), \
            (recorded_steps(states) if record else contextlib.nullcontext()):
        out = eng.sample(p.c, cond_frame=p.z, uc=p.uc, N=p.z.shape[0], shape=tuple(p.z.shape[1:]), noise=p.noise)
    return states, out


# ==================================================================================================================
# The reference arm
# ==================================================================================================================
@contextlib.contextmanager
def oracle_dtype(dtype):
    """The oracle's timestep embedding (an fp32 island, computed where torch's default device points) handed on in
    ``dtype``, so that an fp64 oracle stays fp64.  A no-op for fp32."""
    saved = vo.timestep_embedding
    if dtype != torch.float32:
        vo.timestep_embedding = lambda t, dim, max_period=10000.0: saved(t, dim, max_period).to(dtype)
    try:
        yield
    finally:
        vo.timestep_embedding = saved


def _cast(d, dtype, T):
    """``d`` in ``dtype`` with every per-clip row repeated over the clip's T frames (video_model.py:463-470 does that
    inside the network; the oracle takes per-frame rows)."""
    out = {}
    for k, v in d.items():
        if torch.is_tensor(v) and v.is_floating_point():
            v = v.to(dtype)
            if k in ("crossattn", "vector", "concat") and v.shape[0] != T:
                v = v.repeat_interleave(T // v.shape[0], dim=0)
        out[k] = v
    return out


def guider_name(sampler):
    """(guider, scale) for ``vo.euler_edm_sample`` when it restates ``sampler``, else (None, None)."""
    from vista_b200.diffusion import EulerEDMSampler, TrianglePredictionGuider, VanillaCFG
    g = sampler.guider
    if type(sampler) is EulerEDMSampler:
        if isinstance(g, TrianglePredictionGuider):
            assert g.min_scale == 1.0, "vo.triangle_scales runs from 1.0"
            return "TrianglePredictionGuider", g.max_scale
        if type(g) is VanillaCFG:
            return "VanillaCFG", g.scale
    return None, None


def run_reference(sd, cfg, sampler, problem: Problem, dtype=torch.float32, autocast: Optional[torch.dtype] = None):
    """The oracle's trajectory on ``problem`` -> (states after steps 1..n with the conditioning frames re-imposed, final
    latent).  Euler under VanillaCFG / TrianglePredictionGuider: ``vo.euler_edm_sample``.  Anything else (2M,
    ActionCFG): ``sampler``'s own torch loop around ``vo.denoise``, recorded at each denoiser call.  ``dtype``: of the
    weights and inputs; ``autocast``: run under torch.autocast at that dtype (weights and state stay ``dtype``)."""
    dev = problem.z.device
    T = problem.z.shape[0]
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    c, uc = _cast(problem.c, dtype, T), _cast(problem.uc, dtype, T)
    noise, z, mask = problem.noise.to(dtype), problem.z.to(dtype), problem.mask().to(dtype)
    n = sampler.num_steps
    ac = torch.autocast(dev.type, dtype=autocast) if autocast is not None else contextlib.nullcontext()
    name, scale = guider_name(sampler)
    with torch.no_grad(), torch.device(dev), oracle_dtype(dtype), ac:
        if name is not None:
            out, traj = vo.euler_edm_sample(sdd, cfg, noise, c, uc, z, mask, n, T, guider=name, scale=scale,
                                            return_all=True)
            states = [impose(x, problem) for x in traj[:-1]]
        else:
            seen = []

            def den(x, sigma, cc, m):
                seen.append(x[:T].clone())
                return vo.denoise(sdd, cfg, x, sigma, cc, m, T)
            out = sampler(den, noise.clone(), c, uc=uc, cond_frame=z, cond_mask=mask)
            states = seen[1:]
    states.append(out)
    assert len(states) == n
    return [s.float() for s in states], out.float()


# ==================================================================================================================
# Bounds and the report
# ==================================================================================================================
def case_bound(yard_err: float):
    """-> (clip bound, per-frame bound, fallback): 5e-3 / 1e-2, or 4x the yardstick's clip error (per frame twice that)
    when the yardstick itself is above 5e-3."""
    if yard_err > BOUND:
        b = YARDSTICK_FACTOR * yard_err
        return b, b * FRAME_BOUND / BOUND, True
    return BOUND, FRAME_BOUND, False


def step_errors(states, ref_states) -> Dict[int, float]:
    n = len(ref_states)
    steps = sorted({s for s in REPORT_STEPS if s <= n} | {n})
    return {s: rel_l2(states[s - 1], ref_states[s - 1]) for s in steps}


class Arm(NamedTuple):
    states: List[torch.Tensor]
    out: torch.Tensor
    seconds: float
    peak_gib: float


def timed(fn, dev) -> Arm:
    """fn() -> (states, out), timed to a device synchronise, with its peak allocated memory."""
    cuda = dev.type == "cuda"
    if cuda:
        torch.cuda.synchronize(dev)
        torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    states, out = fn()
    if cuda:
        torch.cuda.synchronize(dev)
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30 if cuda else float("nan")
    return Arm([s.cpu() for s in states], out.cpu(), time.perf_counter() - t0, peak)


def report(name, problem: Problem, ours: Arm, ref: Arm, yard: Optional[Arm] = None) -> Dict:
    """Prints and returns the case's errors: ours and the yardstick against the reference at the report steps, per frame at
    the last step, time and peak memory of each arm.  Our loop re-imposes the conditioning frames at the start of the
    next step (and after the last), so its states are compared with them re-imposed, like the reference's."""
    eo = step_errors([impose(s, problem) for s in ours.states], ref.states)
    ey = step_errors(yard.states, ref.states) if yard is not None else None
    fo, fy = frame_errors(ours.out, ref.out), (frame_errors(yard.out, ref.out) if yard is not None else None)
    final_o, final_y = rel_l2(ours.out, ref.out), (rel_l2(yard.out, ref.out) if yard is not None else None)
    lines = [f"[{name}] rel-L2 against the reference, per step:"]
    for s in eo:
        lines.append(f"    step {s:3d}: ours {eo[s]:.3e}" + (f"   yardstick {ey[s]:.3e}" if ey else ""))
    lines.append(f"    final latent: ours {final_o:.3e}" + (f"   yardstick {final_y:.3e}" if ey else ""))
    lines.append("    per frame, ours:      " + " ".join(f"{e:.1e}" for e in fo))
    if fy:
        lines.append("    per frame, yardstick: " + " ".join(f"{e:.1e}" for e in fy))
    for label, arm in (("ours", ours), ("reference", ref), ("yardstick", yard)):
        if arm is not None:
            lines.append(f"    {label}: {arm.seconds:.1f} s, peak allocated {arm.peak_gib:.2f} GiB")
    print("\n" + "\n".join(lines))
    return dict(steps=eo, yard_steps=ey, frames=fo, yard_frames=fy, final=final_o, yard_final=final_y)


def check_final(name, r: Dict, n_cond: int):
    """The final latent within the case's bound over the clip and per frame."""
    b, fb, fallback = case_bound(r["yard_final"] if r["yard_final"] is not None else 0.0)
    if fallback:
        print(f"[{name}] the yardstick is at {r['yard_final']:.3e} > {BOUND}: bound {b:.3e} (clip), {fb:.3e} (frame)")
    assert r["final"] <= b, f"{name}: final latent rel-L2 {r['final']:.3e} > {b:.3e}"
    worst = max(range(len(r["frames"])), key=lambda f: r["frames"][f])
    assert r["frames"][worst] <= fb, f"{name}: frame {worst} rel-L2 {r['frames'][worst]:.3e} > {fb:.3e}"
    return b


def assert_graph_equals_eager(name, graph: Arm, eager: Arm):
    assert len(graph.states) == len(eager.states)
    for i, (g, e) in enumerate(zip(graph.states, eager.states)):
        assert torch.equal(g, e), f"{name}: graph replay differs from the eager launches after step {i + 1} " \
                                  f"(max abs {float((g - e).abs().max()):.3e})"
    assert torch.equal(graph.out, eager.out)


# ==================================================================================================================
# Planted systematic defects (test-local; nothing under vista_b200/ changes)
# ==================================================================================================================
def ulp16(x: float) -> float:
    """The spacing of fp16 numbers at |x| (normal range)."""
    return 2.0 ** (math.floor(math.log2(abs(x))) - 10)


@contextlib.contextmanager
def residual_bias(module):
    """Every tap-GEMM with a residual operand adds ``s_res1 x (1 + 2^-11)`` of it: one fp16 rounding's worth of
    systematic gain on the residual stream.  ``module``: vista_b200.ops on the GPU, tests/fake_ops on the CPU twins
    (fake_ops.patched_ops reads its ``gemm`` when it patches)."""
    real = module.gemm

    def gemm(*a, **k):
        if k.get("res1") is not None:
            k["s_res1"] = k.get("s_res1", 1.0) * (1.0 + U16)
        return real(*a, **k)
    module.gemm = gemm
    try:
        yield
    finally:
        module.gemm = real


@contextlib.contextmanager
def alpha_bias():
    """Every UNet time mixer's alpha (ResBlocks and spatial transformers) one fp16 ulp too large, as packed: the blend
    leans one rounding step towards the spatial branch.  Acts on runtimes packed inside the block."""
    from vista_b200 import unet as unet_mod
    real = unet_mod.UNetRuntime._pack

    def pack(self):
        real(self)
        for L in self.layers.values():
            if "alpha" in L:
                L["alpha"] = L["alpha"] + ulp16(L["alpha"])
    unet_mod.UNetRuntime._pack = pack
    try:
        yield
    finally:
        unet_mod.UNetRuntime._pack = real


@contextlib.contextmanager
def planted(kind: str, ops_module, net=None):
    """Defect ``kind`` for the duration of the block.  ``net``: a B200Wrapper whose packed runtime is dropped on entry
    and on exit, so that the block samples with a runtime packed under the defect and the code after it without."""
    if net is not None:
        net._rt_invalidate()
    try:
        with {"residual": lambda: residual_bias(ops_module), "alpha": alpha_bias}[kind]():
            yield
    finally:
        if net is not None:
            net._rt_invalidate()


DEFECTS = ("residual", "alpha")
