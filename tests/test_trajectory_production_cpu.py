"""The trajectory harness of tests/trajectory.py without a GPU: the tiny UNet (8 x 16 latents, T = 25) on the operator
twins (tests/fake_ops.py and the sampler updates' twins), against the oracle in fp64 on the CPU.

  * the recording copy of ``fused._run_steps`` gives the un-instrumented run's final latent, bit for bit, and one state
    per step, through both of its branches (fewer than three steps, and the runner's);
  * the three cases of tests/test_trajectory_production_gpu.py at their step counts: within the bound;
  * the bound logic, with the yardstick's fallback;
  * the planted systematic defects: each passes the layer harness (tests/block_shadow.py) on the tiny UNet and reaches
    case A's sample; the error it leaves there is printed against the trajectory bound."""
import types

import pytest
import torch

import test_dpmpp2m_cpu as tdc
import trajectory as tj
from action_fake_ops import patched_action_ops
from test_action_cfg_cpu import action_cfg, triangle_cfg, vanilla_cfg
from test_block_conformance_cpu import run_unet

T = 25
# case -> (sampler, guider, conditioning frames, steps): the table of tests/test_trajectory_production_gpu.py
CASES = {"A": ("euler", vanilla_cfg(2.5), 1, 50), "B": ("euler", triangle_cfg(T), 3, 25),
         "C": ("dpm", action_cfg(5.0, triangle_cfg(T)), 1, 25)}


class TinyEngine(types.SimpleNamespace):
    """The attributes ``DiffusionEngine.sample`` reads, over the tiny UNet on the CPU."""
    from vista_b200.engine import DiffusionEngine
    sample = DiffusionEngine.sample


@pytest.fixture(scope="module")
def tiny():
    cfg, sd, net, den, bden = tdc.tiny_network()
    eng = TinyEngine(model=net, denoiser=den, sampler=None, device=torch.device("cpu"), num_frames=T,
                     replace_cond_frames=False, fixed_cond_frames=None)
    return cfg, {k: torch.from_numpy(v) for k, v in sd.items()}, eng


@pytest.fixture
def emulated():
    with patched_action_ops(), torch.no_grad():
        yield


def problem(cfg, n_cond, seed=7):
    c, uc, noise, z, _ = tdc.tiny_inputs(cfg, n_cond=n_cond, seed=seed)
    return tj.Problem(c, uc, z, noise, n_cond)


def sampler(case, steps=None):
    kind, guider, _, n = CASES[case]
    return tdc.make_sampler(kind, steps or n, guider=guider)


def run_case(tiny, case, steps=None):
    cfg, sd, eng = tiny
    p = problem(cfg, CASES[case][2])
    smp = sampler(case, steps)
    dev = torch.device("cpu")
    ours = tj.timed(lambda: tj.run_ours(eng, smp, p, graph=False), dev)
    ref = tj.timed(lambda: tj.run_reference(sd, cfg, smp, p, torch.float64), dev)
    yard = tj.timed(lambda: tj.run_reference(sd, cfg, smp, p, torch.float32), dev)
    return p, ours, ref, yard


@pytest.mark.parametrize("kind,steps", [("euler", 2), ("euler", 6), ("dpm", 5)])
def test_recording_is_transparent(tiny, emulated, kind, steps):
    """One state per step, the last one the sample; the recorded run's sample equal to the un-instrumented one's."""
    cfg, sd, eng = tiny
    p = problem(cfg, 1)
    smp = tdc.make_sampler(kind, steps)
    states, out = tj.run_ours(eng, smp, p, graph=False)
    _, plain = tj.run_ours(eng, smp, p, graph=False, record=False)
    assert len(states) == steps and torch.equal(states[-1], out) and torch.equal(out, plain)
    assert all(not torch.equal(a, b) for a, b in zip(states, states[1:]))
    assert torch.equal(out[:1], p.z[:1])


def test_reference_records_every_step(tiny):
    """Both reference paths (the oracle's Euler sampler and the torch loop) record the same trajectory for an Euler /
    VanillaCFG sample: the states handed to the denoiser are the oracle's states with the conditioning frames
    re-imposed."""
    cfg, sd, eng = tiny
    p = problem(cfg, 3)
    smp = tdc.make_sampler("euler", 4)
    a, out_a = tj.run_reference(sd, cfg, smp, p, torch.float64)
    smp.__class__ = type("Generic", (type(smp),), {})          # not an EulerEDMSampler by type: the torch-loop path
    assert tj.guider_name(smp) == (None, None)
    b, out_b = tj.run_reference(sd, cfg, smp, p, torch.float64)
    assert len(a) == len(b) == 4
    for x, y in zip(a, b):
        assert tj.rel_l2(x, y) < 1e-6
    assert torch.equal(out_a[:3], p.z[:3].float())


@pytest.mark.parametrize("case", sorted(CASES))
def test_cases_within_bound(tiny, emulated, case):
    p, ours, ref, yard = run_case(tiny, case)
    r = tj.report(f"tiny case {case}", p, ours, ref, yard)
    assert torch.equal(ours.out[:p.n_cond], p.z[:p.n_cond])
    tj.check_final(f"tiny case {case}", r, p.n_cond)


def test_bound_logic():
    assert tj.case_bound(1.2e-3) == (5e-3, 1e-2, False)
    assert tj.case_bound(5e-3) == (5e-3, 1e-2, False)
    b, fb, fallback = tj.case_bound(8e-3)
    assert fallback and b == pytest.approx(3.2e-2) and fb == pytest.approx(6.4e-2)
    ok = dict(final=4.9e-3, frames=[0.0, 9e-3], yard_final=1e-3)
    tj.check_final("ok", ok, 1)
    for bad in (dict(ok, final=5.1e-3), dict(ok, frames=[0.0, 1.1e-2])):
        with pytest.raises(AssertionError):
            tj.check_final("bad", bad, 1)
    tj.check_final("fallback", dict(final=3e-2, frames=[0.0, 6e-2], yard_final=8e-3), 1)
    with pytest.raises(AssertionError):
        tj.check_final("fallback", dict(final=3.3e-2, frames=[0.0, 6e-2], yard_final=8e-3), 1)


def test_ulp16():
    for a in (0.3, 0.5, 0.62, 0.99):
        h = torch.tensor(a, dtype=torch.float16)
        up = float(torch.nextafter(h, torch.tensor(2.0, dtype=torch.float16)))
        assert tj.ulp16(float(h)) == up - float(h)


@pytest.mark.parametrize("defect", tj.DEFECTS)
def test_planted_defect_passes_layers_and_moves_trajectory(tiny, defect):
    """The defect keeps every layer of the tiny UNet within its block_shadow partition bound (only the layer gain check
    fails it), and is live in case A's 50-step sample.  Prints the planted run's error against the trajectory bound and
    how far it moved the sample: neither defect leaves the bound at the tiny preset's depth (DESIGN §2 gives the
    measured ratios, here and at 576 x 1024)."""
    import fake_ops
    cfg, sd, eng = tiny
    with tj.planted(defect, fake_ops):
        bs, _ = run_unet()
    worst = max(v.ratio for v in bs.census.values())
    assert not bs.coverage()
    assert not {k: m for k, m in bs.failures.items() if k[0] != "gain"}, bs.failures
    assert any(k[0] == "gain" for k in bs.failures), "the layer gain check does not see the defect"
    with patched_action_ops(), torch.no_grad():
        p, clean, ref, _ = run_case(tiny, "A")
        with tj.planted(defect, fake_ops, eng.model):
            bad = tj.timed(lambda: tj.run_ours(eng, sampler("A"), p, graph=False), torch.device("cpu"))
    r = tj.report(f"tiny case A, planted {defect}", p, bad, ref)
    e_clean = tj.rel_l2(clean.out, ref.out)
    moved = tj.rel_l2(bad.out, clean.out)
    print(f"planted {defect}: worst layer at {worst:.2f} x its bound; final latent {r['final']:.3e} "
          f"({r['final'] / tj.BOUND:.2f} x the trajectory bound) against {e_clean:.3e} without the defect; "
          f"{moved:.3e} from the clean sample")
    assert worst < 1.0 and moved > 0.0
