"""TEST INFRASTRUCTURE — generates tests/golden/unet_cached_*.npz, the feature-caching fixtures, by running the REAL
reference VideoUNet (/root/reference, via oracle/ref_loader.py) on seeded synthetic weights and inputs.

Run in the build container only:  python -m oracle.make_golden_cached [case ...]
The fixtures hold the reference OUTPUTS plus the checksums of the synthetic weights / inputs that produced them; the
tests regenerate the inputs from the seeds with ``unet_cached_inputs``.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

from oracle import ref_loader
from oracle.make_golden import GOLDEN_DIR, to_t, unet_inputs
from vista_b200 import spec, synth

# name -> (unet preset, latent h, latent w, frames, cache branches, keep the full forwards); small stays under 1 MB
UNET_CACHED_CASES = {
    "unet_cached_tiny": ("tiny", 8, 16, 25, (0, 1, 3), True),
    "unet_cached_small": ("small", 16, 32, 25, (1, 11), False),
}


def unet_cached_inputs(cfg, h, w, T):
    """Two forwards of one conditioning (seed 7's, a conditioning frame): x0 at sigma 5, whose deep feature is cached,
    and x1 at sigma 2 (seed 8's noise), which reuses it -> (x0, sigma0, x1, sigma1, cc, mask2)."""
    x0, cc, mask2 = unet_inputs(7, cfg, h, w, T, sigma=5.0)
    x1 = unet_inputs(8, cfg, h, w, T, sigma=2.0)[0]
    return x0, 5.0, x1, 2.0, cc, mask2


def gen_unet_cached(name):
    """Feature caching on the REAL VideoUNet: a full forward at (x0, sigma0) with a hook recording the output of
    output_blocks[n-2-b] (the middle block for the last branch), then the full forward at (x1, sigma1) with a hook
    returning that recording in place of the block's output.  Nothing deeper feeds anything else, so the second pass is
    the cached forward of branch b, run by the reference's own code.  Raw network outputs (preconditioning removed)."""
    preset, h, w, T, branches, keep_full = UNET_CACHED_CASES[name]
    cfg = spec.unet_preset(preset)
    sd = synth.synth_state_dict(spec.unet_param_specs(cfg), seed=1)
    unet = ref_loader.build_ref_unet(cfg)
    unet.load_state_dict(to_t(sd), strict=True)
    ref = ref_loader.load_reference()
    net = ref.OpenAIWrapper(unet)
    den = ref_loader.build_ref_denoiser(T)
    x0, s0, x1, s1, cc, mask2 = unet_cached_inputs(cfg, h, w, T)
    cct, m2 = to_t(cc), torch.from_numpy(mask2)
    n = len(unet.output_blocks)
    out = {}

    def raw(x, sigma):
        c_skip, c_out, c_in, c_noise = den.scaling(torch.full((2 * T, 1, 1, 1), sigma))
        return net(torch.from_numpy(x) * c_in, c_noise.reshape(-1), cct, m2, T)
    t0 = time.time()
    with torch.no_grad():
        out["full0"] = raw(x0, s0).numpy()
        out["full1"] = raw(x1, s1).numpy()
        for b in branches:
            mod = unet.middle_block if b == n - 1 else unet.output_blocks[n - 2 - b]
            kept = {}
            hook = mod.register_forward_hook(lambda m, a, o: kept.__setitem__("h", o.clone()))
            assert np.array_equal(raw(x0, s0).numpy(), out["full0"])
            hook.remove()
            hook = mod.register_forward_hook(lambda m, a, o: kept["h"])
            out[f"cached_b{b}"] = raw(x1, s1).numpy()
            hook.remove()
    print(f"{name}: {time.time() - t0:.0f}s; cached vs full at x1 rel-L2 " + ", ".join(
        f"b{b} {np.linalg.norm(out[f'cached_b{b}'] - out['full1']) / np.linalg.norm(out['full1']):.3e}" for b in branches))
    if not keep_full:
        del out["full0"], out["full1"]
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), weight_checksum=synth.state_dict_checksum(sd),
                        input_checksum=synth.checksum([x0, x1, mask2] + [cc[k] for k in sorted(cc)]),
                        branches=np.array(branches, dtype=np.int64), **out)


def main(argv):
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for cname in argv or list(UNET_CACHED_CASES):
        gen_unet_cached(cname)


if __name__ == "__main__":
    main(sys.argv[1:])
