"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/edm_samplers.npz by running the REFERENCE's own sgm samplers.

Runs only where the reference checkout exists (third-party gaps are filled by oracle/_stubs.py).  Nothing is copied
from the reference: the fixture holds the outputs its classes produce on seeded inputs.  Re-run:
    python -m oracle.make_golden_edm_samplers

Setup: DiscreteDenoiser(EpsScaling, 1000) + VanillaCFG(6.5) on LegacyDDPMDiscretization around
oracle.fixtures.toy_network(), on the 8x8 corner of oracle.fixtures.sampler_inputs()'s x / cond (edm_samplers.inputs();
the toy network is per pixel, so the crop only keeps the fixture small); ancestral noise is injected by patching
`torch.randn_like` with oracle.edm_samplers.step_noise(steps) (the count of draws is recorded).
Keys, for S in (10, 3):
  {name}_{S}           final x of HeunEDMSampler, EulerAncestralSampler, DPMPP2SAncestralSampler, DPMPP2MSampler,
                       LinearMultistepSampler (order 4)
  {name}_{S}_draws     number of randn_like draws
  lms_coeff_{S}        (S, 4) linear_multistep_coeff(min(i+1, 4), sigmas, i, j) as the sampler calls it (float32
                       nodes), NaN-padded
  lms_coeff64_{S}      the same with the nodes in float64 (the reference's integrand then evaluates in float64)
  sigma_down_{S}, sigma_up_{S}   get_ancestral_step(sigmas[i], sigmas[i+1], eta=1)
  sigmas_{S}           the schedule
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import _stubs  # noqa: E402
from oracle import edm_samplers as oes  # noqa: E402
from oracle import fixtures as fx  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "edm_samplers.npz")


def main():
    _stubs.install()
    import sgm.modules.diffusionmodules.sampling as smp
    from sgm.modules.diffusionmodules.denoiser import DiscreteDenoiser
    from sgm.modules.diffusionmodules.sampling_utils import get_ancestral_step, linear_multistep_coeff
    disc = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
    guider = {"target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": oes.SCALE}}
    den = DiscreteDenoiser(scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
                           num_idx=1000, discretization_config=disc)
    toy = fx.toy_network()
    x0, c, uc = oes.inputs()
    out = {}
    for S in (10, 3):
        for name in oes.SAMPLERS:
            sampler = getattr(smp, name)(discretization_config=disc, num_steps=S, device="cpu", guider_config=guider)
            noise = oes.step_noise(S, tuple(x0.shape))
            n = [0]

            def fake_randn_like(v, *a, **k):
                n[0] += 1
                return noise[n[0] - 1]

            orig = torch.randn_like
            torch.randn_like = fake_randn_like
            try:
                with torch.no_grad():
                    y = sampler(lambda inp, sig, cc: den(toy, inp, sig, cc), x0.clone(), c, uc)
            finally:
                torch.randn_like = orig
            out[f"{name}_{S}"] = y.numpy()
            out[f"{name}_{S}_draws"] = np.int64(n[0])
            print(name, S, n[0], float(y.abs().max()))
        sig = sampler.discretization(S, device="cpu")
        sig_np = sig.numpy()
        lms = np.full((S, 4), np.nan)
        lms64 = np.full((S, 4), np.nan)
        for i in range(S):
            cur = min(i + 1, 4)
            for j in range(cur):
                lms[i, j] = linear_multistep_coeff(cur, sig_np, i, j)
                lms64[i, j] = linear_multistep_coeff(cur, sig_np.astype(np.float64), i, j)
        sd, su = get_ancestral_step(sig[:-1], sig[1:], eta=1.0)
        out.update({f"lms_coeff_{S}": lms, f"lms_coeff64_{S}": lms64, f"sigma_down_{S}": sd.numpy(),
                    f"sigma_up_{S}": su.numpy(), f"sigmas_{S}": sig_np})
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
