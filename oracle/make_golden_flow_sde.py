"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/flow_sde.npz by running the REFERENCE's own
`Sampler(create_transport(snr_type='lognorm')).sample_sde` (transport/transport.py:313-372).

Runs only where the reference checkout exists (third-party gaps are filled by oracle/_stubs.py).  Nothing is copied
from the reference: the fixture holds the outputs its classes produce on seeded inputs.  Re-run:
    python oracle/make_golden_flow_sde.py

Setup (oracle/flow_sde.py): the CFG-shaped toy network `toy_cfg` on cat([zs, zs]) with zs = randn(2, 12, 8, 8) after
manual_seed(7), CFG 4.0, 10 steps; the sampler's noise comes from the global CPU generator, as in the engine.
Keys, for method in (Euler, Heun), form in flow_sde.FORMS, last in (None, Mean, Tweedie, Euler):
  {method}_{form}_{last}          final state (4, 12, 8, 8) fp32 (Heun / None is recorded as a failure instead)
  {method}_{form}_{last}_calls    model calls;  _len  length of the returned list
  rng_after                       CPU generator state after any run (every run draws num_steps - 1 times)
  heun_none_finite_{form}         False: the reference's Heun with last_step=None gives NaN
  sbdm_diffusion                  compute_diffusion(form='SBDM') at t = 0 and t = 0.004
  sbdm_finite                     whether Euler / SBDM / Mean returned finite values
  constant_error, increasing_decreasing_error   the exception class the reference raises
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import _stubs  # noqa: E402
from oracle import flow_sde as ofs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "flow_sde.npz")


def _run(Sampler, create_transport, method, form, last):
    zs, ctx = ofs.inputs()
    model = ofs.toy_cfg()
    fn = Sampler(create_transport(snr_type="lognorm")).sample_sde(sampling_method=method, diffusion_form=form,
                                                                 last_step=last, num_steps=ofs.STEPS)
    with torch.no_grad():
        xs = fn(torch.cat([zs, zs], 0), model, context=ctx, cfg_scale=ofs.CFG)
    return xs, model.calls


def main():
    _stubs.install()
    sys.path.insert(0, _stubs.REFERENCE_ROOT)
    from transport import Sampler, create_transport
    from transport import path as rpath
    out, rng = {}, None
    for method in ("Euler", "Heun"):
        for form in ofs.FORMS:
            for last in ofs.LASTS:
                xs, calls = _run(Sampler, create_transport, method, form, last)
                after = torch.get_rng_state()
                assert rng is None or torch.equal(rng, after)
                rng = after
                y = xs[-1]
                if method == "Heun" and last is None:
                    out[f"heun_none_finite_{form}"] = np.bool_(bool(torch.isfinite(y).all()))
                    continue
                assert bool(torch.isfinite(y).all()), (method, form, last)
                key = f"{method}_{form}_{last}"
                out[key] = y.numpy()
                out[key + "_calls"] = np.int64(calls)
                out[key + "_len"] = np.int64(len(xs))
                print(key, calls, len(xs), float(y.abs().max()))
    out["rng_after"] = rng.numpy()
    x = torch.zeros(2, 4)
    plan = rpath.ICPlan()
    out["sbdm_diffusion"] = np.array([float(plan.compute_diffusion(x, torch.tensor([t, t]), form="SBDM")[0])
                                      for t in (0.0, 0.004)], dtype=np.float32)
    xs, _ = _run(Sampler, create_transport, "Euler", "SBDM", "Mean")
    out["sbdm_finite"] = np.bool_(bool(torch.isfinite(xs[-1]).all()))
    for name, form in (("constant_error", "constant"), ("increasing_decreasing_error", "increasing-decreasing")):
        try:
            _run(Sampler, create_transport, "Euler", form, "Mean")
            out[name] = np.array("none")
        except Exception as e:  # noqa: BLE001 -- the class is what is recorded
            out[name] = np.array(type(e).__name__)
    print({k: out[k] for k in ("sbdm_diffusion", "sbdm_finite", "constant_error", "increasing_decreasing_error")})
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
