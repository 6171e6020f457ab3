"""GPU measurement, not a test: batched image-to-3D sampling (pipeline.sample_flow_batched) with each ODE solver it
runs, alternated with the dopri5 default in the same process.

  model     DiT-PixArt-L/2 (the I23D release denoiser) with random weights; context shaped like the I23D conditioner's
            (pooled (768,), tokens (256, 2048)), zero unconditional half
  batch     P = 4 conditions x N = 1 sample, CFG 4.0, 250 output points (sample_ode's default grid: the fixed-grid
            methods take 249 steps, the adaptive ones integrate to t = 1 with rtol 1e-3, atol 1e-6)
  methods   dopri5, bosh3, fehlberg2, adaptive_heun, rk4, euler, midpoint, heun

Per method: ms, latents/s, forwards per condition and per batch, and the relative L2 distance of the final latents
from a tight dopri5 solve of the same batch (rtol 1e-6, atol 1e-6).  Each method runs alternated with dopri5
(method first on odd repeats), so the dopri5 numbers beside it were taken under the same conditions.  With random
weights neither the forward counts nor the distances say anything about a trained checkpoint's sample quality.
Prints one JSON line with the card name and power limit read in the same run.

Run:  python tools/flow_solver_bench.py [--methods bosh3 rk4 ...] [--repeats 2] [--P 4] [--N 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

METHODS = ("bosh3", "fehlberg2", "adaptive_heun", "rk4", "euler", "midpoint", "heun")


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


def timed(fn):
    """(result, ms) of one call (device-synchronised host clock)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def conditions(P: int, N: int, dev, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    vec, tok = torch.randn(P, 768, generator=g), torch.randn(P, 256, 2048, generator=g)
    c = {"vector": vec.repeat_interleave(N, 0).to(dev), "crossattn": tok.repeat_interleave(N, 0).to(dev)}
    return c, {k: torch.zeros_like(v) for k, v in c.items()}


def reference(model, c, uc, N, P, num_steps, seed=42):
    """The batch's latents from a tight grouped dopri5 solve (rtol 1e-6), with sample_flow_batched's noise and
    context."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.transport.rk import odeint_rk_adaptive_grouped
    C = 3 * model.in_channels if model.roll_out else model.in_channels
    shape = (C, model.input_size, model.input_size)
    zs = pipeline.flow_batch_noise(P, N, shape, seed).to(c["vector"].device)
    ctx = pipeline.flow_batch_context(c, uc, zs.device)
    grid = torch.linspace(0, 1, num_steps)
    y, st = odeint_rk_adaptive_grouped(lambda t, x: model.forward_with_cfg(x, t, ctx, 4.0), torch.cat([zs, zs], 0),
                                       pipeline.flow_batch_row_groups(P, N), P, t0=float(grid[0]),
                                       t1=float(grid[-1]), method="dopri5", rtol=1e-6, atol=1e-6)
    return y[:P * N].reshape(P, N, *shape), st


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--methods", nargs="+", default=list(METHODS))
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--P", type=int, default=4)
    ap.add_argument("--N", type=int, default=1)
    ap.add_argument("--num-steps", type=int, default=250)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_solver_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_i23d
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    P, N, steps = args.P, args.N, args.num_steps
    res = {"gpu": name, "power_limit_w": float(power_limit), "model": "DiT-PixArt-L/2 (random weights)",
           "P": P, "N": N, "num_steps": steps, "cfg_scale": 4.0, "rtol": 1e-3, "atol": 1e-6, "methods": {}}
    model = build_i23d("DiT-PixArt-L/2", device=dev)
    c, uc = conditions(P, N, dev)
    x = torch.zeros(2 * P * N, 12, 32, 32, device=dev)          # warm-up: capture the 2PN-row forward graph
    model.forward_with_cfg(x, torch.full((2 * P * N,), 0.5, device=dev), pipeline.flow_batch_context(c, uc, dev), 4.0)
    (ref, ref_st), ref_ms = timed(lambda: reference(model, c, uc, N, P, steps))
    res["reference"] = {"solver": "dopri5 rtol 1e-6 atol 1e-6", "ms": ref_ms, "nfe": ref_st["nfe"],
                        "batch_nfe": ref_st["batch_nfe"]}
    print(json.dumps(res["reference"]), file=sys.stderr, flush=True)

    def run(method):
        (lat, st), ms = timed(lambda: pipeline.sample_flow_batched(model, c, uc, N, num_steps=steps,
                                                                   sampling_method=method))
        return {"ms": ms, "latents_per_s": P * N / (ms * 1e-3), "nfe": st["nfe"], "batch_nfe": st["batch_nfe"],
                "rel_l2_to_reference": [rel_l2(lat[i], ref[i]) for i in range(P)]}

    for method in args.methods:
        rows = {"runs": [], "dopri5_runs": []}
        for r in range(args.repeats):
            for m in ((method, "dopri5") if r % 2 == 0 else ("dopri5", method)):
                rows["runs" if m == method else "dopri5_runs"].append(run(m))
        for key in ("runs", "dopri5_runs"):
            ms = sorted(x["ms"] for x in rows[key])
            rows[key.replace("runs", "median_ms")] = ms[len(ms) // 2]
        rows["median_latents_per_s"] = P * N / (rows["median_ms"] * 1e-3)
        rows["dopri5_median_latents_per_s"] = P * N / (rows["dopri5_median_ms"] * 1e-3)
        res["methods"][method] = rows
        print(json.dumps({method: {k: v for k, v in rows.items() if "runs" not in k},
                          "nfe": rows["runs"][0]["nfe"], "batch_nfe": rows["runs"][0]["batch_nfe"],
                          "rel_l2": rows["runs"][0]["rel_l2_to_reference"],
                          "dopri5_nfe": rows["dopri5_runs"][0]["nfe"],
                          "dopri5_rel_l2": rows["dopri5_runs"][0]["rel_l2_to_reference"]}), file=sys.stderr,
              flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
