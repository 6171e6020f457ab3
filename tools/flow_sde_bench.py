"""GPU measurement, not a test: image-to-3D SDE sampling (pipeline.sample_flow(..., sde=)) with Euler-Maruyama and
Heun at 50 / 100 / 250 steps against the release's dopri5 with 250 output points, alternated in one process.

  model     DiT-PixArt-L/2 (the I23D release denoiser) with random weights; context shaped like the I23D conditioner's
            (pooled (768,), tokens (256, 2048)), zero unconditional half; N = 4 samples, CFG 4.0
  SDE       diffusion_form 'sigma', last_step 'Mean' (the command-line defaults)

Per case: median ms per call over the rounds, latents/s, forwards per latent batch and ms per forward (call time over
forwards; the SDE's host-side noise draws are included).  With random weights the dopri5 NFE is not that of a trained
checkpoint.  Prints one JSON line with the card name and power limit read in the same run.

Run:  python tools/flow_sde_bench.py [--steps 50 100 250] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, nargs="+", default=[50, 100, 250])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--N", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_sde_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import pipeline
    from ln3diff_b200.dit._graph import ForwardGraph
    from ln3diff_b200.utils import build_i23d
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    N = args.N
    model = build_i23d("DiT-PixArt-L/2", device=dev)
    g = torch.Generator().manual_seed(0)
    c = {"vector": torch.randn(1, 768, generator=g).repeat(N, 1).to(dev),
         "crossattn": torch.randn(1, 256, 2048, generator=g).repeat(N, 1, 1).to(dev)}
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    cases = {"dopri5-250": dict(num_steps=250)}
    for method in ("Euler", "Heun"):
        for s in args.steps:
            cases[f"{method}-{s}"] = dict(num_steps=s, sde=dict(sampling_method=method))
    replays = [0]
    orig = ForwardGraph.replay

    def counting(self):
        replays[0] += 1
        return orig(self)
    ForwardGraph.replay = counting
    ms, fwd = {k: [] for k in cases}, {}
    for k, kw in cases.items():          # warm-up: graph capture and first launches of every case
        pipeline.sample_flow(model, c, uc, N, **{**kw, "num_steps": min(kw["num_steps"], 5)})
    for _ in range(args.rounds):
        for k, kw in cases.items():
            replays[0] = 0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = pipeline.sample_flow(model, c, uc, N, **kw)
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)
            fwd[k] = replays[0]
            assert bool(torch.isfinite(out).all()), k
    ForwardGraph.replay = orig
    res = {"gpu": name, "power_limit_w": float(power_limit), "model": "DiT-PixArt-L/2 (random weights)",
           "num_samples": N, "cfg_scale": 4.0, "sde": "diffusion_form sigma, last_step Mean", "rounds": args.rounds,
           "cases": []}
    for k in cases:
        m = statistics.median(ms[k])
        res["cases"].append({"case": k, "ms": round(m, 1), "latents_per_s": round(N / (m / 1e3), 3),
                             "forwards": fwd[k], "ms_per_forward": round(m / fwd[k], 3)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
