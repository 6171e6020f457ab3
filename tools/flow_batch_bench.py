"""GPU measurement, not a test: batched image-to-3D sampling (pipeline.sample_flow_batched, one grouped dopri5 solve for
P conditions x N samples) against P sequential pipeline.sample_flow calls, alternated in the same process.

  model     DiT-PixArt-L/2 (the I23D release denoiser) with random weights; context shaped like the I23D conditioner's
            (pooled (768,), tokens (256, 2048)), zero unconditional half
  solver    dopri5 with 250 output points, CFG 4.0 (the release default)
  cases     P in {1, 4, 8, 16} conditions at N = 1 (gradio demo) and N = 4 (release scripts)

Per case: ms and latents/s of both paths, NFE per condition (batched) and per call (sequential), and the useful-row
fraction of the batch -- the row-forwards spent on unfinished conditions over all row-forwards the batch ran (rows of
finished conditions keep flowing through the forward until the last one ends).  With random weights the NFE counts
are not those of a trained checkpoint.  Prints one JSON line with the card name and power limit read in the same run.

Run:  python tools/flow_batch_bench.py [--P 1 4 8 16] [--N 1 4]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[1, 4, 8, 16])
    ap.add_argument("--N", type=int, nargs="+", default=[1, 4])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_batch_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_i23d
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    res = {"gpu": name, "power_limit_w": float(power_limit), "model": "DiT-PixArt-L/2 (random weights)",
           "solver": "dopri5, 250 points", "cfg_scale": 4.0, "cases": []}
    model = build_i23d("DiT-PixArt-L/2", device=dev)
    fwd = model.forward_with_cfg
    nfe = [0]

    def counted(*a, **k):
        nfe[0] += 1
        return fwd(*a, **k)

    for N in args.N:
        for P in args.P:
            c, uc = conditions(P, N, dev)
            sl = lambda d, i: {k: v[i * N:(i + 1) * N] for k, v in d.items()}
            # warm-up: capture the forward graphs of both batch sizes (2PN and 2N rows)
            x = torch.zeros(2 * P * N, 12, 32, 32, device=dev)
            ctx = pipeline.flow_batch_context(c, uc, dev)
            model.forward_with_cfg(x, torch.full((2 * P * N,), 0.5, device=dev), ctx, 4.0)
            ctx1 = pipeline.flow_batch_context(sl(c, 0), sl(uc, 0), dev)
            model.forward_with_cfg(x[:2 * N], torch.full((2 * N,), 0.5, device=dev), ctx1, 4.0)
            case = {"P": P, "N": N, "batch_rows": 2 * P * N}
            for order in ((0, 1) if (P + N) % 2 else (1, 0)):     # alternate which path runs first
                if order == 0:
                    (lat, st), ms = timed(lambda: pipeline.sample_flow_batched(model, c, uc, N))
                    useful = sum(st["nfe"]) / (P * st["batch_nfe"])
                    case["batched"] = {"ms": ms, "latents_per_s": P * N / (ms * 1e-3), "nfe": st["nfe"],
                                       "batch_nfe": st["batch_nfe"], "useful_row_fraction": useful}
                else:
                    model.forward_with_cfg = counted
                    nfes, total = [], 0.0
                    for i in range(P):
                        nfe[0] = 0
                        _, ms = timed(lambda: pipeline.sample_flow(model, sl(c, i), sl(uc, i), N))
                        nfes.append(nfe[0])
                        total += ms
                    del model.forward_with_cfg
                    case["sequential"] = {"ms": total, "latents_per_s": P * N / (total * 1e-3), "nfe": nfes}
            case["speedup"] = case["sequential"]["ms"] / case["batched"]["ms"]
            res["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
