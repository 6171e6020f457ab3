"""GPU measurement, not a test: the sgm sampler family of pipeline.sample_t23d against the engine's Euler-EDM.

  speed        DiT-L/2 T23D on random seeded weights, 8 prompts with their zero-embedding halves (B' = 16), CFG 6.5:
               Euler-250 and each of Heun, Euler-ancestral, DPM++ 2S-a, DPM++ 2M and LMS at 25 and 50 steps.  Every
               configuration runs once to warm up (graph capture, plan tables), then the configurations take turns
               for ROUNDS rounds; medians of CUDA-event times.  Reports latents/s and ms per denoiser evaluation.
  convergence  rel-L2 of the final latents to a Heun-1000 solution for the deterministic samplers (Heun, DPM++ 2M,
               LMS and Euler) at 10 / 25 / 50 / 100 / 250 steps, same noise and prompts.  On random weights this
               shows how fast the discretisation error falls; it says nothing about sample quality.
Prints one JSON line with the card name and power limit.

Run:  python tools/edm_sampler_bench.py [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NEW = ("HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
       "LinearMultistepSampler")


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prompts", type=int, default=8)
    args = ap.parse_args()
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_t23d
    dev = torch.device("cuda", 0)
    m = build_t23d("DiT-L/2", seed=0, device=dev)
    P = args.prompts
    g = torch.Generator().manual_seed(41)
    x0 = torch.randn(P, 12, 32, 32, generator=g).to(dev)
    c = {"crossattn": torch.randn(P, 77, 768, generator=g).to(dev)}
    uc = {"crossattn": torch.zeros(P, 77, 768, device=dev)}

    def run(name, steps):
        return pipeline.sample_t23d(m, x0, c, uc, steps, 6.5, sampler=name)

    configs = [("EulerEDMSampler", 250)] + [(n, s) for n in NEW for s in (25, 50)]
    forwards = {(n, s): (s if n == "EulerEDMSampler" else len(pipeline.edm_sampler_plan(n, s, 6.5)["evals"]))
                for n, s in configs}
    for n, s in configs:                                          # warm-up: graphs, modulation tables, plans
        run(n, s)
    torch.cuda.synchronize()
    times = {k: [] for k in configs}
    for _ in range(args.rounds):
        for k in configs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.manual_seed(0)
            e0.record()
            run(*k)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    speed = {}
    for k in configs:
        ms = statistics.median(times[k])
        speed[f"{k[0]}-{k[1]}"] = dict(ms=round(ms, 2), latents_per_s=round(P / ms * 1e3, 3), forwards=forwards[k],
                                       ms_per_eval=round(ms / forwards[k], 3))
    euler = speed["EulerEDMSampler-250"]
    for v in speed.values():
        v["speedup_vs_euler250"] = round(v["latents_per_s"] / euler["latents_per_s"], 2)
        v["ms_per_eval_vs_euler"] = round(v["ms_per_eval"] / euler["ms_per_eval"], 3)

    ref = run("HeunEDMSampler", 1000)
    conv = {}
    for n in ("HeunEDMSampler", "DPMPP2MSampler", "LinearMultistepSampler", "EulerEDMSampler"):
        conv[n] = {str(s): round(rel(run(n, s), ref), 5) for s in (10, 25, 50, 100, 250)}
    name, power = smi("name,power.limit")
    print(json.dumps(dict(gpu=name, power_limit_w=float(power), arch="DiT-L/2", prompts=P, batch=2 * P, cfg=6.5,
                          rounds=args.rounds, speed=speed, rel_l2_to_heun1000=conv,
                          note="random weights: convergence of the discretisation only, not sample quality")))


if __name__ == "__main__":
    main()
