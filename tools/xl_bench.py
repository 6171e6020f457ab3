"""GPU measurement, not a test: DiT-XL/2 text-to-3D (hidden 1152, 16 heads of 72, cross-attention 16 x 64).

  fmha      the self-attention shape of one XL forward at B' = 16 (768 tokens, 16 heads of 72) against the 64-wide
            kernel at matched FLOPs (18 heads of 64: the same 1152 columns), launches alternated, CUDA-event medians;
            TFLOP/s (4 B H L^2 d) and the share of the data-sheet dense bf16 peak.
  forward   one DiT-XL/2 CFG forward (graph replay) at B' = 16 (8 prompts + their zero-embedding halves), and its
            algorithmic FLOPs (MAC = 2, every GEMM and attention of the reference's forward) over that time.
  sampling  pipeline.sample_t23d latents/s at 8 prompts: 25 DPM++ 2M steps and 250 Euler-EDM steps, the two
            alternated over --sampling-rounds rounds; median, min and max per sampler.
Random seeded weights (no XL checkpoint exists): the times do not depend on the weights.  Data-sheet peak: 989 dense
bf16 TFLOP/s for the H100 SXM at 700 W; the card's name and power limit are printed beside the numbers.
Prints one JSON line.

Run:  python tools/xl_bench.py [--reps 50] [--sampling-rounds 7]
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

PEAK_BF16 = 989e12
T, D, HEADS, DEPTH, E, LC, MLP = 768, 1152, 16, 28, 1024, 77, 4608


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


def event_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns: dict, reps: int, inner: int = 1) -> dict:
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t[k].append(event_ms(f, inner))
    return {k: statistics.median(v) for k, v in t.items()}


def forward_flops_per_sample() -> float:
    """Algorithmic FLOPs of one DiT-XL/2 T23D forward for one sample (MAC = 2), as the reference computes it: per layer
    qkv, self-attention (QK^T and PV), proj, cross q, cross k / v over the 77 tokens, cross-attention, cross out,
    fc1, fc2, the block's adaLN; plus the timestep MLP, the final adaLN / linear and the patch embed."""
    per_layer = (2 * T * D * 3 * D + 4 * T * T * D + 2 * T * D * D + 2 * T * D * E + 4 * LC * D * E + 4 * T * LC * E
                 + 2 * T * E * D + 2 * 2 * T * D * MLP + 2 * D * 6 * D)
    head = 2 * 256 * D + 2 * D * D + 2 * D * 2 * D + 2 * T * D * 16 + 2 * T * 16 * D
    return DEPTH * per_layer + head


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--sampling-rounds", type=int, default=7)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "xl_bench measures on the GPU"
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.utils import build_t23d
    dev = torch.device("cuda", 0)
    name, power = smi("name,power.limit")
    res = {"gpu": name, "power_limit_w": float(power)}

    # ---------------------------------------------------------------- fmha 72 vs 64 at matched FLOPs
    g = torch.Generator(device=dev).manual_seed(0)
    Bp = 16
    qkv = torch.randn(Bp, T, 3 * D, device=dev, generator=g).bfloat16()
    o72, o64 = torch.empty(Bp, T, D, device=dev, dtype=torch.bfloat16), torch.empty(Bp, T, D, device=dev,
                                                                                    dtype=torch.bfloat16)
    q, k, v = qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]
    ms = alternate({"hd72": lambda: ops.fmha(q, k, v, HEADS, out=o72),
                    "hd64": lambda: ops.fmha(q, k, v, D // 64, out=o64)}, args.reps, inner=10)
    fl = 4 * Bp * T * T * D
    res["fmha"] = {k: {"ms": round(t, 4), "tflops": round(fl / t / 1e9, 1), "peak_frac": round(fl / t / PEAK_BF16 * 1e3, 3)}
                   for k, t in ms.items()}

    # ---------------------------------------------------------------- one CFG forward at B' = 16
    m = build_t23d("DiT-XL/2").to(dev)
    gc = torch.Generator().manual_seed(41)
    B = 8
    x0 = torch.randn(B, 12, 32, 32, generator=gc).to(dev)
    c = {"crossattn": torch.randn(B, 77, 768, generator=gc).to(dev)}
    uc = {"crossattn": torch.zeros(B, 77, 768, device=dev)}
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    gr = m.capture_graph(2 * B, ctx)
    gr.x.copy_(torch.cat([x0, x0]))
    gr.t.fill_(500.0)
    fwd = alternate({"fwd": gr.replay}, args.reps)["fwd"]
    ff = forward_flops_per_sample() * 2 * B
    res["forward_b16"] = {"ms": round(fwd, 3), "gflop": round(ff / 1e9, 1), "tflops": round(ff / fwd / 1e9, 1),
                          "peak_frac": round(ff / fwd / PEAK_BF16 * 1e3, 3)}

    # ---------------------------------------------------------------- sampling
    runs = {("DPMPP2MSampler", 25): [], ("EulerEDMSampler", 250): []}
    for sampler, steps in runs:
        pipeline.sample_t23d(m, x0, c, uc, steps, 6.5, sampler=sampler)
    torch.cuda.synchronize()
    finite = True
    for _ in range(args.sampling_rounds):          # the two samplers alternate, round by round
        for (sampler, steps), times in runs.items():
            t0 = time.perf_counter()
            lat = pipeline.sample_t23d(m, x0, c, uc, steps, 6.5, sampler=sampler)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            finite = finite and bool(torch.isfinite(lat).all())
    res["sampling"] = {f"{s}_{n}": {"rounds": len(t), "s_median": round(statistics.median(t), 3),
                                    "s_min": round(min(t), 3), "s_max": round(max(t), 3),
                                    "latents_per_s_median": round(B / statistics.median(t), 3),
                                    "latents_per_s_range": [round(B / max(t), 3), round(B / min(t), 3)]}
                       for (s, n), t in runs.items()}
    res["sampling_finite"] = finite
    res["forward_flops_per_sample_gflop"] = round(forward_flops_per_sample() / 1e9, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
