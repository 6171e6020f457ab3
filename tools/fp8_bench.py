"""GPU measurement, not a test: the fp8 GEMM precision (set_gemm_precision("fp8")) against the default bf16 path.

  gemms     the three fp8 GEMM shapes of DiT-L/2 at B' = 16 (M = 12288): qkv (N 3072, K 1024), fc1 + GELU (N 4096,
            K 1024; bf16 output vs fp8 output), fc2 (N 1024, K 4096).  bf16 (ops.gemm) and fp8 (ops.gemm_fp8) launches
            alternate; CUDA-event medians over REPS launches each; TFLOP/s and the share of the data-sheet dense peaks
            (989 bf16, 1979 fp8 TFLOP/s for the H100 SXM at 700 W; the card's own limit is printed beside them).
  forward   one denoiser forward (graph replay) at T23D DiT-L/2 B' = 16 and I23D DiT-PixArt-L/2 B' = 64, both modes
            alternated, medians.
  sampling  250-step pipeline.sample_t23d (DiT-L/2, 8 prompts + their zero-embedding halves, CFG 6.5), latents/s per
            mode, the rel-L2 between the fp8 and bf16 final latents on the same seeds, and of the 128x128 views
            rendered from them (DiT2-L/2 decoder, 4 orbit cameras, the same render noise).
Random seeded weights throughout (no checkpoint): the deviations are those of this weight distribution.
Prints one JSON line.

Run:  python tools/fp8_bench.py [--steps 250] [--reps 50]
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
    """Median ms per call of each fn, taking turns, after one warm-up each."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t[k].append(event_ms(f, inner))
    return {k: statistics.median(v) for k, v in t.items()}


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def gemm_section(reps):
    from ln3diff_b200 import ops
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    M = 12288
    res = {}
    for name, N, K, act in (("qkv", 3072, 1024, None), ("fc1_gelu", 4096, 1024, ops.ACT_GELU_ERF),
                            ("fc2", 1024, 4096, None)):
        a = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device=dev, generator=g) * K ** -0.5).to(torch.bfloat16)
        b = torch.randn(N, device=dev, generator=g)
        aq, as_ = ops.quantize_fp8(a)
        wq, ws = ops.quantize_weight_fp8(w)
        ob = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        if act is None:
            of = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            f8 = lambda: ops.gemm_fp8(aq, as_, wq, ws, b, out=of)
            fb = lambda: ops.gemm(a, w, b, out=ob)
        else:
            of, os_ = torch.empty(M, N, device=dev, dtype=ops.FP8), torch.empty(M, N // 128, device=dev)
            f8 = lambda: ops.gemm_fp8(aq, as_, wq, ws, b, act=act, out_kind=ops.OUT_FP8, out=of, out_scale=os_)
            fb = lambda: ops.gemm(a, w, b, act=act, out=ob)
        ms = alternate({"bf16": fb, "fp8": f8}, reps, inner=10)
        flop = 2.0 * M * N * K
        tb, tf = flop / ms["bf16"] / 1e9, flop / ms["fp8"] / 1e9
        res[name] = {"M": M, "N": N, "K": K, "bf16_us": ms["bf16"] * 1e3, "fp8_us": ms["fp8"] * 1e3,
                     "bf16_tflops": tb, "fp8_tflops": tf, "bf16_share_of_989": tb / 989, "fp8_share_of_1979": tf / 1979,
                     "speedup": ms["bf16"] / ms["fp8"]}
    return res


def forward_section(reps):
    from ln3diff_b200.utils import build_i23d, build_t23d
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(1)
    res = {}
    for name, build, B, ctx in (
            ("t23d_L2_B16", lambda: build_t23d("DiT-L/2", device=dev), 16, lambda B: torch.randn(B, 77, 768, generator=g)),
            ("i23d_pixart_L2_B64", lambda: build_i23d("DiT-PixArt-L/2", device=dev), 64,
             lambda B: {"vector": torch.randn(B, 768, generator=g), "crossattn": torch.randn(B, 256, 2048, generator=g)})):
        m = build()
        c = ctx(B)
        c = c.to(dev) if torch.is_tensor(c) else {k: v.to(dev) for k, v in c.items()}
        x = torch.randn(B, 12, 32, 32, generator=g).to(dev)
        t = torch.rand(B, generator=g).to(dev) * (900.0 if name.startswith("t23d") else 1.0)
        outs, ms = {}, {}
        for mode in ("bf16", "fp8"):                      # warm (graph capture) both modes
            m.set_gemm_precision(mode)
            outs[mode] = m(x, t, c)
        # alternating needs both modes' graphs resident: keep two models' worth of state by switching per sample
        times = {"bf16": [], "fp8": []}
        for _ in range(reps):
            for mode in ("bf16", "fp8"):
                m.set_gemm_precision(mode)
                m(x, t, c)                                  # capture after the switch (not timed)
                times[mode].append(event_ms(lambda: m(x, t, c), 5))
        ms = {k: statistics.median(v) for k, v in times.items()}
        res[name] = {"bf16_ms": ms["bf16"], "fp8_ms": ms["fp8"], "speedup": ms["bf16"] / ms["fp8"],
                     "rel_l2_fp8_vs_bf16": rel(outs["fp8"], outs["bf16"])}
        del m
        torch.cuda.empty_cache()
    return res


def sampling_section(steps):
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_ae_decoder, build_t23d, orbit_cameras
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(2)
    P = 8
    m = build_t23d("DiT-L/2", device=dev)
    x0 = torch.randn(P, 12, 32, 32, generator=g).to(dev)
    c = {"crossattn": torch.randn(P, 77, 768, generator=g).to(dev)}
    uc = {"crossattn": torch.zeros(P, 77, 768, device=dev)}
    dec = build_ae_decoder("DiT2-L/2", image_size=128, device=dev)
    cams = orbit_cameras(4).to(dev)
    res, lat, views = {}, {}, {}
    for mode in ("bf16", "fp8", "bf16", "fp8"):        # the second pass of each mode is the timed one
        m.set_gemm_precision(mode)
        pipeline.sample_t23d(m, x0, c, uc, 2, 6.5)      # graph capture outside the timed window
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lat[mode] = pipeline.sample_t23d(m, x0, c, uc, steps, 6.5)
        e1.record()
        torch.cuda.synchronize()
        res[f"{mode}_latents_per_s"] = P / (e0.elapsed_time(e1) / 1e3)
        torch.manual_seed(5)
        views[mode] = pipeline.decode_and_render(dec, lat[mode], cams, 128)
    res["rel_l2_latents"] = rel(lat["fp8"], lat["bf16"])
    res["rel_l2_views"] = {k: rel(views["fp8"][k], views["bf16"][k]) for k in views["bf16"]
                           if torch.is_tensor(views["bf16"][k]) and views["bf16"][k].is_floating_point()}
    res["steps"], res["prompts"] = steps, P
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=250)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py measures on a GPU; none is visible")
    name, power = smi("name,power.limit")
    out = {"gpu": name, "power_limit_w": float(power), "gemm": gemm_section(args.reps),
           "forward": forward_section(max(3, args.reps // 6)), "sample_t23d": sampling_section(args.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
