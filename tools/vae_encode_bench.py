"""GPU measurement, not a test: the stage-1 VAE encoder path (vae_reconstruction.sh: MVEncoder with sd_E_ch=64,
sd_E_num_res_blocks=1, 4 views of 10 x 256^2 per object, the DiT2-L/2 decoder) on random weights.  Prints one JSON line
with the card name and power limit read in the same run.

  encode_B1, encode_B8   pipeline.encode_latents (encoder + posterior sample) for 1 and 8 objects: ms per object and
                         the algorithmic TFLOP/s of the encoder (encoder_flops below, from the shapes)
  reconstruct_24x128     pipeline.reconstruct for one object: encode, decode, render 24 views at 128^2
  kernels_B8             per-kernel CUDA time of one encode_latents at B = 8, from a separate torch.profiler run

Times come from CUDA events around `reps` calls after warm-up (the profiler is off during them).

Run:  python tools/vae_encode_bench.py [--reps N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CH, CH_MULT, IN_CH, Z2, D = 64, (1, 2, 4, 4), 10, 24, 512


def encoder_flops(n_obj: int, res: int = 256, views: int = 4) -> float:
    """Algorithmic FLOPs (2 per multiply-add) of MVEncoder (one res block per level) for n_obj objects of `views` views
    at res^2: convolutions, the mid-block transformer (projections, attn1 over all views of an object, attn2 per view,
    GEGLU) and the fusion layer.  GroupNorm / LayerNorm / softmax element-wise work is not counted."""
    conv = lambda hw, cin, cout, k: 2.0 * hw * cin * cout * k * k
    r, cin = res, CH
    per_view = conv(r * r, IN_CH, CH, 3)
    for lvl, m in enumerate(CH_MULT):
        cout = CH * m
        per_view += conv(r * r, cin, cout, 3) + conv(r * r, cout, cout, 3) + (conv(r * r, cin, cout, 1) if cin != cout else 0)
        cin = cout
        if lvl != len(CH_MULT) - 1:
            r //= 2
            per_view += conv(r * r, cin, cin, 3)                          # Downsample
    L = r * r
    per_view += 2 * 2 * conv(L, cin, cin, 3)                              # mid block_1 / block_2
    per_view += conv(L, cin, D, 1) + conv(L, D, cin, 1)                   # proj_in / proj_out
    per_view += 2 * (2.0 * L * D * 4 * D)                                 # to_q/k/v + to_out of attn1 and attn2
    per_view += 2.0 * L * D * 8 * D + 2.0 * L * 4 * D * D                 # GEGLU in (D -> 8D) and ff out (4D -> D)
    per_view += 4.0 * L * L * D                                           # attn2 core (QK^T, PV) within the view
    per_view += conv(L, cin, Z2, 3)                                       # conv_out
    attn1 = 4.0 * (views * L) ** 2 * D                                    # attn1 core over the object's views * L tokens
    return n_obj * (views * per_view + attn1 + conv(L, views * Z2, Z2, 3))


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


def timed(fn, reps: int) -> float:
    """ms per call: CUDA events around `reps` calls."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def kernel_split(fn, top: int = 12) -> list:
    """[(kernel name, CUDA ms, share)] of one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            tot[e.name] = tot.get(e.name, 0.0) + e.device_time_total / 1e3
    total = sum(tot.values())
    rows = sorted(tot.items(), key=lambda kv: -kv[1])[:top]
    return [{"kernel": k[:90], "ms": round(v, 3), "share": round(v / total, 3)} for k, v in rows] + \
        [{"kernel": "TOTAL", "ms": round(total, 3), "share": 1.0}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_encode_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_ae_decoder, build_ae_encoder, orbit_cameras
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    res = {"gpu": name, "power_limit_w": float(power_limit), "views_per_object": 4, "input": [10, 256, 256],
           "conv_tf32": True}
    enc = build_ae_encoder(device=dev)
    dec = build_ae_decoder("DiT2-L/2", device=dev)
    g = torch.Generator().manual_seed(0)
    for B in (1, 8):
        x = (torch.rand(B * 4, 10, 256, 256, generator=g) * 2 - 1).to(dev)
        run = lambda: pipeline.encode_latents(enc, dec, x)
        for _ in range(3):
            run()
        ms = timed(run, args.reps)
        fl = encoder_flops(B)
        res[f"encode_B{B}"] = {"ms": round(ms, 3), "ms_per_object": round(ms / B, 3),
                               "algorithmic_gflop": round(fl / 1e9, 1), "tflops": round(fl / (ms * 1e-3) / 1e12, 1)}
        if B == 8:
            res["kernels_B8"] = kernel_split(run)
    x = (torch.rand(4, 10, 256, 256, generator=g) * 2 - 1).to(dev)
    cams = orbit_cameras(24).to(dev)
    run = lambda: pipeline.reconstruct(enc, dec, x, cams, resolution=128)
    run()
    ms = timed(run, max(1, args.reps // 2))
    res["reconstruct_24x128"] = {"ms": round(ms, 3), "objects": 1, "views": 24}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
