"""GPU measurement, not a test: the multi-view-to-3D release path (sample_obajverse_mv23d_dit.sh: 6 conditioning views,
ViT-B/14 9-channel DINOv2 conditioner, DiT-PixArt-MV-L/2, 4 samples, CFG 4.0, flow matching, 24 views at 192^2) on
random weights.  Prints one JSON line with the card name and power limit read in the same run.

  conditioner   GeneralConditioner.get_unconditional_conditioning on one 6-view condition (both passes, as eval_cldm)
  forward       one DiT-PixArt-MV-L/2 forward at B' = 8 (4 samples x CFG), context K/V cached, CUDA-graph replay;
                TFLOP/s from the algorithmic FLOPs of the shapes (flops_per_forward below)
  euler50       pipeline.sample_flow with a 50-point Euler ODE (49 forwards)
  dopri5        pipeline.sample_flow with the release default (dopri5, 250 output points); its NFE count depends on
                the velocity field, so with random weights it is not the count a trained checkpoint gives
  render        pipeline.decode_and_render of the 4 latents, 24 views at 192^2 (DiT2-L/2 decoder)

Run:  python tools/mv23d_bench.py [--skip-dopri5]
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


def flops_per_forward(B: int, T: int = 768, D: int = 1024, Lc: int = 1536, depth: int = 24) -> float:
    """Algorithmic FLOPs of the transformer blocks of one forward (2 per multiply-add), context K/V cached."""
    per = (2 * T * D * 3 * D          # qkv
           + 4 * T * T * D            # self-attention QK^T and PV
           + 2 * T * D * D            # proj
           + 2 * T * D * D            # cross q
           + 4 * T * Lc * D           # cross-attention core
           + 2 * T * D * D            # cross out
           + 2 * 2 * T * D * 4 * D)   # MLP
    return float(B * depth * per)


def timed(fn, reps: int = 1) -> float:
    """ms per call of fn (device-synchronised host clock)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-dopri5", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mv23d_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, build_mv23d, orbit_cameras
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    V, S = 6, 4
    res = {"gpu": name, "power_limit_w": float(power_limit), "views": V, "num_samples": S, "cfg_scale": 4.0}

    emb = FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", device=dev, n_cond_frames=V, enable_bf16=True, aug_c=True,
                                             random_init=True)
    emb._emb_config = {"input_key": "img-c", "ucg_rate": 0.1}
    cond = GeneralConditioner([emb])
    g = torch.Generator().manual_seed(0)
    imgs = (torch.rand(1, V, 3, 256, 256, generator=g) * 2 - 1).to(dev)
    mv_cams = orbit_cameras(V)[None].to(dev)
    run_cond = lambda: cond.get_unconditional_conditioning({"img-c": {"img": imgs, "c": mv_cams.clone()}},
                                                           force_uc_zero_embeddings=["img-c"])
    run_cond()
    res["conditioner_ms"] = timed(run_cond, 10)

    model = build_mv23d("DiT-PixArt-MV-L/2", device=dev)
    c, uc = pipeline.condition_prompt(cond, "img-c", {"img": imgs, "c": mv_cams.clone()}, S, device=dev)
    ctx = {"concat": torch.cat([c["concat"], uc["concat"]]).contiguous()}
    x = torch.randn(2 * S, 12, 32, 32, generator=g).to(dev)
    t = torch.full((2 * S,), 0.5, device=dev)
    for _ in range(3):
        model(x, t, ctx)
    ms = timed(lambda: model(x, t, ctx), 20)
    fl = flops_per_forward(2 * S)
    res["forward"] = {"batch": 2 * S, "context_tokens": V * 256, "ms": ms, "tflops": fl / (ms * 1e-3) / 1e12,
                      "algorithmic_tflop": fl / 1e12}

    pipeline.sample_flow(model, c, uc, S, num_steps=3, sampling_method="euler")
    ms = timed(lambda: pipeline.sample_flow(model, c, uc, S, num_steps=50, sampling_method="euler"))
    res["euler50"] = {"ms": ms, "latents_per_s": S / (ms * 1e-3), "forwards": 49}

    latents = pipeline.sample_flow(model, c, uc, S, num_steps=50, sampling_method="euler")
    if not args.skip_dopri5:
        nfe = [0]
        fwd = model.forward_with_cfg

        def counted(*a, **k):
            nfe[0] += 1
            return fwd(*a, **k)
        model.forward_with_cfg = counted
        ms = timed(lambda: pipeline.sample_flow(model, c, uc, S, num_steps=250))
        del model.forward_with_cfg
        res["dopri5_250"] = {"ms": ms, "latents_per_s": S / (ms * 1e-3), "nfe": nfe[0],
                             "note": "random weights: the NFE count of a trained checkpoint is not measured"}

    dec = build_ae_decoder("DiT2-L/2", device=dev)
    cams = orbit_cameras(24).to(dev)
    pipeline.decode_and_render(dec, latents, cams, 192)
    ms = timed(lambda: pipeline.decode_and_render(dec, latents, cams, 192), 3)
    res["decode_render_24x192"] = {"ms": ms, "latents": S, "views_per_latent": 24, "views_per_s": S * 24 / (ms * 1e-3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
