"""GPU measurement, not a test: reconstruction with the DiT2-L/2 VAE (vae_xl_reconstruction.sh: MVEncoderGSDynamicInp
with sd_E_ch=64, sd_E_num_res_blocks=1, 6 views of 10 x 256^2 per object, the DiT2-L/2 decoder, 192^2 renders at
96 + 96 samples per ray) on random weights.  Prints one JSON line with the card name and power limit read in the same
run.

  encode_xl_F6        pipeline.encode_latents with the XL encoder, 8 objects x 6 views: ms per object
  encode_mv_F4        the same with MVEncoder, 8 objects x 4 views: ms per object
  view_mean           ln3_view_mean_nhwc alone on the XL encoder's (48, 32, 32, 24) per-view moments: us per call
  render_192          render_views of one object's 8 views at 192^2, 64 + 64 and 96 + 96 samples (TF32 MLP): the median
                      over rounds of ms per view, the two sample counts alternated within each round
  reconstruct_xl      pipeline.reconstruct for 8 objects x 24 views at 192^2 (96 + 96): objects / s

Times come from CUDA events around `reps` calls after warm-up.

Run:  python tools/vae_xl_bench.py [--reps N]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_xl_bench.py measures the GPU path: no CUDA device")
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.utils import build_ae_decoder, build_ae_encoder, orbit_cameras
    dev = torch.device("cuda", 0)
    name, power_limit = smi("name,power.limit")
    res = {"gpu": name, "power_limit_w": float(power_limit), "conv_tf32": True, "mlp_tf32": True}
    g = torch.Generator().manual_seed(0)
    dec = build_ae_decoder("DiT2-L/2", image_size=192, depth_resolution=96, device=dev)
    B = 8
    for key, version, F in (("encode_xl_F6", "mv-sd-dit-dynaInp-trilatent", 6), ("encode_mv_F4", "mv-sd-dit", 4)):
        enc = build_ae_encoder(dino_version=version, device=dev)
        x = (torch.rand(B * F, 10, 256, 256, generator=g) * 2 - 1).to(dev)
        run = lambda: pipeline.encode_latents(enc, dec, x)
        for _ in range(3):
            run()
        ms = timed(run, args.reps)
        res[key] = {"objects": B, "views_per_object": F, "ms": round(ms, 3), "ms_per_object": round(ms / B, 3)}
    h = torch.randn(B * 6, 32, 32, 24, generator=g).to(dev)
    ops.view_mean_nhwc(h, 6)
    res["view_mean"] = {"shape": [B * 6, 32, 32, 24], "us": round(1e3 * timed(lambda: ops.view_mean_nhwc(h, 6), 200), 2)}

    # renderer: one object's planes from the decoder, 8 views at 192^2
    V, R = 8, 192
    lat = torch.randn(1, 12, 32, 32, generator=g).to(dev)
    planes_cl = dec.decode_to_channels_last(lat, in_mul=1.0)
    o, d = ops.generate_rays(orbit_cameras(V).to(dev).contiguous(), R)
    osg = dec.triplane_decoder.decoder.raw_parameters()
    noise = {S: (torch.rand(V, R * R, S, device=dev), torch.rand(V, R * R, S, device=dev)) for S in (64, 96)}
    render = {S: (lambda S=S: ops.render_views(planes_cl, o, d, noise[S][0], noise[S][1], osg, views_per_obj=V,
                                               mlp_tf32=True, samples_per_ray=S)) for S in (64, 96)}
    for S in (64, 96):
        render[S]()
    per_view = {64: [], 96: []}
    for _ in range(args.reps):
        for S in (64, 96):
            per_view[S].append(timed(render[S], 3) / V)
    med = {S: statistics.median(v) for S, v in per_view.items()}
    res["render_192"] = {"views": V, "ms_per_view_64_64": round(med[64], 3), "ms_per_view_96_96": round(med[96], 3),
                         "ratio_96_over_64": round(med[96] / med[64], 3), "rounds": args.reps}

    enc = build_ae_encoder(dino_version="mv-sd-dit-dynaInp-trilatent", device=dev)
    x = (torch.rand(B * 6, 10, 256, 256, generator=g) * 2 - 1).to(dev)
    cams = orbit_cameras(24).to(dev)
    run = lambda: pipeline.reconstruct(enc, dec, x, cams, resolution=R)
    run()
    ms = timed(run, max(1, args.reps // 5))
    res["reconstruct_xl"] = {"objects": B, "views": 24, "resolution": R, "samples_per_ray": 96, "ms": round(ms, 1),
                             "objects_per_s": round(B / (ms * 1e-3), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
