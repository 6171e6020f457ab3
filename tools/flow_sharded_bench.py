"""GPU measurement, not a test: sharded image-to-3D (pipeline.images_to_3d_sharded), one rank per GPU over NCCL, for
G = 1 up to the visible device count (or the counts given with --gpus).

  workload  the I23D release path on random weights: OpenCLIP ViT-L/14 + DINOv2 ViT-L/14-reg conditioner (both
            towers on every image, in its conditional and unconditional pass), DiT-PixArt-L/2, N = 4 samples per
            image, CFG 4.0, dopri5 with 250 output points, DiT2-L/2 decode and 24 views at 192^2 (64 + 64 samples),
            uint8 frames all-gathered once per batch
  scale     P = 8 images per GPU in one local batch, so G GPUs run 8 G distinct images
  check     before timing, every rank compares the latents of its images with a 1-GPU run of the same images (the
            G = 1 phase runs all 8 Gmax images once, untimed, in batches of 4, so every timed batch of 8 holds a
            different mix of images than the reference batches that produced its images' latents): rel-L2 <= 1e-2
            per image, the tolerance tests/test_gpu_flow_batch.py applies between batched and single calls
  timing    per G: that untimed run (also the warm-up: graphs captured, NCCL set up), then --repeats timed runs.  A
            run's time is the slowest rank's (host clock from a barrier to a device synchronise after the call,
            all-reduced with MAX); the median run is reported.

Reports conditions/s, latents/s, rendered views/s, the per-image dopri5 forward counts and the scaling efficiency
(the G-GPU rate over G times the 1-GPU rate), with the card name and power limit read in the same run.  A batch ends
when its slowest image ends, so a rank's time follows the slowest image of its batch; on random weights dopri5's
forward counts say nothing about a trained checkpoint.  Every worker is joined before the tool exits.  Prints one
JSON line.

Run:  python tools/flow_sharded_bench.py [--gpus 1 2 4 8] [--repeats 3]
"""
import argparse
import datetime
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PER_GPU, N, VIEWS, RES, TOL = 8, 4, 24, 192, 1e-2


def smi(query: str) -> list[list[str]]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout
    return [[f.strip() for f in line.split(",")] for line in out.strip().splitlines()]


def images(P: int) -> torch.Tensor:
    """P seeded images; the first k are the same whatever P is."""
    g = torch.Generator().manual_seed(0)
    return torch.cat([torch.rand(1, 3, 256, 256, generator=g) * 2 - 1 for _ in range(P)])


def build(dev):
    from ln3diff_b200.sgm.modules.encoders.modules import (FrozenDinov2ImageEmbedder, FrozenOpenCLIPImageEmbedder,
                                                           GeneralConditioner)
    from ln3diff_b200.utils import build_ae_decoder, build_i23d, orbit_cameras
    clip = FrozenOpenCLIPImageEmbedder(device=dev, output_tokens=True, random_init=True)
    dino = FrozenDinov2ImageEmbedder(device=dev, random_init=True)
    for e in (clip, dino):                       # sgm/configs/img23d-clipl-compat-fm-lognorm.yaml
        e._emb_config = {"input_key": "img", "ucg_rate": 0.1}
    return (GeneralConditioner([clip, dino]), build_i23d("DiT-PixArt-L/2", device=dev),
            build_ae_decoder("DiT2-L/2", device=dev), orbit_cameras(VIEWS).to(dev))


def worker(rank, world, port, g_max, repeats, ref_path, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, timeout=datetime.timedelta(minutes=20),
                            device_id=dev)
    try:
        from ln3diff_b200 import _lib, pipeline
        _lib.lib()
        cond, model, dec, cams = build(dev)
        run = lambda imgs, batch=PER_GPU: pipeline.images_to_3d_sharded(cond, model, dec, imgs, cams, num_samples=N,
                                                                        resolution=RES, batch=batch)
        P = PER_GPU * world
        if world == 1:                           # the 1-GPU reference of every image any G runs, in batches of half
            ref = run(images(PER_GPU * g_max), PER_GPU // 2)["latents"].cpu()
            torch.save(ref, ref_path)
        first = run(images(P))
        ref = torch.load(ref_path)
        lo, hi = first["shard"]
        rel = max(float((first["latents"][i].double().cpu() - ref[lo + i].double()).norm() / ref[lo + i].double().norm())
                  for i in range(hi - lo))
        worst = torch.tensor([rel], device=dev)
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        if worst.item() > TOL:
            raise RuntimeError(f"G = {world}: latents differ from the 1-GPU run by rel-L2 {worst.item():.3e} > {TOL}")
        imgs = images(P)
        times, nfe = [], None
        for _ in range(repeats):
            dist.barrier()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run(imgs)
            torch.cuda.synchronize()
            t = torch.tensor([time.perf_counter() - t0], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            times.append(t.item())
            nfe = out["stats"]["nfe"]
        nfes = [None] * world
        dist.all_gather_object(nfes, nfe)
        if rank == 0:
            s = sorted(times)[len(times) // 2]
            ret[world] = {"gpus": world, "conditions": P, "s": s, "s_all": times, "conditions_per_s": P / s,
                          "latents_per_s": P * N / s, "views_per_s": P * N * VIEWS / s, "check_max_rel_l2": worst.item(),
                          "nfe_per_rank": nfes, "gather_bytes_per_rank": out["gather_bytes_per_rank"]}
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, nargs="+", default=None, help="GPU counts to run (default 1 .. visible)")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_sharded_bench.py measures the GPU path: no CUDA device")
    import torch.multiprocessing as mp
    visible = torch.cuda.device_count()
    counts = sorted(set(args.gpus or range(1, visible + 1)) | {1})
    if counts[-1] > visible:
        raise SystemExit(f"--gpus asks for {counts[-1]} GPUs; {visible} visible")
    cards = smi("name,power.limit")[:counts[-1]]
    res = {"gpus_visible": visible, "cards": [{"name": c[0], "power_limit_w": float(c[1])} for c in cards],
           "workload": f"images_to_3d_sharded: OpenCLIP ViT-L/14 + DINOv2 ViT-L/14-reg, DiT-PixArt-L/2 (random "
                       f"weights), {PER_GPU} images per GPU, N = {N}, CFG 4.0, dopri5 250 points, DiT2-L/2 decode, "
                       f"{VIEWS} views at {RES}^2", "runs": []}
    with tempfile.TemporaryDirectory() as tmp, mp.Manager() as mgr:
        ref_path = os.path.join(tmp, "latents_1gpu.pt")
        for i, G in enumerate(counts):
            ret = mgr.dict()
            mp.spawn(worker, args=(G, 29700 + (os.getpid() + i) % 2000, counts[-1], args.repeats, ref_path, ret),
                     nprocs=G, join=True)
            row = dict(ret[G])
            row["efficiency"] = row["conditions_per_s"] / (G * res["runs"][0]["conditions_per_s"]) if res["runs"] else 1.0
            res["runs"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
