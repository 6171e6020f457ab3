"""Time the wgmma flash-attention kernel (`ops.fmha`) on the shapes the project runs, against torch SDPA.

    python tools/fmha_shapes.py [--lib PATH [--lib PATH ...]] [--rounds R] [--window-s S]

The shapes are the attention calls of bench.py's DiT-L/2 forward (self-attention over a packed qkv buffer, and
the conditional half's cross-attention to 77 text tokens with K/V strided per layer) and of the other forwards
that share the kernel: PixArt / MV23D cross-attention, self-attention with a second K/V source, the DiT2 decoder's
in-plane and global attention, and the causal CLIP text tower.  Every entry is timed with CUDA events over CUDA
graph replays filling a window of `--window-s` seconds, after a warm-up, in the same harness as
`tools/gemm_shapes.py`.  Algorithmic TFLOP/s counts 4 B H Lq Lkv 64 (QK^T and PV), halved for causal attention.
The yardstick is `F.scaled_dot_product_attention` in bf16 on the same inputs, with the backend torch chose.
Several `--lib` builds of libln3b200.so are timed alternately in one process, `--rounds` times each; the outputs
of every build are compared with the first build's, bit for bit (max abs and rel-L2 difference when they are not
identical).  Prints one line per (round, build, shape) and a final JSON line with the card name, power limit and
median SM clock sampled during the run.  Needs a GPU; it is a measurement, not a test.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from gemm_shapes import ClockPoll, smi, time_window  # noqa: E402

# name, B, H, Lq, Lkv, Lkv2 (second K/V source), causal, layout
#   packed: q/k/v are column slices of one (B, L, 3 H 64) buffer (dit_trilatent.py:323, vit_triplane.py:209)
#   kv:     q (B, Lq, H 64) and K/V slices of one (B, Lkv, 2 H 64) buffer (dit/_denoiser.py:split_kv)
#   layers: K/V of one layer inside a (B, Lkv, layers, 2, H 64) cache, the output a sub-batch view of a batch of
#           2 B (dit_trilatent.py:337)
SHAPES = [
    ("self_bench", 16, 16, 768, 768, 0, False, "packed"),
    ("cross_bench", 8, 16, 768, 77, 0, False, "layers"),
    ("cross_pixart", 8, 16, 768, 256, 0, False, "kv"),
    ("cross_mv23d", 8, 16, 768, 1536, 0, False, "kv"),
    ("self_second_kv", 8, 16, 768, 768, 257, False, "packed"),
    ("dec_inplane", 12, 16, 256, 256, 0, False, "packed"),
    ("dec_global", 4, 16, 768, 768, 0, False, "packed"),
    ("clip_causal", 8, 12, 77, 77, 0, True, "packed"),
]
LAYERS = 24


def flops(B, H, Lq, Lkv, Lkv2, causal):
    f = 4.0 * B * H * Lq * (Lkv + Lkv2) * 64
    return f / 2 if causal else f


def make_inputs(torch, dev, g, B, H, Lq, Lkv, Lkv2, layout):
    """(q, k, v, k2, v2, out) views laid out as the callers lay them out."""
    D = H * 64
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).bfloat16()
    k2 = v2 = None
    if layout == "packed":
        qkv = rnd(B, max(Lq, Lkv), 3 * D)
        q, k, v = qkv[:, :Lq, :D], qkv[:, :Lkv, D:2 * D], qkv[:, :Lkv, 2 * D:]
        out = torch.empty(B, Lq, D, device=dev, dtype=torch.bfloat16)
    elif layout == "kv":
        q, kv = rnd(B, Lq, D), rnd(B, Lkv, 2 * D)
        k, v = kv[:, :, :D], kv[:, :, D:]
        out = torch.empty(B, Lq, D, device=dev, dtype=torch.bfloat16)
    else:
        q = rnd(2 * B, Lq, D)[B:]
        kv = rnd(2 * B, Lkv, LAYERS, 2, D)
        k, v = kv[B:, :, LAYERS // 2, 0], kv[B:, :, LAYERS // 2, 1]
        out = torch.empty(2 * B, Lq, D, device=dev, dtype=torch.bfloat16)[B:]
    if Lkv2:
        dkv = rnd(B, Lkv2, 2 * D)
        k2, v2 = dkv[:, :, :D], dkv[:, :, D:]
    return q, k, v, k2, v2, out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="libln3b200.so to time (repeatable)")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--window-s", type=float, default=0.5)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend
    from ln3diff_b200 import _lib, ops

    if not torch.cuda.is_available():
        raise RuntimeError("tools/fmha_shapes.py needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    libs = [str(Path(p).resolve()) for p in (args.lib or [str(_lib.LIB_PATH)])]
    name, power_limit = smi("name,power.limit")
    g = torch.Generator(device=dev).manual_seed(0)
    inputs = {s[0]: make_inputs(torch, dev, g, *s[1:6], s[7]) for s in SHAPES}

    def ours(sname, H, causal):
        q, k, v, k2, v2, out = inputs[sname]
        return lambda: ops.fmha(q, k, v, H, out=out, k2=k2, v2=v2, causal=causal)

    def sdpa_args(sname, H):
        q, k, v, k2, v2, _ = inputs[sname]
        if k2 is not None:
            k, v = torch.cat([k, k2], 1), torch.cat([v, v2], 1)
        heads = lambda t: t.unflatten(2, (H, 64)).transpose(1, 2)
        return heads(q), heads(k), heads(v)

    def sdpa(sname, H, causal):
        q, k, v = sdpa_args(sname, H)
        return lambda: F.scaled_dot_product_attention(q, k, v, is_causal=causal)

    def sdpa_backend(sname, H, causal):
        try:
            return SDPBackend(torch._fused_sdp_choice(*sdpa_args(sname, H), is_causal=causal)).name
        except Exception:   # a private helper: the name is informative only
            return "unknown"

    # bit-identity of every build's outputs against the first build's (same inputs, one launch each)
    ref_out, diffs = {}, []
    for lib in libs:
        _lib._lib, _lib.LIB_PATH = None, Path(lib)     # ops.fmha resolves the library on every call
        for sname, B, H, Lq, Lkv, Lkv2, causal, _ in SHAPES:
            inputs[sname][5].fill_(0)
            ours(sname, H, causal)()
            torch.cuda.synchronize()
            o = inputs[sname][5].clone()
            if sname not in ref_out:
                ref_out[sname] = o
                continue
            r = ref_out[sname]
            same = torch.equal(o.view(torch.int16), r.view(torch.int16))
            d = (o.float() - r.float())
            row = {"impl": lib, "shape": sname, "bit_identical": same, "max_abs": d.abs().max().item(),
                   "rel_l2": (d.norm() / r.float().norm()).item()}
            diffs.append(row)
            print(f"compare {sname:15s} bit-identical={same} max_abs={row['max_abs']:.3e} "
                  f"rel_l2={row['rel_l2']:.3e}  {lib}", flush=True)

    clock = ClockPoll()
    rows = []
    try:
        for r in range(args.rounds):
            for lib in libs:
                _lib._lib, _lib.LIB_PATH = None, Path(lib)
                for sname, B, H, Lq, Lkv, Lkv2, causal, _ in SHAPES:
                    ms = time_window(torch, ours(sname, H, causal), args.window_s)
                    tf = flops(B, H, Lq, Lkv, Lkv2, causal) / (ms / 1e3) / 1e12
                    rows.append({"round": r, "impl": lib, "shape": sname, "B": B, "H": H, "Lq": Lq, "Lkv": Lkv,
                                 "Lkv2": Lkv2, "causal": causal, "us": 1e3 * ms, "tflops": tf})
                    print(f"round {r} {sname:15s} B={B:3d} H={H:2d} Lq={Lq:4d} Lkv={Lkv:4d}+{Lkv2:3d} "
                          f"{1e3 * ms:9.1f} us {tf:7.1f} TFLOP/s  {lib}", flush=True)
            for sname, B, H, Lq, Lkv, Lkv2, causal, _ in SHAPES:
                ms = time_window(torch, sdpa(sname, H, causal), args.window_s)
                tf = flops(B, H, Lq, Lkv, Lkv2, causal) / (ms / 1e3) / 1e12
                backend = sdpa_backend(sname, H, causal)
                rows.append({"round": r, "impl": "sdpa", "backend": backend, "shape": sname, "us": 1e3 * ms,
                             "tflops": tf})
                print(f"round {r} {sname:15s} B={B:3d} H={H:2d} Lq={Lq:4d} Lkv={Lkv:4d}+{Lkv2:3d} "
                      f"{1e3 * ms:9.1f} us {tf:7.1f} TFLOP/s  sdpa bf16 ({backend})", flush=True)
    finally:
        sm_mhz = clock.stop()
    print(json.dumps({"gpu": name, "power_limit_w": float(power_limit), "sm_mhz_median": sm_mhz,
                      "window_s": args.window_s, "compare": diffs, "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
