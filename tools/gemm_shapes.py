"""Time the wgmma GEMM (`ops.gemm`) on the DiT-L/2 forward's hot shapes against cuBLAS on the same inputs.

    python tools/gemm_shapes.py [--lib PATH [--lib PATH ...]] [--rounds R] [--window-s S]

The first six shapes are the per-layer GEMMs of `dit/_denoiser.py::run_blocks` at bench.py's batch (8 prompts
with CFG = 16 samples of 768 tokens, D = 1024), each with its production epilogue; fc1 runs the default
erf-GELU.  The last is the CLIP text tower's qkv for 8 prompts (616 rows, a small GEMM of partial tiles).  The
yardstick is `torch.nn.functional.linear` in bf16 (cuBLAS), with `F.gelu` applied separately for fc1.  Every entry is timed with CUDA events over enough back-to-back launches to fill a window of
`--window-s` seconds, after a warm-up.  Several `--lib` builds of libln3b200.so are timed alternately in one
process on the same inputs, `--rounds` times each, so that two builds can be compared under the same clocks; the
outputs of every build are compared with the first build's, bit for bit (max abs and rel-L2 difference when they
are not identical).  Prints one line per (round, build, shape) and a final JSON line with the card name, power limit and the median SM
clock sampled during the run.  Needs a GPU; it is a measurement, not a test.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

B, T, D = 16, 768, 1024
M, MH = B * T, B * T // 2           # all tokens; the conditional half (cross-attention rows)
# name, M, N, K, bias, activation (ops.ACT_*)
SHAPES = [
    ("qkv", M, 3 * D, D, True, "none"),
    ("proj", M, D, D, True, "none"),
    ("cross_q", MH, D, D, False, "none"),
    ("cross_out", MH, D, D, True, "none"),
    ("fc1", M, 4 * D, D, True, "gelu_erf"),
    ("fc2", M, D, 4 * D, True, "none"),
    ("clip_qkv", 8 * 77, 3 * 768, 768, True, "none"),
]


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [f.strip() for f in out.strip().splitlines()[0].split(",")]


class ClockPoll:
    """Samples the SM clock every 100 ms while the timed windows run."""

    def __init__(self):
        self.mhz = []
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                      "-lms", "100", "-i", "0"], stdout=subprocess.PIPE, text=True)
        self.thread = threading.Thread(target=self._read, daemon=True)
        self.thread.start()

    def _read(self):
        for line in self.proc.stdout:
            try:
                self.mhz.append(float(line.strip()))
            except ValueError:
                pass

    def stop(self) -> float | None:
        self.proc.terminate()
        self.proc.wait()
        self.thread.join(timeout=5)
        s = sorted(self.mhz)
        return s[len(s) // 2] if s else None


def time_window(torch, fn, window_s: float, per_graph: int = 20) -> float:
    """Mean ms per call of `fn` over back-to-back launches filling >= window_s, after a warm-up.  The launches are
    replayed from a CUDA graph of `per_graph` calls: the small shapes run ~20 us, about what one call costs on the
    host, so eager launches would time the host."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    n = max(2, int(window_s / (e0.elapsed_time(e1) / 1e3)) + 1)
    e0.record()
    for _ in range(n):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (n * per_graph)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="libln3b200.so to time (repeatable)")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--window-s", type=float, default=0.5)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from ln3diff_b200 import _lib, ops

    if not torch.cuda.is_available():
        raise RuntimeError("tools/gemm_shapes.py needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    libs = [str(Path(p).resolve()) for p in (args.lib or [str(_lib.LIB_PATH)])]
    name, power_limit = smi("name,power.limit")
    g = torch.Generator(device=dev).manual_seed(0)
    inputs = {}
    for sname, m, n, k, bias, act in SHAPES:
        a = torch.randn(m, k, device=dev, generator=g).bfloat16()
        w = (torch.randn(n, k, device=dev, generator=g) / k ** 0.5).bfloat16()
        b = torch.randn(n, device=dev, generator=g) if bias else None
        inputs[sname] = (a, w, b, torch.empty(m, n, device=dev, dtype=torch.bfloat16))

    def ours(sname, act):
        a, w, b, out = inputs[sname]
        return lambda: ops.gemm(a, w, b, act=ops.ACT_GELU_ERF if act == "gelu_erf" else ops.ACT_NONE, out=out)

    def cublas(sname, act):
        a, w, b, _ = inputs[sname]
        bb = b.bfloat16() if b is not None else None
        if act == "gelu_erf":
            return lambda: F.gelu(F.linear(a, w, bb))
        return lambda: F.linear(a, w, bb)

    # bit-identity of every build's outputs against the first build's (same inputs, one launch each)
    ref_out, diffs = {}, []
    for lib in libs:
        _lib._lib, _lib.LIB_PATH = None, Path(lib)     # ops.gemm resolves the library on every call
        for sname, *_, act in SHAPES:
            out = inputs[sname][3]
            out.fill_(0)
            ours(sname, act)()
            torch.cuda.synchronize()
            o = out.clone()
            if sname not in ref_out:
                ref_out[sname] = o
                continue
            r = ref_out[sname]
            same = torch.equal(o.view(torch.int16), r.view(torch.int16))
            d = o.float() - r.float()
            row = {"impl": lib, "shape": sname, "bit_identical": same, "max_abs": d.abs().max().item(),
                   "rel_l2": (d.norm() / r.float().norm()).item()}
            diffs.append(row)
            print(f"compare {sname:10s} bit-identical={same} max_abs={row['max_abs']:.3e} "
                  f"rel_l2={row['rel_l2']:.3e}  {lib}", flush=True)

    clock = ClockPoll()
    rows = []
    try:
        for r in range(args.rounds):
            for lib in libs:
                _lib._lib, _lib.LIB_PATH = None, Path(lib)
                for sname, m, n, k, _, act in SHAPES:
                    ms = time_window(torch, ours(sname, act), args.window_s)
                    tf = 2.0 * m * n * k / (ms / 1e3) / 1e12
                    rows.append({"round": r, "impl": lib, "shape": sname, "M": m, "N": n, "K": k, "act": act,
                                 "us": 1e3 * ms, "tflops": tf})
                    print(f"round {r} {sname:10s} {m:6d}x{n:5d}x{k:5d} {act:8s} {1e3 * ms:9.1f} us "
                          f"{tf:7.1f} TFLOP/s  {lib}", flush=True)
            for sname, m, n, k, _, act in SHAPES:
                ms = time_window(torch, cublas(sname, act), args.window_s)
                tf = 2.0 * m * n * k / (ms / 1e3) / 1e12
                rows.append({"round": r, "impl": "cublas", "shape": sname, "M": m, "N": n, "K": k, "act": act,
                             "us": 1e3 * ms, "tflops": tf})
                print(f"round {r} {sname:10s} {m:6d}x{n:5d}x{k:5d} {act:8s} {1e3 * ms:9.1f} us "
                      f"{tf:7.1f} TFLOP/s  cublas (F.linear bf16{' + F.gelu' if act != 'none' else ''})", flush=True)
    finally:
        sm_mhz = clock.stop()
    print(json.dumps({"gpu": name, "power_limit_w": float(power_limit), "sm_mhz_median": sm_mhz,
                      "window_s": args.window_s, "compare": diffs, "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
