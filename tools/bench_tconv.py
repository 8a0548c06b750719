"""Device time of the persistent TAESD convolution (tconv.cu) alone: 64 -> 64 channels, 3x3, stride 1, bias + ReLU, with
and without a residual, at the 512x512 and 256x256 sizes of the TAESD body.  One JSON line per case:

    python tools/bench_tconv.py [--iters 50] [--reps 20]

Each case captures `--reps` launches into a CUDA graph, replays it warm `--iters` times between two CUDA events and reports
the time of one launch.  flop = 2 x pixels x 64 x 64 x 9; bytes = input once + output (+ residual), counted from the
shapes.  bound: which of flop / 989 TFLOP/s (dense FP16) and bytes / 3.35 TB/s (HBM3), the H100 SXM data-sheet peaks, is the
larger; pct_of_bound is that least time over the measured time.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_controlnet import card  # noqa: E402

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12


def run(h: int, w: int, res: bool, iters: int, reps: int) -> dict:
    import torch
    from ai_rtc_agent_b200.host import ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(h * 131 + w)
    x = torch.randn((1, h, w, 64), generator=g).half().to(dev)
    r = torch.randn((1, h, w, 64), generator=g).half().to(dev) if res else None
    wp = ops.pack_conv_weight((torch.randn((64, 64, 3, 3), generator=g) / math.sqrt(9 * 64)).half().to(dev))
    bias = torch.randn((1, 64), generator=g).float().to(dev)
    out = torch.empty((1, h, w, 64), dtype=torch.float16, device=dev)

    def launch():
        ops.igemm([(x, 9)], wp, out, colbias=bias, res=r, relu=True, tconv=True)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            launch()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            launch()
    for _ in range(3):
        graph.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        graph.replay()
    t1.record()
    torch.cuda.synchronize()
    sec = t0.elapsed_time(t1) / 1e3 / (iters * reps)
    flop = 2.0 * h * w * 64 * 64 * 9
    nbytes = (3 if res else 2) * h * w * 64 * 2
    t_mma, t_hbm = flop / PEAK_FLOPS, nbytes / PEAK_BYTES
    return {"size": f"{h}x{w}", "res": res, "us": round(sec * 1e6, 2), "tflops": round(flop / sec / 1e12, 1),
            "gbps": round(nbytes / sec / 1e9, 1), "bound": "mma" if t_mma >= t_hbm else "hbm",
            "pct_of_bound": round(100.0 * max(t_mma, t_hbm) / sec, 1)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_tconv: no CUDA device (the kernel has no CPU path)")
    info = card()
    for hw in (512, 256):
        for res in (False, True):
            row = run(hw, hw, res, args.iters, args.reps)
            row.update(info)
            print(json.dumps(row), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
