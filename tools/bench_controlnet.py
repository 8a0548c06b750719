"""Frames/s and per-frame latency of the engine without a ControlNet, with one whose control image is the frame itself
(controlnet_processor_id=None) and with one conditioned on the frame's HED edge map ("hed"), on seeded synthetic full-size
weights.  One JSON line per configuration:

    python tools/bench_controlnet.py [--frames 200] [--warmup 20]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) at 512x512 (the agent's default): none, ControlNet + None, ControlNet + HED;
  * SD-Turbo, T=1 ([32]) at 512x512: none, ControlNet + HED.

fps: back-to-back frames on one CUDA stream (one synchronise at the end).  p50/p99: a second pass with a synchronise after
every frame.  gflop_per_frame: the algorithmic FLOPs of the frame program's contractions (implicit GEMMs, halo convolutions,
attention) as the engine counts them from shapes, padded channels included; the direct small-channel convolutions (conv_in
layers, HED's first conv) and HED's projections are not included.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, check=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [v.strip() for v in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as exc:   # noqa: BLE001 - the numbers are still valid, only unlabelled
        return {"gpu": f"unknown ({exc})", "power_limit": "unknown"}


def run(model: str, t_index_list, controlnet: bool, processor, frames: int, warmup: int, hw: int = 512) -> dict:
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    cn = W.synthetic_controlnet(arch) if controlnet else None
    hed = A.synthetic_hed() if controlnet and processor == "hed" else None
    g = torch.Generator().manual_seed(1)
    emb = torch.randn((1, 77, arch.cross_attention_dim), generator=g).half()
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, controlnet_sd=cn, hed_sd=hed)
    sd.prepare("bench", guidance_scale=0.0)
    del usd, vsd, cn, hed
    frame = torch.randint(0, 256, (1, hw, hw, 3), dtype=torch.uint8, generator=g).cuda()
    out = torch.empty((1, 3, hw, hw), dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        sd.step_u8_into(frame, out)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(frames):
        sd.step_u8_into(frame, out)
    torch.cuda.synchronize()
    fps = frames / (time.perf_counter() - t0)
    lat = []
    for _ in range(frames):
        t1 = time.perf_counter()
        sd.step_u8_into(frame, out)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t1) * 1e3)
    lat.sort()
    flops = 0.0
    for kind in ("igemm", "tconv", "attn"):
        try:
            flops += sd.profile_kind(kind, iters=1)["flops"]
        except capi.B2Error:   # no launch of this kind in the program
            pass
    return {"model": arch.name, "t_index_list": list(t_index_list), "size": hw, "controlnet": controlnet,
            "controlnet_processor_id": processor if controlnet else None, "fps": round(fps, 2), "p50_ms": round(lat[len(lat) // 2], 3),
            "p99_ms": round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3), "gflop_per_frame": round(flops / 1e9, 1),
            "launches_per_frame": sd.launches_per_step}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet: no CUDA device (the engine has no CPU path)")
    info = card()
    sd15, turbo = ("lykon/dreamshaper-8", [18, 26, 35, 45]), ("stabilityai/sd-turbo", [32])
    for (model, tl), cn, proc in ((sd15, False, None), (sd15, True, None), (sd15, True, "hed"), (turbo, False, None),
                                  (turbo, True, "hed")):
        r = run(model, tl, cn, proc, args.frames, args.warmup)
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
