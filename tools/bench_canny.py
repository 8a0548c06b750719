"""Cost of the Canny ControlNet processor (DESIGN §4.14) on seeded synthetic full-size weights at 512x512, one JSON line per
measurement:

    python tools/bench_canny.py [--frames 200] [--warmup 20] [--profile-frames 20]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) and SD-Turbo, T=1 ([32]);
  * nets: none, Canny, HED, and Canny + frame;
  * fps and p50 / p99 as tools/bench_multi_controlnet.py measures them, and launches_per_frame;
  * canny_ms: device time of the Canny launches per frame (canny_head and the four hysteresis launches), from torch.profiler's
    CUDA kernel records in a run of its own, over --profile-frames frames;
  * threshold_update_ms: host time of one global and one per-viewer threshold update (host values only: no synchronise is
    needed, none is timed), median of 200.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_controlnet import card  # noqa: E402
from bench_controlnet_scale import rate  # noqa: E402

NETS = {"none": [], "canny": ["canny"], "hed": ["hed"], "canny+frame": ["canny", None]}


def build(model, t_index_list, procs, hw=512):
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    g = torch.Generator().manual_seed(1)
    emb = torch.randn((1, 77, arch.cross_attention_dim), generator=g).half()
    kw = {}
    if procs:
        nets = [W.synthetic_controlnet(arch, seed=5678 + i) for i in range(len(procs))]
        kw = dict(controlnet_sd=nets[0] if len(procs) == 1 else nets, control_processors=procs,
                  hed_sd=A.synthetic_hed() if "hed" in procs else None)
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, **kw)
    sd.prepare("bench", guidance_scale=0.0)
    # a camera-like frame: smooth shapes and noise, so that Canny finds edges of every strength
    from oracle import weights as ow
    return sd, ow.make_frame(hw, hw, seed=3).cuda()


def canny_device_ms(sd, frame, frames):
    """device time of the Canny kernels per frame, from torch.profiler's kernel records"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = torch.empty((1, 3, sd.height, sd.width), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        sd.step_u8_into(frame, out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            sd.step_u8_into(frame, out)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "canny" in e.key)
    return round(us / 1e3 / frames, 4)


def host_ms(fn, n=200):
    ts = []
    for i in range(n):
        t0 = time.perf_counter()
        fn(i)
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ts), 4)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-frames", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_canny: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl in (("lykon/dreamshaper-8", [18, 26, 35, 45]), ("stabilityai/sd-turbo", [32])):
        for name, procs in NETS.items():
            sd, frame = build(model, tl, procs)
            fps, p50, p99 = rate(sd, frame, args.frames, args.warmup)
            r = {"model": sd.arch.name, "t_index_list": tl, "size": 512, "nets": name, "fps": fps, "p50_ms": p50,
                 "p99_ms": p99, "launches_per_frame": sd.launches_per_step}
            if "canny" in procs:
                r["canny_ms"] = canny_device_ms(sd, frame, args.profile_frames)
                st = sd.new_state()
                r["global_threshold_update_ms"] = host_ms(lambda i: sd.set_canny_thresholds(100 + i % 2, 200))
                r["viewer_threshold_update_ms"] = host_ms(lambda i: st.set_canny_thresholds(100 + i % 2, 200))
                st.close()
            r.update(info)
            print(json.dumps(r), flush=True)
            del sd
            torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
