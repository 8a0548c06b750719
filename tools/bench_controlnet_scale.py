"""Cost of the ControlNet conditioning scale and guidance window (DESIGN §4.12) on seeded synthetic full-size weights at
512x512, ControlNet + HED, one JSON line per measurement:

    python tools/bench_controlnet_scale.py [--frames 200] [--warmup 20]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) and SD-Turbo, T=1 ([32]);
  * settings: the defaults (1, 0, 1), scale 0.6, and a window that masks half the slots (T=4: end 0.6 keeps 2 of 4 slots;
    T=1: the one slot masked, start 0.7);
  * fps: back-to-back frames on one CUDA stream (one synchronise at the end); p50 / p99: a second pass with a synchronise
    after every frame;
  * zero_conv_ms: device time per frame of the 13 zero-conv launches (the igemm_ascale_kernel instantiations, which nothing
    else launches), from a torch.profiler run of its own;
  * update_ms: host time of one global update (StreamDiffusion.set_control_scale on the engine) and of one per-viewer update
    (StreamState.set_control_scale), each ending in a device synchronise, median of 50;
  * viewers_fps: four viewers with different settings on the default lanes (T=4: 2 lanes stepping 4 states in turn; T=1: 8
    lanes), frames submitted round-robin on the lanes' own CUDA streams.
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

SETTINGS = {"defaults": (1.0, 0.0, 1.0), "scale 0.6": (0.6, 0.0, 1.0)}
HALF_MASK = {4: (1.0, 0.0, 0.6), 1: (1.0, 0.7, 1.0)}   # T -> a window masking half the slots (T=1: its one slot)


def build(model, t_index_list, hw=512, lanes=1):
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    g = torch.Generator().manual_seed(1)
    emb = torch.randn((1, 77, arch.cross_attention_dim), generator=g).half()
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw,
                         controlnet_sd=W.synthetic_controlnet(arch), hed_sd=A.synthetic_hed())
    if lanes > 1:
        sd.set_concurrency(lanes)
    sd.prepare("bench", guidance_scale=0.0)
    frame = torch.randint(0, 256, (1, hw, hw, 3), dtype=torch.uint8, generator=g).cuda()
    return sd, frame


def rate(sd, frame, frames, warmup):
    import torch
    out = torch.empty((1, 3, sd.height, sd.width), dtype=torch.uint8, device="cuda")
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
    return round(fps, 2), round(lat[len(lat) // 2], 3), round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3)


def zero_conv_ms(sd, frame, n=20):
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = torch.empty((1, 3, sd.height, sd.width), dtype=torch.uint8, device="cuda")
    sd.step_u8_into(frame, out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            sd.step_u8_into(frame, out)
        torch.cuda.synchronize()
    us, count = 0.0, 0
    for e in prof.events():
        if e.device_type.name == "CUDA" and "igemm_ascale_kernel" in e.name:
            us += e.device_time
            count += 1
    return round(us / n / 1e3, 4), count / n


def update_ms(fn, n=50):
    import torch
    ts = []
    for i in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(i)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ts), 4)


def viewers_fps(model, tl, lanes, frames, warmup):
    import torch
    sd, frame = build(model, tl, lanes=lanes)
    pool = [sd] + [sd.add_lane() for _ in range(lanes - 1)]
    streams = [torch.cuda.Stream() for _ in pool]
    states = [sd.new_state() for _ in range(4)]
    states[1].set_control_scale(0.6)
    states[2].set_control_scale(*HALF_MASK[len(tl)])
    states[3].set_control_scale(-0.5, 0.2, 1.0)
    outs = [torch.empty((1, 3, sd.height, sd.width), dtype=torch.uint8, device="cuda") for _ in pool]
    torch.cuda.synchronize()

    def go(n):
        # frame i of viewer k on lane (i * 4 + k) % lanes; one viewer's consecutive frames are ordered by its state's event
        for i in range(n):
            for k, st in enumerate(states):
                j = (i * 4 + k) % lanes
                with torch.cuda.stream(streams[j]):
                    pool[j].step_u8_into(frame, outs[j], state=st)
        torch.cuda.synchronize()
    go(max(1, warmup // 4))
    t0 = time.perf_counter()
    go(max(1, frames // 4))
    return round(4 * max(1, frames // 4) / (time.perf_counter() - t0), 2)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet_scale: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl, lanes in (("lykon/dreamshaper-8", [18, 26, 35, 45], 2), ("stabilityai/sd-turbo", [32], 8)):
        sd, frame = build(model, tl)
        settings = dict(SETTINGS, **{"half the slots masked": HALF_MASK[len(tl)]})
        for name, control in settings.items():
            sd.set_control_scale(*control)
            fps, p50, p99 = rate(sd, frame, args.frames, args.warmup)
            zc, n_zc = zero_conv_ms(sd, frame)
            r = {"model": sd.arch.name, "t_index_list": tl, "size": 512, "controlnet_processor_id": "hed", "settings": name,
                 "control": control, "fps": fps, "p50_ms": p50, "p99_ms": p99, "zero_conv_ms": zc,
                 "zero_conv_launches": n_zc, "launches_per_frame": sd.launches_per_step}
            r.update(info)
            print(json.dumps(r), flush=True)
        st = sd.new_state()
        r = {"model": sd.arch.name, "t_index_list": tl, "measure": "update",
             "global_update_ms": update_ms(lambda i: sd.set_control_scale(0.5 + 0.01 * (i % 2))),
             "viewer_update_ms": update_ms(lambda i: st.set_control_scale(0.5 + 0.01 * (i % 2)))}
        r.update(info)
        print(json.dumps(r), flush=True)
        st.close()
        del sd, st
        torch.cuda.empty_cache()
        r = {"model": model, "t_index_list": tl, "measure": "4 viewers", "lanes": lanes,
             "viewers_fps": viewers_fps(model, tl, lanes, args.frames, args.warmup)}
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
