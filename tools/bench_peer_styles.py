"""Viewers with their own style LoRAs (PeerStream.update_lora) on one per-peer pipeline, on seeded synthetic weights at 512x512:

    python tools/bench_peer_styles.py [--models sd15,turbo] [--frames 48] [--rank 64]

sd15: SD-1.5 topology with the LCM schedule, T = 4, 2 lanes per pool; turbo: SD-Turbo topology, T = 1, 8 pipeline lanes (a
style has 2).  For 2 / 4 / 8 viewers over 1 / 2 / 4 styles (viewer k uses style k mod styles; style 0 is the pipeline's own
weights, so "1 style" runs every viewer on the pipeline's lanes), each viewer keeps 2 frames pending.  One JSON line per
configuration, then per model:
  * fps: aggregate frames/s over all viewers; p50 / p99 of the slowest viewer (submit -> result);
  * build_host_ms / cached_host_ms: wall time of an update_lora that builds a style, and of one that switches to a cached one;
  * build_device_ms: device time of the build's launches and copies (torch.profiler, a build of its own);
  * store_mib / lanes_mib: device memory of one style's weight store (its first engine) and of its further lanes;
  * gap_ms / idle_gap_ms: the longest gap between the device completions of consecutive frames of another viewer when a
    style is built among them, and the same without a build.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import gc
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_controlnet import card  # noqa: E402
from tools.bench_lora_switch import _pct, write_lora  # noqa: E402

MODELS = {"sd15": ("lykon/dreamshaper-8", [18, 26, 35, 45]), "turbo": ("stabilityai/sd-turbo", [32])}


def pipeline(model, tl, usd, vsd):
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    W.register_preloaded(model, A.arch_for(model), usd, vsd)
    try:
        p = StreamDiffusionPipeline(model, t_index_list=tl, width=512, height=512, live_lora=True, per_peer_streams=True)
    finally:
        W._PRELOADED.pop(model, None)
    torch.cuda.synchronize()
    return p


def used():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    return total - free


def run_viewers(views, frames, n):
    """every viewer submits n frames round robin with 2 pending each: (aggregate fps, per-viewer latencies)"""
    lat = [[] for _ in views]
    pending = [[] for _ in views]
    t_start = time.perf_counter()
    for i in range(n):
        for k, v in enumerate(views):
            pending[k].append((time.perf_counter(), v.enqueue(frames[(i + k) % len(frames)])))
            if len(pending[k]) == 2:
                t0, tk = pending[k].pop(0)
                tk.result()
                lat[k].append((time.perf_counter() - t0) * 1e3)
    for k in range(len(views)):
        for t0, tk in pending[k]:
            tk.result()
            lat[k].append((time.perf_counter() - t0) * 1e3)
    return len(views) * n / (time.perf_counter() - t_start), lat


def bench_model(name, args, tmp, dev):
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from ai_rtc_agent_b200.host import arch as A
    from oracle import weights as ow
    model, tl = MODELS[name]
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    loras = [None]
    for s in range(1, 5):
        path = os.path.join(tmp, f"{name}{s}.safetensors")
        write_lora(path, usd, args.rank, s)
        loras.append({path: 1.0})
    frames = [ow.make_frame(512, 512, seed=i).cuda() for i in range(8)]
    os.environ["B200SD_MAX_STYLES"] = "4"
    p = pipeline(model, tl, usd, vsd)
    rows = []
    for viewers, styles in ((2, 1), (2, 2), (4, 1), (4, 2), (4, 4), (8, 1), (8, 2), (8, 4)):
        views = [p.open_stream() for _ in range(viewers)]
        for k, v in enumerate(views):
            if k % styles:
                v.update_lora(loras[k % styles])
        run_viewers(views, frames, 4)   # warm-up: first launches of every lane
        fps, lat = run_viewers(views, frames, args.frames)
        slow = max(lat, key=lambda xs: _pct(xs, 0.5))
        rows.append(dict(model=name, viewers=viewers, styles=styles, fps=fps, slowest_p50_ms=_pct(slow, 0.5),
                         slowest_p99_ms=_pct(slow, 0.99), styles_held=p.styles))
        print(json.dumps(dict(rows[-1], device=dev)), flush=True)
        for v in views:
            v.close()
    # builds and cached switches, and the gaps between another viewer's frames (device completion times) with and without a
    # build in the middle of them
    for key in list(p._styles):
        p._evict(key)
    base = used()
    other, v = p.open_stream(), p.open_stream()
    run_viewers([other, v], frames, 4)

    def gaps_around(update, n=24):
        """the longest gap between consecutive completions of n frames of `other`, with update() called after n // 2"""
        stamps, t0 = [], torch.cuda.Event(enable_timing=True)
        t0.record()
        for i in range(n):
            if i == n // 2:
                update()
            other.enqueue(frames[i % 8])
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(p._lane_streams[(p._next_lane - 1) % p.lanes] or torch.cuda.current_stream())
            stamps.append(ev)
        torch.cuda.synchronize()
        done = sorted(t0.elapsed_time(e) for e in stamps)
        return max(b - a for a, b in zip(done, done[1:]))

    build, cached, gaps, idle_gaps = [], [], [], []
    for k in range(3):
        idle_gaps.append(gaps_around(lambda: None))
        t = []
        gaps.append(gaps_around(lambda: (t.append(time.perf_counter()), v.update_lora(loras[1 + k]),
                                         t.append(time.perf_counter()))))
        build.append((t[1] - t[0]) * 1e3)
        if k == 0:
            store_and_lanes = used() - base
    for k in range(4):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v.update_lora(loras[1 + k % 3])
        cached.append((time.perf_counter() - t0) * 1e3)
    # the memory of one style: its first engine (the store and that engine), then each further lane
    for key in list(p._styles):
        if p._styles[key].users == 0:
            p._evict(key)
    sd = p.model.stream
    u0 = used()
    style = sd.add_style()
    u1 = used()
    style.add_lane()
    u2 = used()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s2 = sd.add_style()
        s2.add_lane()
        from ai_rtc_agent_b200.host.weights import lora_factors
        s2.apply_factors(lora_factors(sd._unet_shapes, loras[4]))
        torch.cuda.synchronize()
    build_device_ms = sum(getattr(e, "device_time_total", 0.0) for e in prof.events() if e.device_type == DeviceType.CUDA) / 1e3
    after = torch.cuda.Stream()
    after.wait_stream(torch.cuda.current_stream())
    sd.drop_style(style, after)
    sd.drop_style(s2, after)
    summary = dict(summary=True, model=name, model_id=model, T=len(tl), size=512, rank=args.rank, pipeline_lanes=p.lanes,
                   build_host_ms=build, cached_host_ms=cached, build_device_ms=build_device_ms, gap_ms=gaps,
                   idle_gap_ms=idle_gaps,
                   store_mib=(u1 - u0) / 2 ** 20, lane_mib=(u2 - u1) / 2 ** 20, style_with_lanes_mib=store_and_lanes / 2 ** 20,
                   device=dev)
    print(json.dumps(summary), flush=True)
    v.close()
    other.close()
    del p
    gc.collect()
    return rows, summary


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="sd15,turbo")
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--rank", type=int, default=64)
    args = ap.parse_args(argv)
    os.environ["NVENC"] = "1"
    os.environ.pop("B200SD_LANES", None)
    dev = card()
    tmp = tempfile.mkdtemp(prefix="b2sd-styles-")
    try:
        for name in args.models.split(","):
            bench_model(name, args, tmp, dev)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
