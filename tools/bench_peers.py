"""Several viewers on one pipeline: per-peer temporal streams (StreamDiffusionPipeline(per_peer_streams=True), one PeerStream
per viewer) against the shared mode with one viewer, on seeded synthetic full-size weights at 512x512.  One JSON line per
measurement, then one summary line per model:

    python tools/bench_peers.py [--frames 200] [--warmup 10] [--repeats 3] [--peers 1,2,4,8] [--lanes 2,3,4]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]);
  * SD-Turbo, T=1 ([32]).

Each measurement submits `frames` device-resident frames round-robin over the peers through the public non-blocking entry,
with as many frames pending as the pipeline has lanes (the next frame is submitted when the oldest has been retired).
fps: frames over the wall time of the loop.  p50 / p99: submit -> result on the host, per peer; the worst peer is reported.
hbm_per_peer_kb: device memory the peers' streams take (cudaMemGetInfo around opening them), per peer; state_kb: the state's
payload, (T-1) * 64 * 64 * 4 fp16 values.  The shared mode with one peer and the per-peer mode with one peer are measured
alternately, `repeats` times each, so that their spread is measured in the same run.  `lanes` (T > 1 only) lists the lane
counts of the per-peer pool to measure; the default lane count for T = 1 is the shared mode's.  The card's name and power
limit are read in the same run.

With --conditioning same,distinct,changing only the per-peer pool with the default lane count (or the first of --lanes) is
measured, at every peer count of --peers from 2 on, the modes alternately, `repeats` times each:
  * same: every viewer has the pipeline's prompt and t_index_list (no conditioning copies);
  * distinct: every viewer has its own prompt (PeerStream.update_prompt) and, at T > 1, its own t_index_list;
  * changing: as distinct, and viewer 0 changes its prompt every 10 of its frames; update_ms: host time of those calls
    (synthetic prompt encoder)."""
from __future__ import annotations

import argparse
import collections
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_controlnet import card  # noqa: E402

MODELS = (("lykon/dreamshaper-8", [18, 26, 35, 45]), ("stabilityai/sd-turbo", [32]))


def _pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def register_weights(model: str) -> None:
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    W.register_preloaded(model, arch, usd, vsd)


def build(model: str, tl, per_peer: bool, lanes, hw: int = 512):
    import torch
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    pipe = StreamDiffusionPipeline(model, t_index_list=tl, width=hw, height=hw, lanes=lanes, per_peer_streams=per_peer)
    torch.cuda.synchronize()
    return pipe, (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20


def measure(pipe, peers: int, frames, n: int, warmup: int, conditioning: str = "same") -> dict:
    """peers = 0: the pipeline's own stream (pipeline.enqueue); else that many PeerStreams, round-robin, with the
    conditioning mode of the module docstring"""
    import torch
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    targets = [pipe.open_stream() for _ in range(peers)] if peers else [pipe]
    if conditioning != "same":
        for k, t in enumerate(targets):
            t.update_prompt(f"viewer {k}")
            if len(pipe.t_index_list) > 1:
                t.update_t_index_list([v - 1 - k % 8 for v in pipe.t_index_list])
    update_ms = []
    torch.cuda.synchronize()
    hbm = (free0 - torch.cuda.mem_get_info()[0]) / max(1, peers) / 1024
    pending_max = pipe.lanes
    lat = collections.defaultdict(list)

    def loop(count, record):
        pend = collections.deque()

        def retire():
            p, t0, tk = pend.popleft()
            tk.result()
            if record:
                lat[p].append((time.perf_counter() - t0) * 1e3)
        for i in range(count):
            p = i % len(targets)
            if conditioning == "changing" and p == 0 and i % (10 * len(targets)) == 0:
                t1 = time.perf_counter()
                targets[0].update_prompt(f"viewer 0, frame {i}")
                if record:
                    update_ms.append((time.perf_counter() - t1) * 1e3)
            pend.append((p, time.perf_counter(), targets[p].enqueue(frames[i % len(frames)])))
            while len(pend) >= pending_max:
                retire()
        while pend:
            retire()

    loop(warmup * pending_max * len(targets), False)
    t0 = time.perf_counter()
    loop(n, True)
    wall = time.perf_counter() - t0
    if peers:
        for t in targets:
            t.close()
    out = {"fps": round(n / wall, 2), "p50_ms": round(max(statistics.median(v) for v in lat.values()), 3),
           "p99_ms": round(max(_pct(v, 0.99) for v in lat.values()), 3), "hbm_per_peer_kb": round(hbm, 1) if peers else None}
    if update_ms:
        out.update(update_ms_p50=round(statistics.median(update_ms), 3), update_ms_max=round(max(update_ms), 3))
    return out


def run_model(model: str, tl, args, info) -> dict:
    import torch
    register_weights(model)
    T = len(tl)
    g = torch.Generator().manual_seed(7)
    frames = [torch.randint(0, 256, (1, 512, 512, 3), dtype=torch.uint8, generator=g).cuda() for _ in range(16)]
    base = dict(model=model, t_index_list=tl, size=512, state_kb=round((T - 1) * 64 * 64 * 8 / 1024, 1), **info)
    rows = []

    def emit(row):
        row = {**base, **row}
        rows.append(row)
        print(json.dumps(row), flush=True)

    lane_counts = args.lanes if T > 1 else [None]
    if args.conditioning:
        from ai_rtc_agent_b200.host.pipeline import DEFAULT_LANES_STATEFUL
        pool, pool_mb = build(model, tl, True, (DEFAULT_LANES_STATEFUL if DEFAULT_LANES_STATEFUL in lane_counts else lane_counts[0])
                              if T > 1 else None)
        for p in (p for p in args.peers if p >= 2):
            for r in range(args.repeats):
                for mode in args.conditioning:
                    emit(dict(mode="per_peer", conditioning=mode, peers=p, lanes=pool.lanes, repeat=r, pool_mb=round(pool_mb),
                              **measure(pool, p, frames, args.frames, args.warmup, mode)))
        fps = collections.defaultdict(list)
        for r in rows:
            fps[(r["peers"], r["conditioning"])].append(r["fps"])
        summary = {**base, "summary": True, "lanes": pool.lanes,
                   "fps": {f"{p}:{m}": [min(v), max(v)] for (p, m), v in sorted(fps.items())}}
        print(json.dumps(summary), flush=True)
        del pool
        from ai_rtc_agent_b200.host import weights as W
        W._PRELOADED.pop(model, None)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return summary
    shared, shared_mb = build(model, tl, False, None)
    pools = {}
    for lanes in lane_counts:
        pools[lanes] = build(model, tl, True, lanes)
    from ai_rtc_agent_b200.host.pipeline import DEFAULT_LANES_STATEFUL
    default = pools.get(DEFAULT_LANES_STATEFUL if T > 1 else None, next(iter(pools.values())))[0]
    # one peer: shared mode and per-peer mode (default lanes) alternately
    for r in range(args.repeats):
        emit(dict(mode="shared", peers=1, lanes=shared.lanes, repeat=r, pool_mb=round(shared_mb), **measure(shared, 0, frames, args.frames, args.warmup)))
        emit(dict(mode="per_peer", peers=1, lanes=default.lanes, repeat=r, **measure(default, 1, frames, args.frames, args.warmup)))
    for lanes, (pool, pool_mb) in pools.items():
        for p in args.peers:
            emit(dict(mode="per_peer", peers=p, lanes=pool.lanes, pool_mb=round(pool_mb), **measure(pool, p, frames, args.frames, args.warmup)))
    sh = [r["fps"] for r in rows if r["mode"] == "shared"]
    pp = [r["fps"] for r in rows if r["mode"] == "per_peer" and r["peers"] == 1 and "repeat" in r]
    # one peer on the per-peer pool is no slower than the shared mode when its median is not below the shared mode's slowest run
    summary = {**base, "summary": True, "shared_1peer_fps": [min(sh), max(sh)], "per_peer_1peer_fps": [min(pp), max(pp)],
               "per_peer_1peer_median_fps": statistics.median(pp), "per_peer_1peer_within_shared_spread": statistics.median(pp) >= min(sh)}
    print(json.dumps(summary), flush=True)
    del shared, pools, default
    from ai_rtc_agent_b200.host import weights as W
    W._PRELOADED.pop(model, None)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return summary


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--peers", default="1,2,4,8")
    ap.add_argument("--lanes", default="2,3,4", help="per-peer lane counts to measure at T > 1")
    ap.add_argument("--models", default="all", choices=["all", "sd15", "turbo"])
    ap.add_argument("--conditioning", default="", help="compare these conditioning modes (same, distinct, changing) instead")
    args = ap.parse_args(argv)
    args.conditioning = [v for v in args.conditioning.split(",") if v]
    if any(v not in ("same", "distinct", "changing") for v in args.conditioning):
        ap.error("--conditioning takes same, distinct and changing")
    args.peers = [int(v) for v in args.peers.split(",")]
    args.lanes = [int(v) for v in args.lanes.split(",")]
    os.environ.setdefault("B200SD_SYNTHETIC_WEIGHTS", "1")
    os.environ["NVENC"] = "1"   # results stay on the device (the pipeline's NVENC branch)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_peers: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl in MODELS:
        if args.models == "all" or (args.models == "turbo") == ("turbo" in model):
            run_model(model, tl, args, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
