"""Switching style LoRAs on a running pipeline (StreamDiffusionPipeline(live_lora=True).update_lora) against building a new
pipeline with the LoRA, on seeded synthetic SD-1.5 weights (LCM-distilled topology) at 512x512, T = 4, 2 lanes:

    python tools/bench_lora_switch.py [--rank 64] [--switches 10] [--frames 60]

The LoRA: rank `rank`, fp16 factors, on every attention projection (to_q / to_k / to_v / to_out.0), feed-forward
(ff.net.0.proj, ff.net.2) and 3x3 convolution of the UNet; two such LoRAs (different seeds) are switched alternately.
Reported, one JSON line each, then a summary line:
  * update_host_ms: wall time of update_lora (reading the files, checking the pairs, uploading the factors, enqueueing);
  * first_frame_ms: from the start of update_lora until the first frame enqueued after it has completed;
  * update_stream_ms: CUDA events on the update's stream around update_lora on an idle device: the host's work inside the call
    (the device waits for it) plus the update's launches;
  * update_device_ms: device time of the update's launches and copies (re-fusing, repacking, conditioning), summed from a
    torch.profiler trace of one switch taken in a run of its own;
  * p99 / p50 of a viewer's frames (submit -> result, 2 frames pending) in a run that switches every 20 frames, and in the
    same run without switches;
  * live_extra_mib: device memory of the live-mode pipeline minus the default-mode pipeline's (cudaMemGetInfo);
  * rebuild_s: building a new default-mode pipeline with the LoRA fused on the host (fuse + engine + prepare + lanes).
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

MODEL, TL = "lykon/dreamshaper-8", [18, 26, 35, 45]


def _pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def write_lora(path, usd, rank, seed):
    import torch
    from safetensors.torch import save_file
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, w in usd.items():
        attn = any(t in k for t in (".to_q.", ".to_k.", ".to_v.", ".to_out.0.", "ff.net.0.proj.", "ff.net.2."))
        if not k.endswith(".weight") or not (attn or (w.dim() == 4 and w.shape[2] == 3)):
            continue
        rows, cols = w.shape[0], w[0].numel()
        down = torch.randn(rank, cols, generator=g) / cols ** 0.5
        up = torch.randn(rows, rank, generator=g) * (0.1 * float(w.float().std()) / rank ** 0.5)
        if w.dim() == 4:
            down, up = down.reshape(rank, *w.shape[1:]), up.reshape(rows, rank, 1, 1)
        m = k[: -len(".weight")]
        sd[f"unet.{m}.lora_A.weight"] = down.half().contiguous()
        sd[f"unet.{m}.lora_B.weight"] = up.half().contiguous()
    save_file(sd, path)
    return len(sd) // 2


def pipeline(usd, vsd, live):
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    W.register_preloaded(MODEL, A.arch_for(MODEL), usd, vsd)
    try:
        p = StreamDiffusionPipeline(MODEL, t_index_list=TL, width=512, height=512, lanes=2, live_lora=live)
    finally:
        W._PRELOADED.pop(MODEL, None)
    torch.cuda.synchronize()
    return p


def viewer_run(p, frames, n, switch_every=0, loras=()):
    """submit -> result times of n frames with 2 pending; update_lora every `switch_every` frames"""
    lat, pending, k = [], [], 0
    for i in range(n):
        if switch_every and i and i % switch_every == 0:
            p.update_lora(loras[k % len(loras)])
            k += 1
        pending.append((time.perf_counter(), p.enqueue(frames[i % len(frames)])))
        if len(pending) == 2:
            t0, tk = pending.pop(0)
            tk.result()
            lat.append((time.perf_counter() - t0) * 1e3)
    for t0, tk in pending:
        tk.result()
        lat.append((time.perf_counter() - t0) * 1e3)
    return lat


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, default=64)
    ap.add_argument("--switches", type=int, default=10)
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args(argv)
    import torch
    os.environ["NVENC"] = "1"
    os.environ.pop("B200SD_LANES", None)
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.weights import fuse_lora, load_lora_file
    from oracle import weights as ow
    dev = card()
    arch = A.arch_for(MODEL)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    tmp = tempfile.mkdtemp(prefix="b2sd-lora-")
    la, lb = os.path.join(tmp, "a.safetensors"), os.path.join(tmp, "b.safetensors")
    modules = write_lora(la, usd, args.rank, 1)
    write_lora(lb, usd, args.rank, 2)
    A_, B_ = {la: 1.0}, {lb: 1.0}
    frames = [ow.make_frame(512, 512, seed=i).cuda() for i in range(8)]

    def used():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[1] - torch.cuda.mem_get_info()[0]

    u0 = used()
    plain = pipeline(usd, vsd, False)
    u_plain = used() - u0
    del plain
    u0 = used()
    p = pipeline(usd, vsd, True)
    p.update_lora(A_)
    viewer_run(p, frames, 8)
    u_live = used() - u0
    # switches on an idle device: host time, stream time, time to the first frame after the switch
    host, device, first = [], [], []
    for k in range(args.switches):
        torch.cuda.synchronize()
        cur = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(cur)
        p.update_lora(B_ if k % 2 == 0 else A_)
        e1.record(cur)
        t1 = time.perf_counter()
        p.enqueue(frames[k % 8]).result()
        t2 = time.perf_counter()
        e1.synchronize()
        host.append((t1 - t0) * 1e3)
        first.append((t2 - t0) * 1e3)
        device.append(e0.elapsed_time(e1))
    # the launches alone: a profiled switch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.update_lora(B_)
        torch.cuda.synchronize()
    launches_ms = sum(getattr(e, "device_time_total", 0.0) for e in prof.events() if e.device_type == DeviceType.CUDA) / 1e3
    kernels = sum(1 for e in prof.events() if e.device_type == DeviceType.CUDA)
    p.update_lora(A_)
    steady = viewer_run(p, frames, args.frames)
    switching = viewer_run(p, frames, args.frames, switch_every=20, loras=(B_, A_))
    del p
    # the alternative: a new pipeline with the LoRA fused on the host
    gc.collect()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fused = dict(usd)
    fuse_lora(fused, load_lora_file(la), 1.0)
    q = pipeline(fused, vsd, False)
    rebuild_s = time.perf_counter() - t0
    del q
    shutil.rmtree(tmp, ignore_errors=True)
    rows = [dict(metric="update_host_ms", values=host), dict(metric="first_frame_ms", values=first),
            dict(metric="update_stream_ms", values=device),
            dict(metric="update_device_ms", value=launches_ms, device_ops=kernels),
            dict(metric="viewer_latency_ms", switching_p50=_pct(switching, 0.5), switching_p99=_pct(switching, 0.99),
                 steady_p50=_pct(steady, 0.5), steady_p99=_pct(steady, 0.99)),
            dict(metric="live_extra_mib", value=(u_live - u_plain) / 2 ** 20, live_mib=u_live / 2 ** 20, plain_mib=u_plain / 2 ** 20),
            dict(metric="rebuild_s", value=rebuild_s)]
    for r in rows:
        print(json.dumps(dict(r, device=dev)))
    med = lambda xs: sorted(xs)[len(xs) // 2]   # noqa: E731
    print(json.dumps(dict(summary=True, model=MODEL, size=512, T=len(TL), lanes=2, rank=args.rank, lora_modules=modules,
                          update_host_ms=med(host), update_stream_ms=med(device), update_device_ms=launches_ms,
                          first_frame_ms=med(first),
                          p99_switching_ms=_pct(switching, 0.99), p99_steady_ms=_pct(steady, 0.99),
                          live_extra_mib=(u_live - u_plain) / 2 ** 20, rebuild_s=rebuild_s, device=dev)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
