"""What IP-Adapter image prompts cost, on seeded synthetic full-size weights and a synthetic adapter.  One JSON line per
configuration:

    python tools/bench_ip_adapter.py [--frames 200] [--warmup 20]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) at 512x512, and SD-Turbo, T=1 ([32]) at 512x512;
  * each as a plain engine, an adapter engine without an image prompt and the same engine with one (4 image tokens, scale 0.8).

fps: back-to-back frames on one CUDA stream (one synchronise at the end).  p50/p99: a second pass with a synchronise after
every frame.  attn_ms: device time of every attention launch of the frame (b2sd_profile_kind("attn"): a CUDA graph of only
those launches), so attn_ms with an image prompt minus attn_ms without one is the cost of the image segment of the 16 UNet
cross-attentions.  update_ms: host time of one image-prompt update, split into the image encoder + projection (here the
seeded synthetic encoder: a real CLIP ViT-H runs in torch and is not measured) and the conditioning refresh (every UNet
cross-attention's image K / V^T on every engine), each ended by a device synchronise, median of 20.  extra_hbm_mib: device
memory the adapter engine holds beyond the plain one (cudaMemGetInfo around building and preparing each).
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


def _engine(arch, t_index_list, hw, adapter):
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
    g = torch.Generator().manual_seed(1)
    emb = torch.randn((1, 77, arch.cross_attention_dim), generator=g).half()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, ip_adapter=adapter)
    sd.prepare("bench", guidance_scale=0.0)
    torch.cuda.synchronize()
    return sd, free0 - torch.cuda.mem_get_info()[0]


def _time(sd, frames, warmup, hw):
    import torch
    g = torch.Generator().manual_seed(2)
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
    return {"fps": round(fps, 2), "p50_ms": round(lat[len(lat) // 2], 3),
            "p99_ms": round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3),
            "attn_ms": round(sd.profile_kind("attn", iters=50)["ms"], 4), "launches_per_frame": sd.launches_per_step}


def run(model, t_index_list, frames, warmup, hw=512):
    import numpy as np
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import image_prompt as I
    arch = A.arch_for(model)
    rows = []
    plain, plain_bytes = _engine(arch, t_index_list, hw, None)
    rows.append(dict(engine="plain", **_time(plain, frames, warmup, hw)))
    del plain
    torch.cuda.empty_cache()
    adapter = I.adapter_from_state_dict(I.synthetic_adapter_state_dict(arch), arch)
    sd, ip_bytes = _engine(arch, t_index_list, hw, adapter)
    rows.append(dict(engine="adapter, no image prompt", **_time(sd, frames, warmup, hw)))
    images = [np.random.default_rng(k).integers(0, 256, (224, 224, 3), dtype=np.uint8) for k in range(20)]
    enc_ms, refresh_ms = [], []
    for img in images:
        t0 = time.perf_counter()
        tok = sd.image_tokens(img)
        t1 = time.perf_counter()
        sd.set_image_tokens(tok, 0.8)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        enc_ms.append((t1 - t0) * 1e3)
        refresh_ms.append((t2 - t1) * 1e3)
    rows.append(dict(engine="adapter, image prompt", **_time(sd, frames, warmup, hw)))
    for r in rows:
        r.update(model=arch.name, t_index_list=list(t_index_list), size=hw)
    rows[-1].update(update_encoder_ms=round(statistics.median(enc_ms), 3),
                    update_refresh_ms=round(statistics.median(refresh_ms), 3),
                    extra_hbm_mib=round((ip_bytes - plain_bytes) / 2 ** 20, 1))
    return rows


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ip_adapter: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl in (("lykon/dreamshaper-8", [18, 26, 35, 45]), ("stabilityai/sd-turbo", [32])):
        for r in run(model, tl, args.frames, args.warmup):
            r.update(info)
            print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
