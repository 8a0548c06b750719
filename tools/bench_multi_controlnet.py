"""Cost of several ControlNets (DESIGN §4.13) on seeded synthetic full-size weights at 512x512, one JSON line per
measurement:

    python tools/bench_multi_controlnet.py [--frames 200] [--warmup 20]

  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) and SD-Turbo, T=1 ([32]);
  * nets: none, the frame (controlnet_processor_id=None), HED, and frame + HED (one HED pass shared);
  * fps: back-to-back frames on one CUDA stream (one synchronise at the end); p50 / p99: a second pass with a synchronise
    after every frame (tools/bench_controlnet_scale.py's rate);
  * launches_per_frame, and hbm_mb: device memory the engine holds after prepare (torch.cuda.mem_get_info before and after
    building it), from which the HBM per added net follows;
  * update_ms: host time of one global and one per-viewer ControlNet update, and of one prompt update, each ending in a device
    synchronise, median of 50.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_controlnet import card  # noqa: E402
from bench_controlnet_scale import rate, update_ms  # noqa: E402

NETS = {"none": [], "frame": [None], "hed": ["hed"], "frame+hed": [None, "hed"]}


def build(model, t_index_list, procs, hw=512):
    """The engine with one synthetic ControlNet per entry of procs (net i seeded by its position) and the device memory it
    took"""
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
    if len(procs) == 1:
        kw = dict(controlnet_sd=W.synthetic_controlnet(arch), hed_sd=A.synthetic_hed() if procs[0] == "hed" else None)
    elif procs:
        kw = dict(controlnet_sd=[W.synthetic_controlnet(arch, seed=5678 + i) for i in range(len(procs))],
                  control_processors=procs, hed_sd=A.synthetic_hed() if "hed" in procs else None)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, **kw)
    sd.prepare("bench", guidance_scale=0.0)
    torch.cuda.synchronize()
    hbm = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
    frame = torch.randint(0, 256, (1, hw, hw, 3), dtype=torch.uint8, generator=g).cuda()
    return sd, frame, round(hbm, 1)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_controlnet: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl in (("lykon/dreamshaper-8", [18, 26, 35, 45]), ("stabilityai/sd-turbo", [32])):
        for name, procs in NETS.items():
            sd, frame, hbm = build(model, tl, procs)
            if len(procs) > 1:
                sd.set_control_scale([0.8, 0.6], [0.0, 0.2], 1.0)
            fps, p50, p99 = rate(sd, frame, args.frames, args.warmup)
            r = {"model": sd.arch.name, "t_index_list": tl, "size": 512, "nets": name, "fps": fps, "p50_ms": p50,
                 "p99_ms": p99, "launches_per_frame": sd.launches_per_step, "hbm_mb": hbm}
            st = sd.new_state()
            if procs:
                one = 0.5 if len(procs) == 1 else [0.5, 0.7]
                other = 0.6 if len(procs) == 1 else [0.6, 0.7]
                r["global_update_ms"] = update_ms(lambda i: sd.set_control_scale(one if i % 2 else other))
                r["viewer_update_ms"] = update_ms(lambda i: st.set_control_scale(one if i % 2 else other))
            r["prompt_update_ms"] = update_ms(lambda i: sd.update_prompt(f"bench {i % 2}"))
            r.update(info)
            print(json.dumps(r), flush=True)
            st.close()
            del sd, st
            torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
