"""Frames/s, latency, FLOPs, VAE device time and HBM per lane with TAESD (use_tiny_vae=True) and with the model's own
AutoencoderKL (use_tiny_vae=False), on seeded synthetic full-size weights.  One JSON line per configuration:

    python tools/bench_vae.py [--frames 100] [--warmup 10]

  * SD-Turbo, T=1 ([32]) at 512x512;
  * SD-1.5 + LCM, T=4 ([18, 26, 35, 45]) at 512x512.

fps: back-to-back frames on one CUDA stream (one synchronise at the end).  p50/p99: a second pass with a synchronise after
every frame.  vae_gflop_per_frame: the AutoencoderKL's encoder / decoder convolutions and attention counted from layer shapes
by this script (2 x MACs; 0 for TAESD, whose cost is in the engine's count).  engine_gflop_per_frame: the contractions of the
frame program as the engine counts them.  encoder_ms / decoder_ms: device time of the encoder's and the decoder's launches,
from an eager replay with an event after every launch (b2sd_profile).  hbm_per_lane_mb: device memory a further lane of the
engine takes (activations and per-program buffers; the bump allocator does not reuse memory).  The card's name and power limit
are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_controlnet import card  # noqa: E402


def _conv(h, w, ci, co, k=3):
    return 2.0 * h * w * ci * co * k * k


def _resnet(h, w, ci, co):
    return _conv(h, w, ci, co) + _conv(h, w, co, co) + (_conv(h, w, ci, co, 1) if ci != co else 0.0)


def _mid(h, w, c):
    n = h * w
    return 2 * _resnet(h, w, c, c) + 4 * 2.0 * n * c * c + 2 * 2.0 * n * n * c


def kl_gflop(height: int, width: int, ch=(128, 256, 512, 512)):
    """(encoder, decoder) GFLOP of diffusers' AutoencoderKL at this image size."""
    h, w = height, width
    enc = _conv(h, w, 3, ch[0])
    ci = ch[0]
    for i, co in enumerate(ch):
        enc += _resnet(h, w, ci, co) + _resnet(h, w, co, co)
        ci = co
        if i < len(ch) - 1:
            h, w = h // 2, w // 2
            enc += _conv(h, w, co, co)
    enc += _mid(h, w, ci) + _conv(h, w, ci, 8) + _conv(h, w, 8, 8, 1)
    dec = _conv(h, w, 4, 4, 1) + _conv(h, w, 4, ch[-1]) + _mid(h, w, ch[-1])
    ci = ch[-1]
    for i, co in enumerate(reversed(ch)):
        dec += _resnet(h, w, ci, co) + 2 * _resnet(h, w, co, co)
        ci = co
        if i < len(ch) - 1:
            h, w = h * 2, w * 2
            dec += _conv(h, w, co, co)
    dec += _conv(h, w, ci, 3)
    return enc / 1e9, dec / 1e9


def run(model: str, t_index_list, tiny_vae: bool, frames: int, warmup: int, hw: int = 512) -> dict:
    import torch
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    arch = A.arch_for(model)
    usd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
    vsd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True) if tiny_vae else A.synthetic_autoencoder_kl()
    g = torch.Generator().manual_seed(1)
    emb = torch.randn((1, 77, arch.cross_attention_dim), generator=g).half()
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, use_tiny_vae=tiny_vae)
    sd.prepare("bench", guidance_scale=0.0)
    del usd, vsd
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
    ops = sd.profile(frame, iters=5)
    names = [o["name"] for o in ops]
    step = names.index("lcm_step")
    enc_ms = ops[0]["ms"] + sum(o["ms"] for o in ops[1:step] if "vae.encoder" in o["name"])
    dec_ms = sum(o["ms"] for o in ops[step + 1:])
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    lane = sd.add_lane()
    torch.cuda.synchronize()
    lane_mb = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20
    del lane
    enc_g, dec_g = (0.0, 0.0) if tiny_vae else kl_gflop(hw, hw)
    return {"model": arch.name, "t_index_list": list(t_index_list), "size": hw, "vae": "taesd" if tiny_vae else "autoencoder_kl",
            "fps": round(fps, 2), "p50_ms": round(lat[len(lat) // 2], 3), "p99_ms": round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3),
            "vae_gflop_per_frame": {"encoder": round(enc_g, 1), "decoder": round(dec_g, 1)},
            "engine_gflop_per_frame": round(flops / 1e9, 1), "encoder_ms": round(enc_ms, 3), "decoder_ms": round(dec_ms, 3),
            "hbm_per_lane_mb": round(lane_mb, 1), "launches_per_frame": sd.launches_per_step}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vae: no CUDA device (the engine has no CPU path)")
    info = card()
    for model, tl in (("stabilityai/sd-turbo", [32]), ("lykon/dreamshaper-8", [18, 26, 35, 45])):
        for tiny in (True, False):
            r = run(model, tl, tiny, args.frames, args.warmup)
            r.update(info)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
