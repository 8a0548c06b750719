"""Weight-pack CLI: the replacement of the reference's `build.py` (build.py:11-32), which instantiates the wrapper once so
that the TensorRT engines end up in the cache directory.  Here the artefact is the packed-weight blob:

    python -m ai_rtc_agent_b200.pack --model-id lykon/dreamshaper-8 --lora /models/ghibli.safetensors:1.0
    python -m ai_rtc_agent_b200.pack --model-id stabilityai/sd-turbo --engine-dir ./models/engines

loads the diffusers-layout checkpoint from disk (or seeded synthetic weights with B200SD_SYNTHETIC_WEIGHTS=1), fuses the
LCM-LoRA (non-turbo models) and the given LoRAs into the UNet (lib/wrapper.py:683-697), lets the engine lay the weights out
in its kernel-native formats and writes `<engine-dir>/engines--<model>/b2sd-<arch>-<hash>.b2pack`.  Every later
StreamDiffusionWrapper / StreamDiffusionPipeline start with the same model + LoRA recipe loads that blob instead of the
checkpoint (no safetensors parsing, no LoRA fusing, no repacking, no raw copy in HBM).  Needs an H100 (packing runs on it)."""
from __future__ import annotations

import argparse
import logging
import os
import sys
import time


def parse_lora(specs):
    out = {}
    for spec in specs or []:
        path, sep, scale = spec.rpartition(":")
        if not sep:
            path, scale = spec, "1.0"
        try:
            out[path] = float(scale)
        except ValueError:
            raise SystemExit(f"--lora expects PATH[:SCALE], got {spec!r}")
    return out


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m ai_rtc_agent_b200.pack", description=__doc__.split("\n\n")[0])
    ap.add_argument("--model-id", default="lykon/dreamshaper-8", help="HF id (looked up under $HF_HUB_CACHE) or a local directory (agent.py:443)")
    ap.add_argument("--lora", action="append", metavar="PATH[:SCALE]", help="LoRA safetensors to fuse (repeatable; build.py:23-25)")
    ap.add_argument("--lcm-lora-id", default=None)
    ap.add_argument("--no-lcm-lora", action="store_true")
    ap.add_argument("--vae-id", default=None, help="TAESD to pack (ignored with --full-vae)")
    ap.add_argument("--full-vae", action="store_true", help="pack the model's own AutoencoderKL instead of TAESD (use_tiny_vae=False)")
    ap.add_argument("--controlnet-id", default=None, help="diffusers ControlNetModel (HF id or local directory) packed with the UNet")
    ap.add_argument("--controlnet-processor-id", default="hed", type=lambda v: None if v.lower() == "none" else v,
                    help="control-image preprocessor: hed (default, the reference's) or none (the frame itself)")
    ap.add_argument("--engine-dir", default=os.getenv("TRT_ENGINES_CACHE", "./models/engines"), help="cache root (lib/pipeline.py:35)")
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--t-index-list", type=int, nargs="+", default=None)
    ap.add_argument("--force", action="store_true", help="rebuild even if the blob exists")
    return ap


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")

    from .host import arch as A
    from .host import weights as W
    from .host.wrapper import StreamDiffusionWrapper
    turbo = "turbo" in args.model_id
    t_index_list = args.t_index_list or ([32] if turbo else [18, 26, 35, 45])
    loras = parse_lora(args.lora)
    repo = W.find_local_repo(args.model_id)
    have_ckpt = repo is not None and os.path.isdir(os.path.join(repo, "unet"))
    blob = W.packed_blob_path(args.engine_dir, args.model_id, A.arch_for(args.model_id).name, not args.no_lcm_lora and not turbo,
                              args.lcm_lora_id, loras, args.vae_id, synthetic=not have_ckpt,
                              variant=W.layout_variant(len(t_index_list), args.height, args.width), controlnet=args.controlnet_id,
                              control_processor=args.controlnet_processor_id, full_vae=args.full_vae)
    if not have_ckpt:
        if not (os.getenv(W.ALLOW_SYNTHETIC_ENV) or args.model_id.startswith(("tiny", "synthetic"))):
            raise SystemExit(f"pack: no checkpoint for '{args.model_id}' on disk (set {W.ALLOW_SYNTHETIC_ENV}=1 to pack seeded synthetic weights)")
        os.environ["B200SD_PACK_CACHE"] = "synthetic"
    if args.force and os.path.exists(blob):
        os.remove(blob)
    t0 = time.time()
    w = StreamDiffusionWrapper(model_id_or_path=args.model_id, t_index_list=t_index_list, lora_dict=loras or None,
                               lcm_lora_id=args.lcm_lora_id, vae_id=None if args.full_vae else args.vae_id,
                               use_lcm_lora=not args.no_lcm_lora, use_tiny_vae=not args.full_vae,
                               controlnet_id_or_path=args.controlnet_id, controlnet_processor_id=args.controlnet_processor_id,
                               width=args.width, height=args.height, output_type="pt", mode="img2img", engine_dir=args.engine_dir)
    reused = w.packed_blob is not None
    w.prepare(prompt="", num_inference_steps=50, guidance_scale=0.0)
    if w.packed_blob is None:
        print(f"pack: the blob could not be written under {args.engine_dir}", file=sys.stderr)
        return 1
    print(f"{'reused' if reused else 'wrote'} {w.packed_blob} ({os.path.getsize(w.packed_blob) / 1e6:.1f} MB) in {time.time() - t0:.1f} s")
    return 0


if __name__ == "__main__":
    sys.exit(main())
