"""Checkpoint plumbing that replaces the reference's TensorRT build (build.py:11-32,
lib/wrapper.py:617-910): locate diffusers-format safetensors on disk, fuse LoRAs into the base weights
(lib/wrapper.py:683-697), or fall back to seeded synthetic weights when explicitly allowed."""
from __future__ import annotations

import glob
import logging
import math
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import arch as A

logger = logging.getLogger(__name__)
ALLOW_SYNTHETIC_ENV = "B200SD_SYNTHETIC_WEIGHTS"


_PRELOADED: Dict[str, tuple] = {}


def register_preloaded(model_id: str, arch, unet_sd, vae_sd) -> None:
    """Make already-materialised weights (e.g. received by NCCL broadcast, host/dist.py) the ones
    `resolve_weights(model_id, ...)` returns on this process."""
    _PRELOADED[model_id] = (arch, unet_sd, vae_sd)


def find_local_repo(model_id_or_path: str) -> Optional[str]:
    """A directory path, or a HF-cache snapshot of `org/name` under $HF_HUB_CACHE (lib/wrapper.py:437)."""
    if os.path.isdir(model_id_or_path):
        return model_id_or_path
    cache = os.getenv("HF_HUB_CACHE") or os.path.join(os.getenv("HF_HOME", os.path.expanduser("~/.cache/huggingface")), "hub")
    snaps = sorted(glob.glob(os.path.join(cache, "models--" + model_id_or_path.replace("/", "--"), "snapshots", "*")))
    return snaps[-1] if snaps else None


def _load_safetensors(path: str) -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file
    return load_file(path)


def load_unet(repo_dir: str) -> Dict[str, torch.Tensor]:
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
        p = os.path.join(repo_dir, "unet", name)
        if os.path.exists(p):
            return {k: v.to(torch.float16) for k, v in _load_safetensors(p).items()}
    raise FileNotFoundError(f"no UNet safetensors under {repo_dir}/unet")


def load_taesd(repo_dir: str) -> Dict[str, torch.Tensor]:
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
        p = os.path.join(repo_dir, name)
        if os.path.exists(p):
            return {k: v.to(torch.float16) for k, v in _load_safetensors(p).items()}
    raise FileNotFoundError(f"no TAESD safetensors under {repo_dir}")


DEFAULT_VAE_SCALING_FACTOR = 0.18215


def load_autoencoder_kl(repo_dir: str, v: A.VaeArch = A.AUTOENCODER_KL) -> Dict[str, torch.Tensor]:
    """The model's own VAE: `<repo>/vae/diffusion_pytorch_model{.fp16,}.safetensors`, legacy attention names accepted, checked
    key by key against the AutoencoderKL inventory (its scaling factor: resolve_vae_scaling_factor)."""
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
        p = os.path.join(repo_dir, "vae", name)
        if os.path.exists(p):
            sd = A.normalize_autoencoder_kl({k: v.to(torch.float16) for k, v in _load_safetensors(p).items()})
            A.validate_exact(sd, A.autoencoder_kl_param_shapes(v), "AutoencoderKL checkpoint")
            return sd
    raise FileNotFoundError(f"no AutoencoderKL safetensors under {repo_dir}/vae")


def load_controlnet(repo_dir: str, arch: A.UNetArch) -> Dict[str, torch.Tensor]:
    """A diffusers ControlNetModel directory (config.json + diffusion_pytorch_model{.fp16,}.safetensors), checked against the
    UNet architecture it will be attached to."""
    import json
    cfg_path = os.path.join(repo_dir, "config.json")
    if os.path.exists(cfg_path):
        with open(cfg_path) as f:
            cfg = json.load(f)
        want = {"block_out_channels": list(arch.block_out_channels), "cross_attention_dim": arch.cross_attention_dim,
                "layers_per_block": arch.layers_per_block,
                "conditioning_embedding_out_channels": list(A.CN_EMBED_CHANNELS)}
        for key, val in want.items():
            if key in cfg and cfg[key] != val:
                raise ValueError(f"ControlNet {repo_dir}: {key} = {cfg[key]}, the {arch.name} UNet needs {val}")
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
        p = os.path.join(repo_dir, name)
        if os.path.exists(p):
            sd = {k: v.to(torch.float16) for k, v in _load_safetensors(p).items()}
            A.validate_state_dict(sd, A.controlnet_param_shapes(arch), "ControlNet checkpoint")
            return sd
    raise FileNotFoundError(f"no ControlNet safetensors under {repo_dir}")


def synthetic_controlnet(arch: A.UNetArch, seed: int = 5678, zero_init: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded ControlNet weights.  zero_init=True: the zero convs and the conditioning embedding's conv_out are zero, as in a
    ControlNet freshly initialised from a UNet (its residuals are then exactly zero)."""
    sd = A.synthetic_state_dict(A.controlnet_param_shapes(arch), seed=seed)
    if zero_init:
        for k in sd:
            if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.", "controlnet_cond_embedding.conv_out.")):
                sd[k] = torch.zeros_like(sd[k])
    return sd


def resolve_controlnet(controlnet_id_or_path: str, arch: A.UNetArch, synthetic_ok: bool, net: int = 0) -> Dict[str, torch.Tensor]:
    """A ControlNet on disk (directory or HF-cache id), else seeded synthetic weights when those are allowed, else an error.
    net: its position among several ControlNets; synthetic weights are seeded by it (net 0 with the single net's seed), so
    that two synthetic nets differ."""
    repo = find_local_repo(controlnet_id_or_path)
    if repo is not None:
        return load_controlnet(repo, arch)
    if synthetic_ok:
        logger.warning("no ControlNet %s on disk: using seeded synthetic weights", controlnet_id_or_path)
        return synthetic_controlnet(arch, seed=5678 + net)
    raise FileNotFoundError(f"ControlNet '{controlnet_id_or_path}' not found on disk; set {ALLOW_SYNTHETIC_ENV}=1 to run with "
                            "seeded synthetic weights")


ANNOTATORS_ID = "lllyasviel/Annotators"


def load_hed(path: str) -> Dict[str, torch.Tensor]:
    """ControlNetHED.pth (a plain state dict, loaded without unpickling code), checked against the HED inventory."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k: v.float() for k, v in sd.items()}
    A.validate_state_dict(sd, A.hed_param_shapes(), "HED checkpoint")
    return sd


def resolve_hed(synthetic_ok: bool) -> Dict[str, torch.Tensor]:
    """ControlNetHED.pth from a local lllyasviel/Annotators snapshot, else seeded synthetic weights when allowed, else an error."""
    repo = find_local_repo(ANNOTATORS_ID)
    if repo is not None and os.path.exists(os.path.join(repo, "ControlNetHED.pth")):
        return load_hed(os.path.join(repo, "ControlNetHED.pth"))
    if synthetic_ok:
        logger.warning("no %s/ControlNetHED.pth on disk: using seeded synthetic HED weights", ANNOTATORS_ID)
        return A.synthetic_hed()
    raise FileNotFoundError(f"{ANNOTATORS_ID}/ControlNetHED.pth not found on disk; set {ALLOW_SYNTHETIC_ENV}=1 to run with seeded "
                            "synthetic weights")


def resolve_lora(unet_keys, lora_sd: Dict[str, torch.Tensor], strict: bool = True
                 ) -> List[Tuple[str, torch.Tensor, torch.Tensor, float, int]]:
    """The UNet parameters a LoRA state dict names: [(parameter key, up, down, alpha, rank)] in the state dict's order, for the
    diffusers/peft key styles `...to_q.lora_A.weight` / `lora.down.weight` and kohya `lora_unet_*` + `.alpha` (LoCon 3x3
    downs included).  unet_keys: the UNet's parameter names.  strict (default): every UNet LoRA pair must land on a parameter,
    and at least one must, otherwise KeyError; text-encoder pairs are skipped."""
    pairs: Dict[str, Dict[str, torch.Tensor]] = {}
    for k, v in lora_sd.items():
        base = None
        for down_tag, up_tag in ((".lora_A.weight", ".lora_B.weight"), (".lora.down.weight", ".lora.up.weight"),
                                 (".lora_down.weight", ".lora_up.weight")):
            if k.endswith(down_tag):
                base, role = k[: -len(down_tag)], "down"
            elif k.endswith(up_tag):
                base, role = k[: -len(up_tag)], "up"
            else:
                continue
            break
        if base is None:
            if k.endswith(".alpha"):
                pairs.setdefault(k[: -len(".alpha")], {})["alpha"] = v
            continue
        pairs.setdefault(base, {})[role] = v
    keys = list(unet_keys)
    index = {k[: -len(".weight")].replace(".", "_"): k for k in keys if k.endswith(".weight")}
    keys = set(keys)
    found = []
    unmatched = []
    for base, d in pairs.items():
        if "up" not in d or "down" not in d:
            continue
        name = base
        for prefix in ("unet.", "lora_unet_", "base_model.model."):
            if name.startswith(prefix):
                name = name[len(prefix):]
        name = name.replace(".processor", "").replace("to_out_lora", "to_out.0").replace("_lora", "")
        key = name + ".weight" if (name + ".weight") in keys else index.get(name.replace(".", "_"))
        if key is None:
            if not base.startswith(("lora_te_", "text_encoder.", "lora_te1_", "lora_te2_")):   # text-encoder LoRA: not on this path
                unmatched.append(base)
            continue
        rank = d["down"].shape[0]
        alpha = float(d["alpha"]) if "alpha" in d else float(rank)
        found.append((key, d["up"], d["down"], alpha, rank))
    if strict and (not found or unmatched):
        # a LoRA that silently does not apply leaves e.g. SD-1.5 un-distilled while it is run at 4 steps
        raise KeyError(f"LoRA fusing matched {len(found)} of {len(found) + len(unmatched)} UNet modules; unmatched (first 5): "
                       f"{unmatched[:5]}")
    return found


def fuse_lora(unet_sd: Dict[str, torch.Tensor], lora_sd: Dict[str, torch.Tensor], scale: float = 1.0, strict: bool = True) -> int:
    """W += scale * (alpha / rank) * up @ down for every UNet module the LoRA names (resolve_lora's key styles).  Returns the
    number of fused layers.  This is the weight-prep step the reference performs with pipe.fuse_lora() before building
    engines.  strict (default): every UNet LoRA pair must land on a parameter, otherwise KeyError."""
    found = resolve_lora(unet_sd.keys(), lora_sd, strict)
    for key, up, down, alpha, rank in found:
        delta = (up.float().flatten(1) @ down.float().flatten(1)) * (scale * alpha / rank)
        w = unet_sd[key]
        unet_sd[key] = (w.float() + delta.reshape(w.shape)).to(w.dtype)
    return len(found)


def load_lora_file(path: str) -> Dict[str, torch.Tensor]:
    """A LoRA file's state dict.  Only safetensors are read (never a pickle, which can run code): anything else is a
    ValueError."""
    if not str(path).endswith(".safetensors"):
        raise ValueError(f"LoRA {path}: only .safetensors files are read")
    try:
        return _load_safetensors(path)
    except FileNotFoundError:
        raise
    except Exception as exc:   # noqa: BLE001 - safetensors raises its own error type on a file that is not safetensors
        raise ValueError(f"LoRA {path}: not a safetensors file ({exc})") from exc


def lora_factors(unet_shapes: Dict[str, Tuple[int, ...]], lora_dict: Optional[Dict[str, float]]
                 ) -> List[Tuple[str, torch.Tensor, torch.Tensor, float]]:
    """What fusing `lora_dict` ({path: scale}, in order) on the base weights means, as factors for the engine's live re-fusing:
    [(parameter key, up [rows][rank], down [rank][cols], scale * alpha / rank)] with cols = the product of the parameter's
    other dimensions.  Reads every file and checks every pair (resolve_lora's strict rule, and each pair's shape against its
    parameter) before returning, so an error leaves nothing half applied."""
    out = []
    for path, scale in (lora_dict or {}).items():
        for key, up, down, alpha, rank in resolve_lora(unet_shapes.keys(), load_lora_file(path)):
            shape = tuple(unet_shapes[key])
            rows, cols = shape[0], math.prod(shape[1:])
            up2, down2 = up.flatten(1), down.flatten(1)
            if up2.shape[0] != rows or down2.shape[1] != cols or up2.shape[1] != down2.shape[0]:
                raise ValueError(f"LoRA {path}: the pair on {key} has up {tuple(up.shape)} / down {tuple(down.shape)}, which do not "
                                 f"fit the parameter's shape {shape}")
            out.append((key, up2, down2, scale * alpha / rank))
    return out


def layout_variant(batch: int, height: int, width: int) -> str:
    """The packed layouts are the same for every batch / resolution except one case: with a stream batch > 1, attention levels
    whose token count is not a multiple of 8 keep separate q/k and v matrices (per-image V^T padding) instead of the fused,
    LayerNorm-folded [q|k|v] -- a different set of packed tensors, hence a different blob."""
    if batch <= 1:
        return ""
    ragged = [i for i in range(4) if ((height // 8) >> i) * ((width // 8) >> i) % 8 != 0]
    return "ragged" + "".join(str(i) for i in ragged) if ragged else ""


def packed_blob_path(engine_dir, model_id_or_path: str, arch_name: str, use_lcm_lora: bool, lcm_lora_id: Optional[str],
                     lora_dict: Optional[Dict[str, float]], vae_id: Optional[str], synthetic: bool, variant: str = "",
                     controlnet=None, control_processor=None, full_vae: bool = False,
                  ip_adapter: Optional[str] = None) -> str:
    """Where the packed-weight blob of this model lives: `<engine_dir>/engines--<model>/b2sd-<arch>-<recipe hash>.b2pack`,
    the directory naming of the reference's TensorRT cache (lib/wrapper.py:593, `engines--` + model id with / -> --).
    The hash covers everything that changes the weight VALUES (LoRAs and their scales, LCM-LoRA, VAE, ControlNet, synthetic
    seed), not
    batch / resolution / prompt (the blob does not depend on them, unlike the reference's static-shape engines).
    full_vae (use_tiny_vae=False) enters the recipe only when set, so the names of TAESD blobs do not change; so does
    ip_adapter (an adapter file or directory, or "synthetic"), with the adapter file's real path, size and mtime.
    Several ControlNets: controlnet and control_processor are lists in net order, and the recipe holds them as lists."""
    import hashlib
    import json
    recipe = {"lcm": bool(use_lcm_lora), "lcm_id": lcm_lora_id, "vae": vae_id, "synthetic": bool(synthetic), "layout": variant,
              "loras": sorted((str(k), float(v)) for k, v in (lora_dict or {}).items())}
    for path, _ in recipe["loras"]:
        if os.path.exists(path):   # a replaced LoRA file must not hit the old blob
            st = os.stat(path)
            recipe.setdefault("lora_files", []).append((path, st.st_size, int(st.st_mtime)))
    if full_vae:
        recipe["vae_kind"] = "autoencoder_kl"
    if controlnet is not None:
        recipe["controlnet"] = controlnet
        recipe["control_processor"] = control_processor
        for i, cn in enumerate(controlnet if isinstance(controlnet, (list, tuple)) else [controlnet]):
            repo = find_local_repo(cn)
            for name in sorted(os.listdir(repo)) if repo else ():   # replaced ControlNet weights must not hit the old blob
                if name.endswith((".safetensors", ".json")):
                    st = os.stat(os.path.join(repo, name))
                    # net 0's entries as a single net's, later nets' tagged with their position
                    entry = (name, st.st_size, int(st.st_mtime)) if i == 0 else (i, name, st.st_size, int(st.st_mtime))
                    recipe.setdefault("controlnet_files", []).append(entry)
    if ip_adapter is not None:
        recipe["ip_adapter"] = ip_adapter
        if os.path.exists(ip_adapter):   # a replaced adapter file must not hit the old blob
            from .image_prompt import adapter_file
            f = os.path.realpath(adapter_file(ip_adapter))
            st = os.stat(f)
            recipe["ip_adapter_file"] = (f, st.st_size, int(st.st_mtime))
    digest = hashlib.sha256(json.dumps(recipe, sort_keys=True).encode()).hexdigest()[:16]
    name = "engines--" + model_id_or_path.strip("/").replace("/", "--")
    return os.path.join(str(engine_dir), name, f"b2sd-{arch_name}-{digest}.b2pack")


def resolve_vae_scaling_factor(repo_dir: Optional[str]) -> float:
    """AutoencoderKL scaling_factor of a checkpoint directory (vae/config.json), 0.18215 without one."""
    import json
    p = os.path.join(repo_dir, "vae", "config.json") if repo_dir else None
    if p and os.path.exists(p):
        with open(p) as f:
            return float(json.load(f).get("scaling_factor", DEFAULT_VAE_SCALING_FACTOR))
    return DEFAULT_VAE_SCALING_FACTOR


def resolve_weights(model_id_or_path: str, vae_id: Optional[str], lcm_lora_id: Optional[str], use_lcm_lora: bool,
                    lora_dict: Optional[Dict[str, float]], sd_turbo: bool, use_tiny_vae: bool = True
                    ) -> Tuple[A.UNetArch, Dict[str, torch.Tensor], Dict[str, torch.Tensor], Optional[str]]:
    """Returns (arch, unet_sd, vae_sd, repo_dir or None).  Order: real checkpoint on disk -> synthetic weights if
    $B200SD_SYNTHETIC_WEIGHTS is set (or the id starts with "tiny"/"synthetic") -> error.  use_tiny_vae=False: vae_sd is the
    model's own AutoencoderKL (scaling factor: resolve_vae_scaling_factor); vae_id applies to TAESD only, as in the reference."""
    if not use_tiny_vae and vae_id is not None:
        logger.warning("vae_id=%s is ignored with use_tiny_vae=False: the model's own AutoencoderKL is used", vae_id)
    if model_id_or_path in _PRELOADED:
        if not use_tiny_vae:
            raise NotImplementedError("preloaded weights carry TAESD only; use_tiny_vae=False loads the AutoencoderKL from disk")
        arch, unet_sd, vae_sd = _PRELOADED[model_id_or_path]
        return arch, unet_sd, vae_sd, find_local_repo(model_id_or_path)
    arch = A.arch_for(model_id_or_path)
    repo = find_local_repo(model_id_or_path)
    if repo is not None and os.path.isdir(os.path.join(repo, "unet")):
        unet_sd = load_unet(repo)
        if use_tiny_vae:
            vae_repo = find_local_repo(vae_id or "madebyollin/taesd")
            if vae_repo is None:
                raise FileNotFoundError("TAESD weights (madebyollin/taesd) not found locally; run download.py where network exists")
            vae_sd = load_taesd(vae_repo)
        else:
            vae_sd = load_autoencoder_kl(repo, A.vae_arch_for(model_id_or_path))
        if use_lcm_lora and not sd_turbo:
            lrepo = find_local_repo(lcm_lora_id or "latent-consistency/lcm-lora-sdv1-5")
            if lrepo is None:
                raise FileNotFoundError("LCM-LoRA weights not found locally")
            n = fuse_lora(unet_sd, _load_safetensors(os.path.join(lrepo, "pytorch_lora_weights.safetensors")), 1.0)
            logger.info("fused %d LCM-LoRA layers", n)
        for path, scale in (lora_dict or {}).items():
            n = fuse_lora(unet_sd, _load_safetensors(path), scale)
            logger.info("fused %d layers of %s (scale %s)", n, path, scale)
        A.validate_state_dict(unet_sd, A.unet_param_shapes(arch), "UNet checkpoint")
        if use_tiny_vae:
            A.validate_state_dict(vae_sd, A.taesd_param_shapes(), "TAESD checkpoint")
        return arch, unet_sd, vae_sd, repo
    if os.getenv(ALLOW_SYNTHETIC_ENV) or model_id_or_path.startswith(("tiny", "synthetic")):
        logger.warning("no checkpoint for %s on disk: using seeded synthetic weights (%s)", model_id_or_path, arch.name)
        unet_sd = A.synthetic_state_dict(A.unet_param_shapes(arch), seed=1234)
        if use_tiny_vae:
            vae_sd = A.synthetic_state_dict(A.taesd_param_shapes(), seed=4321, relu_net=True)
        else:
            vae_sd = A.synthetic_autoencoder_kl(A.vae_arch_for(model_id_or_path))
        return arch, unet_sd, vae_sd, None
    raise FileNotFoundError(
        f"model '{model_id_or_path}' not found on disk (no network for download.py); set {ALLOW_SYNTHETIC_ENV}=1 to run "
        "with seeded synthetic weights")
