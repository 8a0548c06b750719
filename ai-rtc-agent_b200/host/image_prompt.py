"""IP-Adapter image prompts (h94 `ip-adapter_sd15.safetensors` layout): the adapter file, its mapping onto the UNet's
cross-attentions, the image projection, and the image encoder.

An image prompt is one CLIP image embedding turned into `n_tok` extra context tokens by the adapter's projection
(Linear -> reshape (n_tok, D) -> LayerNorm, `ImageProjModel`); every UNet cross-attention then adds a second, separately
normalised attention over those tokens with the adapter's own to_k_ip / to_v_ip.  The encoder and the projection run once per
image prompt, on the host side, never per frame: the CLIP vision encoder in torch fp16 (as the CLIP text encoder in
prompt.py), the projection in fp32."""
from __future__ import annotations

import hashlib
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import arch as A

Shape = Tuple[int, ...]

IP_TOKENS = 4            # ImageProjModel's clip_extra_context_tokens of ip-adapter_sd15
IMAGE_EMBED_DIM = 1024   # CLIP ViT-H/14 image_embeds (the h94 image_encoder/)
IP_ADAPTER_ENV = "B200SD_IP_ADAPTER"


def cross_attention_modules(a: A.UNetArch) -> List[str]:
    """The UNet's cross-attentions (`...transformer_blocks.0.attn2`) in the order IP-Adapter numbers them: diffusers'
    `unet.attn_processors` order, down blocks, then up blocks, then the mid block; the adapter's ip_adapter.{i} with
    i = 1, 3, ..., 2n-1 is the k-th of them for i = 2k + 1 (the even i are the self-attentions, which carry no weights).
    This order is recalled from the upstream projects, not checked against them here; it is pinned by a test, and this is the
    one place that knows it."""
    ch = a.block_out_channels
    mods = []
    for i in range(len(ch)):
        if a.down_attn[i]:
            mods += [f"down_blocks.{i}.attentions.{j}.transformer_blocks.0.attn2" for j in range(a.layers_per_block)]
    for i in range(len(ch)):
        if a.down_attn[len(ch) - 1 - i]:
            mods += [f"up_blocks.{i}.attentions.{j}.transformer_blocks.0.attn2" for j in range(a.layers_per_block + 1)]
    return mods + ["mid_block.attentions.0.transformer_blocks.0.attn2"]


def _attn2_channels(a: A.UNetArch) -> Dict[str, int]:
    shapes = A.unet_param_shapes(a)
    return {m: shapes[m + ".to_q.weight"][0] for m in cross_attention_modules(a)}


def adapter_key_map(a: A.UNetArch) -> Dict[str, str]:
    """adapter file key -> the UNet key the engine reads beside to_k / to_v"""
    out = {}
    for k, m in enumerate(cross_attention_modules(a)):
        for w in ("to_k_ip", "to_v_ip"):
            out[f"ip_adapter.{2 * k + 1}.{w}.weight"] = f"{m}.{w}.weight"
    return out


def adapter_shapes(a: A.UNetArch, embed_dim: int = IMAGE_EMBED_DIM, n_tok: int = IP_TOKENS) -> Dict[str, Shape]:
    """every key of an adapter file for this UNet and its shape"""
    D = a.cross_attention_dim
    out: Dict[str, Shape] = {"image_proj.proj.weight": (n_tok * D, embed_dim), "image_proj.proj.bias": (n_tok * D,),
                             "image_proj.norm.weight": (D,), "image_proj.norm.bias": (D,)}
    chans = _attn2_channels(a)
    for key, unet_key in adapter_key_map(a).items():
        out[key] = (chans[unet_key.rsplit(".", 2)[0]], D)
    return out


@dataclass
class IPAdapter:
    """A loaded adapter: the projection (fp32) and the UNet's to_k_ip / to_v_ip under UNet names (fp16)"""
    proj_w: torch.Tensor
    proj_b: torch.Tensor
    norm_w: torch.Tensor
    norm_b: torch.Tensor
    n_tok: int
    unet: Dict[str, torch.Tensor]
    path: Optional[str] = None

    @property
    def embed_dim(self) -> int:
        return self.proj_w.shape[1]

    def tokens(self, image_embeds: torch.Tensor) -> torch.Tensor:
        """ImageProjModel: (E,) or (1, E) CLIP image embedding -> (1, n_tok, D) fp16 tokens, computed in fp32"""
        x = image_embeds.detach().reshape(1, -1).float().cpu()
        D = self.norm_w.shape[0]
        t = F.linear(x, self.proj_w, self.proj_b).reshape(1, self.n_tok, D)
        return F.layer_norm(t, (D,), self.norm_w, self.norm_b, 1e-5).to(torch.float16)


def adapter_from_state_dict(sd: Dict[str, torch.Tensor], a: A.UNetArch, path: Optional[str] = None) -> IPAdapter:
    """Check every key and shape of an adapter state dict against the UNet and name the first one that does not fit"""
    what = f"IP-Adapter {path}" if path else "IP-Adapter"
    D = a.cross_attention_dim
    for key in ("image_proj.proj.weight", "image_proj.norm.weight"):
        if key not in sd:
            raise ValueError(f"{what}: missing '{key}'")
    nw = tuple(sd["image_proj.norm.weight"].shape)
    if nw != (D,):
        raise ValueError(f"{what}: 'image_proj.norm.weight' has shape {nw}: the adapter's cross_attention_dim is "
                         f"{nw[0] if nw else '?'}, the UNet's {D}")
    pw = tuple(sd["image_proj.proj.weight"].shape)
    if len(pw) != 2 or pw[0] % D or not 1 <= pw[0] // D <= 64:
        raise ValueError(f"{what}: 'image_proj.proj.weight' has shape {pw}, expected [n_tok * {D}, embed_dim] with "
                         "1 <= n_tok <= 64")
    n_tok, embed_dim = pw[0] // D, pw[1]
    n_want = len(cross_attention_modules(a))
    n_got = len({k.split(".")[1] for k in sd if k.startswith("ip_adapter.")})
    if n_got != n_want:
        raise ValueError(f"{what}: weights for {n_got} cross-attentions, the UNet ({a.name}) has {n_want}")
    shapes = adapter_shapes(a, embed_dim, n_tok)
    for key, shape in shapes.items():
        if key not in sd:
            raise ValueError(f"{what}: missing '{key}'")
        if tuple(sd[key].shape) != shape:
            raise ValueError(f"{what}: '{key}' has shape {tuple(sd[key].shape)}, expected {shape}")
    extra = sorted(set(sd) - set(shapes))
    if extra:
        raise ValueError(f"{what}: unexpected key '{extra[0]}'")
    f32 = {k: sd[k].float() for k in ("image_proj.proj.weight", "image_proj.proj.bias", "image_proj.norm.weight",
                                      "image_proj.norm.bias")}
    unet = {u: sd[k].to(torch.float16).contiguous() for k, u in adapter_key_map(a).items()}
    return IPAdapter(f32["image_proj.proj.weight"], f32["image_proj.proj.bias"], f32["image_proj.norm.weight"],
                     f32["image_proj.norm.bias"], n_tok, unet, path)


def adapter_file(path: str) -> str:
    """The adapter file of `path`: the file itself, or the single ip-adapter*.safetensors of a directory"""
    if os.path.isdir(path):
        found = sorted(n for n in os.listdir(path) if n.startswith("ip-adapter") and n.endswith(".safetensors"))
        if len(found) != 1:
            raise FileNotFoundError(f"{path}: expected one ip-adapter*.safetensors, found {found or 'none'}")
        return os.path.join(path, found[0])
    return path


def load_adapter(path: str, a: A.UNetArch) -> IPAdapter:
    """An adapter file (or a directory holding one).  Only safetensors are read, never a pickle (which can run code)."""
    path = adapter_file(path)
    if not str(path).endswith(".safetensors"):
        raise ValueError(f"IP-Adapter {path}: only .safetensors files are read")
    from safetensors.torch import load_file
    try:
        sd = load_file(path)
    except FileNotFoundError:
        raise
    except Exception as exc:   # noqa: BLE001 - safetensors raises its own error type on a file that is not safetensors
        raise ValueError(f"IP-Adapter {path}: not a safetensors file ({exc})") from exc
    return adapter_from_state_dict(sd, a, path)


def synthetic_adapter_state_dict(a: A.UNetArch, seed: int = 9753, embed_dim: int = IMAGE_EMBED_DIM,
                                 n_tok: int = IP_TOKENS) -> Dict[str, torch.Tensor]:
    """Seeded adapter weights in the file's naming (tests, benchmarks without a checkpoint)"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for key, shape in adapter_shapes(a, embed_dim, n_tok).items():
        if key == "image_proj.norm.weight":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            t = 0.1 * torch.randn(shape, generator=g)
        else:
            t = torch.randn(shape, generator=g) / shape[1] ** 0.5
        out[key] = t.to(torch.float16)
    return out


# ---- images -------------------------------------------------------------------------------------------------------------
def image_array(image) -> np.ndarray:
    """A PIL image, or an HWC uint8 array / tensor, as a contiguous HWC uint8 RGB array.  Never a path: a client must not be able
    to make the server open files."""
    if isinstance(image, (str, bytes, os.PathLike)):
        raise TypeError("an image prompt is a PIL image or an HWC uint8 array / tensor, not a path")
    if hasattr(image, "convert") and hasattr(image, "size"):   # PIL.Image
        return np.ascontiguousarray(np.asarray(image.convert("RGB"), dtype=np.uint8))
    if isinstance(image, torch.Tensor):
        image = image.detach().cpu().numpy()
    if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] not in (3, 4):
        raise TypeError("an image prompt is a PIL image or an HWC uint8 array / tensor with 3 or 4 channels")
    return np.ascontiguousarray(image[:, :, :3])


class SyntheticImageEncoder:
    """Deterministic stand-in for the CLIP vision encoder: seeds a CPU generator from sha256 of the image's shape and bytes."""

    def __init__(self, embed_dim: int = IMAGE_EMBED_DIM):
        self.embed_dim = embed_dim

    def __call__(self, image) -> torch.Tensor:
        arr = image_array(image)
        h = hashlib.sha256(repr(arr.shape).encode() + arr.tobytes()).digest()
        g = torch.Generator().manual_seed(int.from_bytes(h[:8], "little") % (2 ** 63))
        return torch.randn((1, self.embed_dim), generator=g)


class ClipImageEncoder:
    """CLIPVisionModelWithProjection + CLIPImageProcessor from a local image_encoder/ directory, fp16"""

    def __init__(self, encoder_dir: str, device: str = "cuda"):
        from transformers import CLIPImageProcessor, CLIPVisionModelWithProjection
        self.processor = CLIPImageProcessor.from_pretrained(encoder_dir)
        self.model = CLIPVisionModelWithProjection.from_pretrained(encoder_dir, dtype=torch.float16).to(device).eval()
        self.device = device
        self.embed_dim = self.model.config.projection_dim

    @torch.no_grad()
    def __call__(self, image) -> torch.Tensor:
        px = self.processor(images=image_array(image), return_tensors="pt").pixel_values.to(self.device, torch.float16)
        return self.model(px).image_embeds


def make_image_encoder(adapter_path: Optional[str], embed_dim: int, device: str = "cuda", allow_synthetic: bool = False):
    """The image_encoder/ beside the adapter file (or in the adapter directory) must load when it exists or when the adapter is a
    real checkpoint; the synthetic encoder is for synthetic adapter weights only (as make_prompt_encoder)."""
    if adapter_path:
        base = adapter_path if os.path.isdir(adapter_path) else os.path.dirname(os.path.abspath(adapter_path))
        for d in (os.path.join(base, "image_encoder"), os.path.join(os.path.dirname(base), "image_encoder")):
            if os.path.isdir(d):
                enc = ClipImageEncoder(d, device)
                if enc.embed_dim != embed_dim:
                    raise ValueError(f"image encoder under {d} has projection_dim {enc.embed_dim}, the adapter expects "
                                     f"{embed_dim}")
                return enc
        if not allow_synthetic:
            raise FileNotFoundError(f"no image_encoder/ beside {adapter_path}: cannot encode image prompts for a real adapter "
                                    "(set B200SD_SYNTHETIC_WEIGHTS=1 to run with synthetic embeddings)")
    return SyntheticImageEncoder(embed_dim)
