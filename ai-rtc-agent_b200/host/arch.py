"""Architectures the reference can select (lib/wrapper.py:133: `"turbo" in model_id_or_path`) and the
parameter inventory of their checkpoints in diffusers' naming (used to validate loaded state dicts and
to build synthetic weights for benchmarking when no checkpoint is on disk -- download.py needs network).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Iterator, Tuple

import torch

Shape = Tuple[int, ...]


@dataclass(frozen=True)
class UNetArch:
    name: str
    block_out_channels: Tuple[int, int, int, int]
    heads: Tuple[int, int, int, int]          # diffusers `attention_head_dim` (= number of heads)
    cross_attention_dim: int
    use_linear_projection: bool
    down_attn: Tuple[int, int, int, int] = (1, 1, 1, 0)
    layers_per_block: int = 2
    norm_groups: int = 32
    ctx_tokens: int = 77


SD15 = UNetArch("sd15", (320, 640, 1280, 1280), (8, 8, 8, 8), 768, False)
SD_TURBO = UNetArch("sd-turbo", (320, 640, 1280, 1280), (5, 10, 20, 20), 1024, True)
# 1/5-width variants with the same topology (tests, smoke)
TINY_SD15 = UNetArch("tiny-sd15", (64, 128, 256, 256), (8, 8, 8, 8), 64, False)
TINY_TURBO = UNetArch("tiny-turbo", (64, 128, 256, 256), (1, 2, 4, 4), 128, True)


def arch_for(model_id: str) -> UNetArch:
    if model_id.rstrip("/").rsplit("/", 1)[-1].startswith("tiny"):   # a model id or a local directory name
        return TINY_TURBO if "turbo" in model_id else TINY_SD15
    return SD_TURBO if "turbo" in model_id else SD15


def _norm(prefix: str, c: int) -> Iterator[Tuple[str, Shape]]:
    yield prefix + ".weight", (c,)
    yield prefix + ".bias", (c,)


def _conv(prefix: str, co: int, ci: int, k: int, bias: bool = True) -> Iterator[Tuple[str, Shape]]:
    yield prefix + ".weight", (co, ci, k, k)
    if bias:
        yield prefix + ".bias", (co,)


def _linear(prefix: str, co: int, ci: int, bias: bool = True) -> Iterator[Tuple[str, Shape]]:
    yield prefix + ".weight", (co, ci)
    if bias:
        yield prefix + ".bias", (co,)


def _resnet(prefix: str, ci: int, co: int, tdim: int) -> Iterator[Tuple[str, Shape]]:
    yield from _norm(prefix + ".norm1", ci)
    yield from _conv(prefix + ".conv1", co, ci, 3)
    yield from _linear(prefix + ".time_emb_proj", co, tdim)
    yield from _norm(prefix + ".norm2", co)
    yield from _conv(prefix + ".conv2", co, co, 3)
    if ci != co:
        yield from _conv(prefix + ".conv_shortcut", co, ci, 1)


def _transformer(prefix: str, c: int, a: UNetArch) -> Iterator[Tuple[str, Shape]]:
    yield from _norm(prefix + ".norm", c)
    for proj in ("proj_in", "proj_out"):
        if a.use_linear_projection:
            yield from _linear(f"{prefix}.{proj}", c, c)
        else:
            yield from _conv(f"{prefix}.{proj}", c, c, 1)
    blk = prefix + ".transformer_blocks.0"
    for i in (1, 2, 3):
        yield from _norm(f"{blk}.norm{i}", c)
    for attn, kv in (("attn1", c), ("attn2", a.cross_attention_dim)):
        yield from _linear(f"{blk}.{attn}.to_q", c, c, bias=False)
        yield from _linear(f"{blk}.{attn}.to_k", c, kv, bias=False)
        yield from _linear(f"{blk}.{attn}.to_v", c, kv, bias=False)
        yield from _linear(f"{blk}.{attn}.to_out.0", c, c)
    yield from _linear(f"{blk}.ff.net.0.proj", 8 * c, c)
    yield from _linear(f"{blk}.ff.net.2", c, 4 * c)


def unet_param_shapes(a: UNetArch) -> Dict[str, Shape]:
    ch = a.block_out_channels
    tdim = 4 * ch[0]
    out: Dict[str, Shape] = {}
    out.update(_conv("conv_in", ch[0], 4, 3))
    out.update(_linear("time_embedding.linear_1", tdim, ch[0]))
    out.update(_linear("time_embedding.linear_2", tdim, tdim))
    skip = [ch[0]]
    cur = ch[0]
    for i, co in enumerate(ch):
        for j in range(a.layers_per_block):
            out.update(_resnet(f"down_blocks.{i}.resnets.{j}", cur, co, tdim))
            cur = co
            if a.down_attn[i]:
                out.update(_transformer(f"down_blocks.{i}.attentions.{j}", co, a))
            skip.append(cur)
        if i < len(ch) - 1:
            out.update(_conv(f"down_blocks.{i}.downsamplers.0.conv", co, co, 3))
            skip.append(cur)
    out.update(_resnet("mid_block.resnets.0", cur, cur, tdim))
    out.update(_transformer("mid_block.attentions.0", cur, a))
    out.update(_resnet("mid_block.resnets.1", cur, cur, tdim))
    for i, co in enumerate(reversed(ch)):
        for j in range(a.layers_per_block + 1):
            out.update(_resnet(f"up_blocks.{i}.resnets.{j}", cur + skip.pop(), co, tdim))
            cur = co
            if a.down_attn[len(ch) - 1 - i]:
                out.update(_transformer(f"up_blocks.{i}.attentions.{j}", co, a))
        if i < len(ch) - 1:
            out.update(_conv(f"up_blocks.{i}.upsamplers.0.conv", co, co, 3))
    out.update(_norm("conv_norm_out", ch[0]))
    out.update(_conv("conv_out", 4, ch[0], 3))
    return out


CN_EMBED_CHANNELS = (16, 32, 96, 256)   # ControlNetModel conditioning_embedding_out_channels (diffusers default)


def controlnet_param_shapes(a: UNetArch) -> Dict[str, Shape]:
    """diffusers ControlNetModel with the UNet's architecture fields: the conditioning embedding, a copy of the UNet's conv_in /
    time_embedding / down blocks / mid block, and one zero conv (1x1) per down residual plus the mid-block one."""
    ch = a.block_out_channels
    emb = CN_EMBED_CHANNELS
    out: Dict[str, Shape] = {}
    p = "controlnet_cond_embedding"
    out.update(_conv(f"{p}.conv_in", emb[0], 3, 3))
    for i in range(len(emb) - 1):
        out.update(_conv(f"{p}.blocks.{2 * i}", emb[i], emb[i], 3))
        out.update(_conv(f"{p}.blocks.{2 * i + 1}", emb[i + 1], emb[i], 3))
    out.update(_conv(f"{p}.conv_out", ch[0], emb[-1], 3))
    unet = unet_param_shapes(a)
    out.update({k: v for k, v in unet.items() if k.startswith(("conv_in.", "time_embedding.", "down_blocks.", "mid_block."))})
    skip = [ch[0]]
    for i, co in enumerate(ch):
        skip += [co] * (a.layers_per_block + (1 if i < len(ch) - 1 else 0))
    for k, c in enumerate(skip):
        out.update(_conv(f"controlnet_down_blocks.{k}", c, c, 1))
    out.update(_conv("controlnet_mid_block", ch[-1], ch[-1], 1))
    return out


HED_BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))   # (in, out, convs)


def hed_param_shapes() -> Dict[str, Shape]:
    """controlnet_aux ControlNetHED_Apache2 (lllyasviel/Annotators ControlNetHED.pth): the input offset `norm` and five
    DoubleConvBlocks of 3x3 convs with a 1x1 projection to one channel each."""
    out: Dict[str, Shape] = {"norm": (1, 3, 1, 1)}
    for b, (ci, co, n) in enumerate(HED_BLOCKS, start=1):
        for k in range(n):
            out.update(_conv(f"block{b}.convs.{k}", co, ci if k == 0 else co, 3))
        out.update(_conv(f"block{b}.projection", 1, co, 1))
    return out


def synthetic_hed(seed: int = 2468) -> Dict[str, torch.Tensor]:
    """Seeded fp32 HED weights.  Its input is on the 0..255 scale: He gain on the ReLU convs keeps the activations' second
    moment (~70^2) through block 5, far inside fp16; the projections are scaled so that the side outputs are O(1) and the
    sigmoid of their mean gives a graded edge map rather than a saturated one."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in hed_param_shapes().items():
        if name == "norm":
            t = 100.0 + 30.0 * torch.rand(shape, generator=g)
        elif name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=g)
        elif ".projection." in name:
            t = torch.randn(shape, generator=g) * (0.03 / math.sqrt(shape[1]))
        else:
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / math.prod(shape[1:]))
        sd[name] = t
    return sd


def taesd_param_shapes() -> Dict[str, Shape]:
    """madebyollin/taesd AutoencoderTiny: nn.Sequential indices as diffusers builds them."""
    out: Dict[str, Shape] = {}

    def block(p: str):
        for k in (0, 2, 4):
            out.update(_conv(f"{p}.conv.{k}", 64, 64, 3))

    idx = 0
    for stage, nblk in enumerate((1, 3, 3, 3)):
        out.update(_conv(f"encoder.layers.{idx}", 64, 3 if stage == 0 else 64, 3, bias=(stage == 0)))
        idx += 1
        for _ in range(nblk):
            block(f"encoder.layers.{idx}")
            idx += 1
    out.update(_conv(f"encoder.layers.{idx}", 4, 64, 3))
    out.update(_conv("decoder.layers.0", 64, 4, 3))
    idx = 2
    for stage, nblk in enumerate((3, 3, 3, 1)):
        for _ in range(nblk):
            block(f"decoder.layers.{idx}")
            idx += 1
        if stage < 3:
            idx += 1  # nn.Upsample
            out.update(_conv(f"decoder.layers.{idx}", 64, 64, 3, bias=False))
        else:
            out.update(_conv(f"decoder.layers.{idx}", 3, 64, 3))
        idx += 1
    return out


@dataclass(frozen=True)
class VaeArch:
    """diffusers AutoencoderKL (vae/config.json): DownEncoderBlock2D / UpDecoderBlock2D, SiLU, GroupNorm eps 1e-6."""
    name: str
    block_out_channels: Tuple[int, int, int, int]
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_groups: int = 32


AUTOENCODER_KL = VaeArch("autoencoder-kl", (128, 256, 512, 512))          # SD-1.5, SD-2.1, SD-Turbo
# a narrower variant for tests; its last level stays 512 wide, the width of the engine's single-head attention
TINY_AUTOENCODER_KL = VaeArch("tiny-autoencoder-kl", (64, 128, 128, 512))


def vae_arch_for(model_id: str) -> VaeArch:
    return TINY_AUTOENCODER_KL if model_id.rstrip("/").rsplit("/", 1)[-1].startswith("tiny") else AUTOENCODER_KL


def _vae_resnet(prefix: str, ci: int, co: int) -> Iterator[Tuple[str, Shape]]:
    yield from _norm(prefix + ".norm1", ci)
    yield from _conv(prefix + ".conv1", co, ci, 3)
    yield from _norm(prefix + ".norm2", co)
    yield from _conv(prefix + ".conv2", co, co, 3)
    if ci != co:
        yield from _conv(prefix + ".conv_shortcut", co, ci, 1)


def _vae_mid(prefix: str, c: int) -> Iterator[Tuple[str, Shape]]:
    yield from _vae_resnet(prefix + ".resnets.0", c, c)
    yield from _norm(prefix + ".attentions.0.group_norm", c)
    for proj in ("to_q", "to_k", "to_v", "to_out.0"):
        yield from _linear(f"{prefix}.attentions.0.{proj}", c, c)
    yield from _vae_resnet(prefix + ".resnets.1", c, c)


def autoencoder_kl_param_shapes(v: VaeArch = AUTOENCODER_KL) -> Dict[str, Shape]:
    """State-dict inventory of a diffusers AutoencoderKL with the current attention names (to_q / to_k / to_v / to_out.0)."""
    ch, lat, n = v.block_out_channels, v.latent_channels, len(v.block_out_channels)
    out: Dict[str, Shape] = {}
    out.update(_conv("encoder.conv_in", ch[0], 3, 3))
    cur = ch[0]
    for i, co in enumerate(ch):
        for j in range(v.layers_per_block):
            out.update(_vae_resnet(f"encoder.down_blocks.{i}.resnets.{j}", cur, co))
            cur = co
        if i < n - 1:
            out.update(_conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co, 3))
    out.update(_vae_mid("encoder.mid_block", cur))
    out.update(_norm("encoder.conv_norm_out", cur))
    out.update(_conv("encoder.conv_out", 2 * lat, cur, 3))
    out.update(_conv("quant_conv", 2 * lat, 2 * lat, 1))
    out.update(_conv("post_quant_conv", lat, lat, 1))
    out.update(_conv("decoder.conv_in", ch[-1], lat, 3))
    out.update(_vae_mid("decoder.mid_block", ch[-1]))
    cur = ch[-1]
    for i, co in enumerate(reversed(ch)):
        for j in range(v.layers_per_block + 1):
            out.update(_vae_resnet(f"decoder.up_blocks.{i}.resnets.{j}", cur, co))
            cur = co
        if i < n - 1:
            out.update(_conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", co, co, 3))
    out.update(_norm("decoder.conv_norm_out", cur))
    out.update(_conv("decoder.conv_out", 3, cur, 3))
    return out


_LEGACY_VAE_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def normalize_autoencoder_kl(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Current diffusers names for a state dict saved with the legacy attention names (query / key / value / proj_attn), and the
    mid-block q / k / v / out projections as [C, C] matrices however they were stored ([C, C, 1, 1] in older checkpoints), as
    diffusers' loader does."""
    out: Dict[str, torch.Tensor] = {}
    for k, t in sd.items():
        parts = k.split(".")
        if ".attentions." in k and len(parts) >= 2 and parts[-2] in _LEGACY_VAE_ATTN:
            k = ".".join(parts[:-2] + [_LEGACY_VAE_ATTN[parts[-2]], parts[-1]])
        if ".attentions." in k and k.endswith(".weight") and t.dim() == 4 and t.shape[2:] == (1, 1):
            t = t.reshape(t.shape[0], t.shape[1])
        out[k] = t
    return out


def validate_exact(sd: Dict[str, torch.Tensor], shapes: Dict[str, Shape], what: str) -> None:
    """Every tensor of the inventory present with exactly its shape, and nothing else."""
    missing = [k for k in shapes if k not in sd]
    if missing:
        raise ValueError(f"{what}: {len(missing)} missing tensors, e.g. {missing[:4]}")
    extra = [k for k in sd if k not in shapes]
    if extra:
        raise ValueError(f"{what}: {len(extra)} unexpected tensors, e.g. {extra[:4]}")
    for k, shp in shapes.items():
        if tuple(sd[k].shape) != tuple(shp):
            raise ValueError(f"{what}: {k} has shape {tuple(sd[k].shape)}, expected {shp}")


def synthetic_autoencoder_kl(v: VaeArch = AUTOENCODER_KL, seed: int = 8765) -> Dict[str, torch.Tensor]:
    """Seeded fp16 AutoencoderKL weights: fan-in scaled convs (residual branches' last layers at half gain), GroupNorm affine
    near identity, nonzero biases everywhere (quant_conv / post_quant_conv included, so that a bias folded across a zero-padded
    conv shows up on the border pixels), and a decoder conv_out that keeps the image mostly inside [-1, 1]."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in autoencoder_kl_param_shapes(v).items():
        leaf = name.rsplit(".", 1)[-1]
        if "norm" in name.rsplit(".", 2)[-2]:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g) if leaf == "weight" else 0.1 * torch.randn(shape, generator=g)
        elif leaf == "bias":
            t = 0.05 * torch.randn(shape, generator=g)
        else:
            gain = 0.5 if name.endswith(("conv2.weight", "to_out.0.weight")) else 1.0
            if name == "decoder.conv_out.weight":
                gain = 0.35
            t = torch.randn(shape, generator=g) * (gain / math.sqrt(math.prod(shape[1:])))
        sd[name] = t.to(torch.float16)
    return sd


def synthetic_state_dict(shapes: Dict[str, Shape], seed: int, relu_net: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded fp16 weights with fan-in scaling (activations stay O(1) through the whole network); used by
    bench.py / smoke when no checkpoint exists.  Not a trained model: outputs are noise-like images.  A ControlNet's zero
    convs are drawn like any other layer (non-zero), so that its residuals reach the output."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in shapes.items():
        leaf = name.rsplit(".", 1)[-1]
        if ".norm" in name or name.startswith("conv_norm_out"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g) if leaf == "weight" else 0.1 * torch.randn(shape, generator=g)
        elif leaf == "bias":
            t = 0.05 * torch.randn(shape, generator=g)
        else:
            fan_in = math.prod(shape[1:])
            gain = math.sqrt(2.0) if relu_net else 1.0
            if any(k in name for k in ("conv2.", "to_out.0.", "ff.net.2.", "proj_out.", "conv.4.")):
                gain = 0.5 if not relu_net else 0.7
            t = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        sd[name] = t.to(torch.float16)
    if relu_net:  # keep the decoded image around mid-grey
        last = max(int(k.split(".")[2]) for k in sd if k.startswith("decoder.layers."))
        sd[f"decoder.layers.{last}.bias"] = torch.full((3,), 0.5, dtype=torch.float16)
        sd[f"decoder.layers.{last}.weight"] = (sd[f"decoder.layers.{last}.weight"].float() * 0.25).to(torch.float16)
    return sd


def validate_state_dict(sd: Dict[str, torch.Tensor], shapes: Dict[str, Shape], what: str) -> None:
    missing = [k for k in shapes if k not in sd]
    if missing:
        raise ValueError(f"{what}: {len(missing)} missing tensors, e.g. {missing[:4]}")
    for k, shp in shapes.items():
        if tuple(sd[k].shape) != tuple(shp):
            # diffusers stores 1x1 conv projections as (c, c, 1, 1); linear ones as (c, c)
            if math.prod(sd[k].shape) != math.prod(shp):
                raise ValueError(f"{what}: {k} has shape {tuple(sd[k].shape)}, expected {shp}")
