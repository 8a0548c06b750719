"""fp32 restatement of diffusers' `AutoencoderKL` as StreamDiffusion drives it with use_tiny_vae=False (lib/wrapper.py:699-705):
models/autoencoders/autoencoder_kl.py + vae.py (Encoder, Decoder), resnet.py (ResnetBlock2D without a time embedding),
downsampling.py (Downsample2D with padding=0: F.pad(x, (0, 1, 0, 1)) then a stride-2 conv), upsampling.py (nearest 2x + conv),
attention_processor.py (Attention(heads=1, residual_connection=True, bias=True, upcast_softmax=True)).  GroupNorm: 32 groups,
eps 1e-6.  encode_mean returns the mean of the latent distribution (channels 0-3 after quant_conv), not a sample of it.  Test
infrastructure only (see oracle/__init__)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
EPS = 1e-6
GROUPS = 32
SCALING_FACTOR = 0.18215   # vae/config.json of SD-1.5 / SD-2.1 / SD-Turbo


@dataclass(frozen=True)
class KLConfig:
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4


FULL = KLConfig()
TINY = KLConfig((64, 128, 128, 512))


def param_shapes(cfg: KLConfig = FULL) -> Dict[str, Tuple[int, ...]]:
    """Parameter inventory, written from diffusers' module tree (independently of host/arch.py, which it is tested against)."""
    s: Dict[str, Tuple[int, ...]] = {}

    def conv(p, co, ci, k):
        s[p + ".weight"] = (co, ci, k, k)
        s[p + ".bias"] = (co,)

    def norm(p, c):
        s[p + ".weight"] = (c,)
        s[p + ".bias"] = (c,)

    def resnet(p, ci, co):
        norm(p + ".norm1", ci); conv(p + ".conv1", co, ci, 3)
        norm(p + ".norm2", co); conv(p + ".conv2", co, co, 3)
        if ci != co:
            conv(p + ".conv_shortcut", co, ci, 1)

    def mid(p, c):
        resnet(p + ".resnets.0", c, c)
        norm(p + ".attentions.0.group_norm", c)
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            s[f"{p}.attentions.0.{n}.weight"] = (c, c)
            s[f"{p}.attentions.0.{n}.bias"] = (c,)
        resnet(p + ".resnets.1", c, c)

    ch, z = cfg.block_out_channels, cfg.latent_channels
    conv("encoder.conv_in", ch[0], 3, 3)
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg.layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        if i != len(ch) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", c, c, 3)
        prev = c
    mid("encoder.mid_block", ch[-1])
    norm("encoder.conv_norm_out", ch[-1])
    conv("encoder.conv_out", 2 * z, ch[-1], 3)
    conv("quant_conv", 2 * z, 2 * z, 1)
    conv("post_quant_conv", z, z, 1)
    conv("decoder.conv_in", ch[-1], z, 3)
    mid("decoder.mid_block", ch[-1])
    rev = list(reversed(ch))
    prev = rev[0]
    for i, c in enumerate(rev):
        for j in range(cfg.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        if i != len(rev) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", c, c, 3)
        prev = c
    norm("decoder.conv_norm_out", rev[-1])
    conv("decoder.conv_out", 3, rev[-1], 3)
    return s


def _gn(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    return F.group_norm(x, GROUPS, sd[p + ".weight"], sd[p + ".bias"], EPS)


def _conv(sd: SD, p: str, x: torch.Tensor, stride: int = 1, padding: int = 1) -> torch.Tensor:
    return F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], stride=stride, padding=padding)


def _resnet(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    h = _conv(sd, p + ".conv1", F.silu(_gn(sd, p + ".norm1", x)))
    h = _conv(sd, p + ".conv2", F.silu(_gn(sd, p + ".norm2", h)))
    sc = _conv(sd, p + ".conv_shortcut", x, padding=0) if (p + ".conv_shortcut.weight") in sd else x
    return sc + h


def _attention(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    b, c, h, w = x.shape
    t = _gn(sd, p + ".group_norm", x).reshape(b, c, h * w).transpose(1, 2)
    lin = lambda n, v: F.linear(v, sd[f"{p}.{n}.weight"].reshape(c, c), sd[f"{p}.{n}.bias"])
    q, k, v = lin("to_q", t), lin("to_k", t), lin("to_v", t)
    a = torch.softmax((q @ k.transpose(1, 2)).float() / c ** 0.5, dim=-1).to(q.dtype)
    o = lin("to_out.0", a @ v)
    return o.transpose(1, 2).reshape(b, c, h, w) + x


def _mid(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    x = _resnet(sd, p + ".resnets.0", x)
    x = _attention(sd, p + ".attentions.0", x)
    return _resnet(sd, p + ".resnets.1", x)


def encode_mean(sd: SD, images: torch.Tensor, cfg: KLConfig = FULL, taps: Dict[str, torch.Tensor] = None) -> torch.Tensor:
    """images in [-1, 1] (B,3,H,W) -> mean of the latent distribution (B,4,H/8,W/8), before scaling_factor."""
    x = _conv(sd, "encoder.conv_in", images)
    for i in range(len(cfg.block_out_channels)):
        for j in range(cfg.layers_per_block):
            x = _resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}", x)
        if i != len(cfg.block_out_channels) - 1:
            x = _conv(sd, f"encoder.down_blocks.{i}.downsamplers.0.conv", F.pad(x, (0, 1, 0, 1)), stride=2, padding=0)
        if taps is not None:
            taps[f"vae.enc.down.{i}"] = x
    x = _mid(sd, "encoder.mid_block", x)
    if taps is not None:
        taps["vae.enc.mid"] = x
    x = _conv(sd, "encoder.conv_out", F.silu(_gn(sd, "encoder.conv_norm_out", x)))
    moments = _conv(sd, "quant_conv", x, padding=0)
    return moments[:, :cfg.latent_channels]


def decode(sd: SD, z: torch.Tensor, cfg: KLConfig = FULL, taps: Dict[str, torch.Tensor] = None) -> torch.Tensor:
    """AutoencoderKL.decode(z).sample: latents (already divided by scaling_factor) -> image, roughly [-1, 1]."""
    x = _conv(sd, "post_quant_conv", z, padding=0)
    x = _conv(sd, "decoder.conv_in", x)
    x = _mid(sd, "decoder.mid_block", x)
    if taps is not None:
        taps["vae.dec.mid"] = x
    n = len(cfg.block_out_channels)
    for i in range(n):
        for j in range(cfg.layers_per_block + 1):
            x = _resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}", x)
        if i != n - 1:
            x = _conv(sd, f"decoder.up_blocks.{i}.upsamplers.0.conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))
        if taps is not None:
            taps[f"vae.dec.up.{i}"] = x
    return _conv(sd, "decoder.conv_out", F.silu(_gn(sd, "decoder.conv_norm_out", x)))
