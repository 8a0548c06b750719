"""fp32 restatement of diffusers 0.24 `ControlNetModel` (models/controlnet.py) for the UNet architectures of oracle/unet.py.
[EXT] Recalled from the public upstream project, not verifiable offline; the tests pin this restatement.

  * ControlNetConditioningEmbedding: conv_in 3->16 + SiLU, then for (16, 32, 96, 256) a 3x3 conv keeping the width and a
    stride-2 3x3 conv to the next width, each + SiLU, then conv_out 256 -> block_out_channels[0] (no activation): image
    resolution in, latent resolution out.
  * sample = conv_in(x) + cond_embedding(control); its own time_embedding; the UNet's down blocks and mid block.
  * zero convs: controlnet_down_blocks.{k} (1x1, one per down residual in the UNet's push order) and controlnet_mid_block.
  * conditioning scale 1.0 (the diffusers default).

The state dict uses diffusers' ControlNetModel key names (no prefix).  Also here: the UNet forward with
`down_block_additional_residuals` / `mid_block_additional_residual`, the stream oracle that runs both, and seeded weights.
Test infrastructure only (see oracle/__init__)."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from . import hed, unet
from . import weights as ow
from .stream import StreamOracle, image_preprocess

EMBED_CHANNELS = (16, 32, 96, 256)


def param_shapes(cfg: unet.UNetConfig) -> Dict[str, Tuple[int, ...]]:
    s: Dict[str, Tuple[int, ...]] = {}
    e = EMBED_CHANNELS
    p = "controlnet_cond_embedding."
    s[p + "conv_in.weight"] = (e[0], 3, 3, 3); s[p + "conv_in.bias"] = (e[0],)
    for i in range(len(e) - 1):
        s[p + f"blocks.{2 * i}.weight"] = (e[i], e[i], 3, 3); s[p + f"blocks.{2 * i}.bias"] = (e[i],)
        s[p + f"blocks.{2 * i + 1}.weight"] = (e[i + 1], e[i], 3, 3); s[p + f"blocks.{2 * i + 1}.bias"] = (e[i + 1],)
    c0 = cfg.block_out_channels[0]
    s[p + "conv_out.weight"] = (c0, e[-1], 3, 3); s[p + "conv_out.bias"] = (c0,)
    for k, v in unet.param_shapes(cfg).items():
        if k.startswith(("conv_in.", "time_embedding.", "down_blocks.", "mid_block.")):
            s[k] = v
    for k, c in enumerate(down_residual_channels(cfg)):
        s[f"controlnet_down_blocks.{k}.weight"] = (c, c, 1, 1); s[f"controlnet_down_blocks.{k}.bias"] = (c,)
    cm = cfg.block_out_channels[-1]
    s["controlnet_mid_block.weight"] = (cm, cm, 1, 1); s["controlnet_mid_block.bias"] = (cm,)
    return s


def down_residual_channels(cfg: unet.UNetConfig) -> List[int]:
    ch = cfg.block_out_channels
    out = [ch[0]]
    for i, co in enumerate(ch):
        out += [co] * (cfg.layers_per_block + (1 if i != len(ch) - 1 else 0))
    return out


def cond_embedding(sd: unet.SD, control: torch.Tensor) -> torch.Tensor:
    """control (B,3,H,W) in [0,1] -> (B, C0, H/8, W/8)."""
    p = "controlnet_cond_embedding."
    h = F.silu(F.conv2d(control, sd[p + "conv_in.weight"], sd[p + "conv_in.bias"], padding=1))
    for k in range(2 * (len(EMBED_CHANNELS) - 1)):
        h = F.silu(F.conv2d(h, sd[p + f"blocks.{k}.weight"], sd[p + f"blocks.{k}.bias"], padding=1, stride=1 + k % 2))
    return F.conv2d(h, sd[p + "conv_out.weight"], sd[p + "conv_out.bias"], padding=1)


def controlnet_forward(sd: unet.SD, cfg: unet.UNetConfig, sample: torch.Tensor, timesteps: torch.Tensor,
                       encoder_hidden_states: torch.Tensor, control: torch.Tensor,
                       taps: Optional[Dict[str, torch.Tensor]] = None) -> Tuple[List[torch.Tensor], torch.Tensor]:
    """(down_block_res_samples, mid_block_res_sample) after the zero convs.  control: (1 or B, 3, H, W) in [0,1]; a single
    control image conditions every batch item.  `taps` collects "cond" (the embedding), "conv_in" (conv_in(x) + cond) and
    "down.I.J" / "mid" before the zero convs (the names of oracle/unet.py)."""
    ch = cfg.block_out_channels
    emb = unet.time_embed(sd, cfg, timesteps)
    ctx = encoder_hidden_states
    cond = cond_embedding(sd, control)
    h = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1) + cond
    if taps is not None:
        taps["cond"] = cond
        taps["conv_in"] = h
    feats = [h]
    for i in range(len(ch)):
        for j in range(cfg.layers_per_block):
            h = unet.resnet(sd, f"down_blocks.{i}.resnets.{j}.", cfg, h, emb)
            if cfg.down_attn[i]:
                h = unet.transformer(sd, f"down_blocks.{i}.attentions.{j}.", cfg, cfg.heads[i], h, ctx)
            feats.append(h)
            if taps is not None:
                taps[f"down.{i}.{j}"] = h
        if i != len(ch) - 1:
            p = f"down_blocks.{i}.downsamplers.0.conv."
            h = F.conv2d(h, sd[p + "weight"], sd[p + "bias"], stride=2, padding=1)
            feats.append(h)
    h = unet.resnet(sd, "mid_block.resnets.0.", cfg, h, emb)
    h = unet.transformer(sd, "mid_block.attentions.0.", cfg, cfg.heads[-1], h, ctx)
    h = unet.resnet(sd, "mid_block.resnets.1.", cfg, h, emb)
    if taps is not None:
        taps["mid"] = h
    res = [F.conv2d(f, sd[f"controlnet_down_blocks.{k}.weight"], sd[f"controlnet_down_blocks.{k}.bias"])
           for k, f in enumerate(feats)]
    mid = F.conv2d(h, sd["controlnet_mid_block.weight"], sd["controlnet_mid_block.bias"])
    return res, mid


def unet_forward(sd: unet.SD, cfg: unet.UNetConfig, sample: torch.Tensor, timesteps: torch.Tensor,
                 encoder_hidden_states: torch.Tensor, down_block_additional_residuals: List[torch.Tensor],
                 mid_block_additional_residual: torch.Tensor, taps: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
    """oracle/unet.py unet_forward with a ControlNet's residuals (UNet2DConditionModel.forward): they are added to the skips the
    up path concatenates and to the mid-block output; the down path itself runs on the unmodified tensors.  `taps` gets the
    UNet's names plus "res.K" (skip K + residual K) and "cn_mid" (mid + residual)."""
    ch = cfg.block_out_channels
    emb = unet.time_embed(sd, cfg, timesteps)
    ctx = encoder_hidden_states
    h = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    skips = [h]
    if taps is not None:
        taps["conv_in"] = h
    for i in range(len(ch)):
        for j in range(cfg.layers_per_block):
            h = unet.resnet(sd, f"down_blocks.{i}.resnets.{j}.", cfg, h, emb)
            if cfg.down_attn[i]:
                h = unet.transformer(sd, f"down_blocks.{i}.attentions.{j}.", cfg, cfg.heads[i], h, ctx)
            skips.append(h)
            if taps is not None:
                taps[f"down.{i}.{j}"] = h
        if i != len(ch) - 1:
            p = f"down_blocks.{i}.downsamplers.0.conv."
            h = F.conv2d(h, sd[p + "weight"], sd[p + "bias"], stride=2, padding=1)
            skips.append(h)
    h = unet.resnet(sd, "mid_block.resnets.0.", cfg, h, emb)
    h = unet.transformer(sd, "mid_block.attentions.0.", cfg, cfg.heads[-1], h, ctx)
    h = unet.resnet(sd, "mid_block.resnets.1.", cfg, h, emb)
    if taps is not None:
        taps["mid"] = h
    if len(skips) != len(down_block_additional_residuals):
        raise ValueError(f"{len(down_block_additional_residuals)} down residuals for {len(skips)} skips")
    skips = [s + r for s, r in zip(skips, down_block_additional_residuals)]
    h = h + mid_block_additional_residual
    if taps is not None:
        taps.update({f"res.{k}": v for k, v in enumerate(skips)})
        taps["cn_mid"] = h
    rheads = list(reversed(cfg.heads))
    for i in range(len(ch)):
        for j in range(cfg.layers_per_block + 1):
            h = torch.cat([h, skips.pop()], dim=1)
            h = unet.resnet(sd, f"up_blocks.{i}.resnets.{j}.", cfg, h, emb)
            if cfg.up_attn[i]:
                h = unet.transformer(sd, f"up_blocks.{i}.attentions.{j}.", cfg, rheads[i], h, ctx)
            if taps is not None:
                taps[f"up.{i}.{j}"] = h
        if i != len(ch) - 1:
            p = f"up_blocks.{i}.upsamplers.0.conv."
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, sd[p + "weight"], sd[p + "bias"], padding=1)
    h = F.silu(F.group_norm(h, cfg.norm_groups, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], cfg.norm_eps))
    return F.conv2d(h, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


class ControlNetStreamOracle(StreamOracle):
    """StreamOracle with a ControlNet; every stream-batch slot is conditioned on the current frame's control image: with
    hed_sd (controlnet_processor_id="hed") the HED edge map of the frame (oracle/hed.py), without it (None) the frame itself,
    in [0,1], after the encoder's nearest resize."""

    def __init__(self, unet_sd, unet_cfg, vae_sd, controlnet_sd: Dict[str, torch.Tensor], t_index_list, width: int = 512,
                 height: int = 512, hed_sd: Optional[Dict[str, torch.Tensor]] = None, **kw):
        super().__init__(unet_sd, unet_cfg, vae_sd, t_index_list, width, height, **kw)
        self.controlnet_sd = controlnet_sd
        self.hed_sd = hed_sd
        self.control: Optional[torch.Tensor] = None

    def to(self, device, dtype: torch.dtype = torch.float32) -> "ControlNetStreamOracle":
        super().to(device, dtype)
        self.controlnet_sd = {k: v.to(device=self.device, dtype=dtype) for k, v in self.controlnet_sd.items()}
        if self.hed_sd is not None:
            self.hed_sd = {k: v.to(device=self.device, dtype=dtype) for k, v in self.hed_sd.items()}
        return self

    def unet_step(self, x: torch.Tensor):
        cn_taps: Dict[str, torch.Tensor] = {}
        res, mid = controlnet_forward(self.controlnet_sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds,
                                      self.control, cn_taps)
        taps: Dict[str, torch.Tensor] = {}
        eps = unet_forward(self.unet_sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds, res, mid, taps)
        self.last.update(cn_taps={k: v for k, v in cn_taps.items()}, unet_taps=taps)
        return self.scheduler_step_batch(eps, x), eps

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        img = image_preprocess(x.to(device=self.device, dtype=self.dtype), self.height, self.width, self.assume_unit_range)
        self.control = (img + 1.0) * 0.5
        if self.hed_sd is not None:
            self.control, self.last["control"] = hed.control_image(self.hed_sd, self.control)
        return super().__call__(x)


def make_weights(cfg: unet.UNetConfig, seed: int = 5678, zero_init: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded fp16 ControlNetModel state dict (oracle/weights.py's fan-in scaling).  The zero convs are drawn non-zero, like
    every other layer, so that the residuals reach the output; zero_init=True zeroes them and the conditioning embedding's
    conv_out, as in a freshly initialised ControlNet."""
    sd = ow._fill(param_shapes(cfg), seed, 0.5)
    if zero_init:
        for k in sd:
            if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.", "controlnet_cond_embedding.conv_out.")):
                sd[k] = torch.zeros_like(sd[k])
    return sd
