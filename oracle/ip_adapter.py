"""fp32 restatement of IP-Adapter (image prompts): ImageProjModel and the decoupled cross-attention

    out = softmax(Q Ktxt^T / sqrt(d)) Vtxt + scale * softmax(Q Kip^T / sqrt(d)) Vip,  Kip = tokens Wk_ip^T,  Vip = tokens Wv_ip^T

image_prompt() hooks it into the UNet oracle (oracle.unet, and through it the stream and ControlNet oracles): inside the
`with`, every cross-attention whose weight dict holds `to_k_ip.weight` / `to_v_ip.weight` beside `to_k` / `to_v` (the UNet's,
not the ControlNet's) adds the image term."""
from __future__ import annotations

import contextlib
from typing import Dict, Iterator

import torch
import torch.nn.functional as F

from . import unet


def image_proj(proj_w: torch.Tensor, proj_b: torch.Tensor, norm_w: torch.Tensor, norm_b: torch.Tensor,
               image_embeds: torch.Tensor) -> torch.Tensor:
    """ImageProjModel: (1, E) -> Linear -> (1, n_tok, D) -> LayerNorm (eps 1e-5), fp32"""
    D = norm_w.shape[0]
    t = F.linear(image_embeds.float().reshape(1, -1), proj_w.float(), proj_b.float())
    return F.layer_norm(t.reshape(1, -1, D), (D,), norm_w.float(), norm_b.float(), 1e-5)


def decoupled_attention(sd: Dict[str, torch.Tensor], p: str, heads: int, x: torch.Tensor, ctx: torch.Tensor,
                        tokens: torch.Tensor, scale: float) -> torch.Tensor:
    """attention_processor.Attention with IPAdapterAttnProcessor's image term, before to_out.0"""
    b, n, c = x.shape
    d = c // heads
    q = F.linear(x, sd[p + "to_q.weight"]).view(b, n, heads, d).transpose(1, 2)

    def attend(kv, wk, wv):
        k = F.linear(kv, sd[p + wk]).view(kv.shape[0], -1, heads, d).transpose(1, 2)
        v = F.linear(kv, sd[p + wv]).view(kv.shape[0], -1, heads, d).transpose(1, 2)
        s = torch.softmax((q @ k.transpose(-1, -2)) * (d ** -0.5), dim=-1)
        return (s @ v).transpose(1, 2).reshape(b, n, c)
    o = attend(ctx, "to_k.weight", "to_v.weight") + scale * attend(tokens.to(x.dtype), "to_k_ip.weight", "to_v_ip.weight")
    return F.linear(o, sd[p + "to_out.0.weight"], sd[p + "to_out.0.bias"])


@contextlib.contextmanager
def image_prompt(tokens: torch.Tensor, scale: float = 1.0) -> Iterator[None]:
    """Within the block the UNet oracle's cross-attentions with IP weights attend to `tokens` (1, n_tok, D) as well"""
    text_only = unet.attention

    def attention(sd, p, heads, x, ctx):
        if p + "to_k_ip.weight" not in sd:
            return text_only(sd, p, heads, x, ctx)
        return decoupled_attention(sd, p, heads, x, ctx, tokens.to(x.device), scale)
    unet.attention = attention
    try:
        yield
    finally:
        unet.attention = text_only
