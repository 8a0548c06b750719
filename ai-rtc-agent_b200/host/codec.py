"""Codec boundary of the frame path (SURVEY.md 8f-1).  The reference's aiortc fork decodes h264 with NVDEC and encodes with
NVENC (requirements.txt:12-13; env NVDEC / NVENC*, docs/environment.md:17-25) and exchanges RGB tensors in HBM with
lib/pipeline.py:50-51,83,96.  What exists here:

  * nv12_to_rgb / rgb_to_nv12: the colour conversions that sit between the fixed-function engines' NV12 surfaces and the
    engine's frame formats (u8 NHWC RGB in, u8 NCHW RGB out), as CUDA kernels behind the C ABI;
  * codec_libraries(): dlopen probe of libnvcuvid / libnvidia-encode.

What does not: decoder / encoder sessions.  Without those libraries and the Video Codec SDK headers, open_decoder /
open_encoder raise CodecUnavailable and the synthetic feeder stays the frame source -- stated, not silently faked."""
from __future__ import annotations

import torch

from . import capi

BT709, BT601, FULL_RANGE = 0, 1, 2


class CodecUnavailable(RuntimeError):
    pass


def codec_libraries() -> dict:
    mask = capi.lib().b2sd_codec_probe()
    return {"nvdec": bool(mask & 1), "nvenc": bool(mask & 2)}


def _need(kind: str, lib: str):
    have = codec_libraries()[kind]
    if not have:
        raise CodecUnavailable(f"codec unavailable: {lib} cannot be loaded on this machine (no {kind.upper()} session possible); "
                               "feed CUDA u8 NHWC tensors to the pipeline instead")
    raise CodecUnavailable(f"{lib} is present but this build has no session wrapper (Video Codec SDK headers were not available "
                           "to build against)")


def open_decoder(*_a, **_k):
    _need("nvdec", "libnvcuvid")


def open_encoder(*_a, **_k):
    _need("nvenc", "libnvidia-encode")


def nv12_to_rgb(y: torch.Tensor, uv: torch.Tensor, flags: int = BT709) -> torch.Tensor:
    """y: (H, pitch>=W) u8, uv: (H/2, pitch>=W) u8 interleaved Cb/Cr, both CUDA -> (1,H,W,3) u8 NHWC RGB."""
    h, w = y.shape[0], uv.shape[1] if uv.shape[1] <= y.shape[1] else y.shape[1]
    w = min(y.shape[1], uv.shape[1])
    out = torch.empty((1, h, w, 3), dtype=torch.uint8, device=y.device)
    capi.check(capi.lib().b2sd_op_nv12_to_rgb(y.data_ptr(), y.stride(0), uv.data_ptr(), uv.stride(0), out.data_ptr(), h, w, flags,
                                              capi.current_stream_ptr()), "b2sd_op_nv12_to_rgb")
    return out


def rgb_to_nv12(rgb_nchw: torch.Tensor, flags: int = BT709):
    """(1,3,H,W) u8 NCHW CUDA (what the pipeline returns) -> (Y (H,W), UV (H/2,W)) u8 planes."""
    _, _, h, w = rgb_nchw.shape
    y = torch.empty((h, w), dtype=torch.uint8, device=rgb_nchw.device)
    uv = torch.empty(((h + 1) // 2, (w + 1) // 2 * 2), dtype=torch.uint8, device=rgb_nchw.device)
    capi.check(capi.lib().b2sd_op_rgb_to_nv12(rgb_nchw.contiguous().data_ptr(), y.data_ptr(), y.stride(0), uv.data_ptr(), uv.stride(0),
                                              h, w, flags, capi.current_stream_ptr()), "b2sd_op_rgb_to_nv12")
    return y, uv
