"""The oracle's restatement executed by torch's GPU library kernels (cuDNN convolutions, cuBLAS GEMMs, fused SDPA)
instead of CPU loops -- same functions (oracle/unet.py, taesd.py, stream.py), other device / dtype:

  * fp32 on the GPU (TF32 off): the full-size reference for configurations where the CPU oracle needs minutes per frame
    (SD-1.5 4-step at 512x512 and 768x768); tied to the CPU oracle by tests/test_thirdimpl_gpu.py at the tiny sizes;
  * fp16 on the GPU, optionally captured in a CUDA graph: what a plain torch/diffusers fp16 deployment of the reference
    computes (lib/wrapper.py:923-925 falls back to exactly that when TensorRT is missing).  It is the THIRD independent
    implementation SURVEY.md 8(c) states the u8 tolerance against, and `bench.py --impl library`'s baseline.

Test / benchmark-baseline infrastructure only: nothing under ai-rtc-agent_b200/ or lib/ may import this module."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import pipeline as opipe
from . import stream as ostream
from . import unet as ounet


def build(cfg: ounet.UNetConfig, unet_sd16: Dict[str, torch.Tensor], vae_sd16: Dict[str, torch.Tensor],
          t_index_list: List[int], hw: int, prompt_embeds: torch.Tensor, init_noise: Optional[torch.Tensor],
          dtype: torch.dtype = torch.float32, device: str = "cuda", width: Optional[int] = None) -> ostream.StreamOracle:
    """StreamOracle on `device` in `dtype`, prepared like the engine (guidance 0.0, the engine's fp16-rounded noise).
    The frame is hw x hw, or hw high and `width` wide."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    orc = ostream.StreamOracle({k: v.float() for k, v in unet_sd16.items()}, cfg, {k: v.float() for k, v in vae_sd16.items()},
                               t_index_list, hw if width is None else width, hw)
    orc.prepare(prompt_embeds.float(), guidance_scale=0.0, init_noise=None if init_noise is None else init_noise.float())
    if init_noise is None:
        orc.init_noise = orc.init_noise.half().float()
    return orc.to(device, dtype)


class fused_attention:
    """Context: route oracle.unet.attention through F.scaled_dot_product_attention (flash / mem-efficient kernels)."""

    def __enter__(self):
        self.prev = ounet.FUSED_ATTENTION
        ounet.FUSED_ATTENTION = True

    def __exit__(self, *a):
        ounet.FUSED_ATTENTION = self.prev
        return False


class GraphedFrame:
    """One frame (u8 NHWC in HBM -> u8 NCHW in HBM) of the torch-library path, captured once in a CUDA graph: the
    strongest configuration of the library baseline (no Python / launch overhead inside the timed region)."""

    def __init__(self, orc: ostream.StreamOracle, hw: int, use_graph: bool = True):
        self.orc = orc
        orc.assume_unit_range = True   # u8 frames are in [0,1] after /255: skips the image.min() host sync
        orc.static_buffers = True
        self.static_in = torch.zeros((1, hw, hw, 3), dtype=torch.uint8, device=orc.device)
        self.static_out = None
        self.graph = None
        self.use_graph = use_graph

    def _run(self):
        return opipe.frame_to_u8(self.orc, self.static_in)

    @torch.no_grad()
    def __call__(self, frame_u8_nhwc: torch.Tensor) -> torch.Tensor:
        self.static_in.copy_(frame_u8_nhwc, non_blocking=True)
        if not self.use_graph:
            with fused_attention():
                return self._run()
        if self.graph is None:
            with fused_attention():
                state = None if self.orc.x_t_latent_buffer is None else self.orc.x_t_latent_buffer.clone()
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for _ in range(3):   # warm-up (cuDNN algorithm selection) outside the capture
                        self._run()
                torch.cuda.current_stream().wait_stream(side)
                if state is not None:
                    self.orc.x_t_latent_buffer.copy_(state)   # the warm-up frames must not advance the stream batch
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self.static_out = self._run()
                if state is not None:
                    self.orc.x_t_latent_buffer.copy_(state)   # capture does not execute, but keep the invariant explicit
        self.graph.replay()
        return self.static_out
