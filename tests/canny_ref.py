"""fp32 restatement of ControlNets on Canny edge maps, on top of tests/multi_controlnet_ref.py (oracle/controlnet.py stays as it
is): a net with processor "canny" reads oracle/canny.py's control image of the frame after the engine's resize, the frame as
u8 rint(frame * 255), computed once per frame with one threshold pair for every Canny net."""
from typing import Optional, Sequence

import numpy as np
import torch

from oracle import canny as ocanny
from oracle import hed
from oracle.stream import StreamOracle, image_preprocess
from tests.multi_controlnet_ref import MultiControlNetStreamOracle


def canny_control(frame01: torch.Tensor, low: float, high: float) -> torch.Tensor:
    """(1, 3, H, W) frame in [0, 1] -> (1, 3, H, W) control image (0 or 1) in the frame's dtype and device"""
    u8 = torch.round(frame01[0].float().clamp(0, 1) * 255).to(torch.uint8).permute(1, 2, 0).cpu().numpy()
    e = ocanny.control_image(u8, low, high)
    return torch.from_numpy(np.ascontiguousarray(e)).permute(2, 0, 1)[None].to(frame01) / 255.0


class CannyStreamOracle(MultiControlNetStreamOracle):
    """MultiControlNetStreamOracle whose processors may also be "canny"; `thresholds` is the frame's (low, high)"""

    def __init__(self, unet_sd, unet_cfg, vae_sd, controlnet_sds, processors: Sequence[Optional[str]], t_index_list,
                 width: int = 512, height: int = 512, hed_sd=None, **kw):
        super().__init__(unet_sd, unet_cfg, vae_sd, controlnet_sds, processors, t_index_list, width, height, hed_sd=hed_sd, **kw)
        self.thresholds = (100.0, 200.0)
        self.last_canny = None   # the last frame's Canny control image

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        img = image_preprocess(x.to(device=self.device, dtype=self.dtype), self.height, self.width, self.assume_unit_range)
        frame = (img + 1.0) * 0.5
        edge = canny = None
        if "hed" in self.processors:
            edge, self.last["control"] = hed.control_image(self.hed_sd, frame)
        if "canny" in self.processors:
            canny = self.last_canny = canny_control(frame, *self.thresholds)
        self.controls = [edge if p == "hed" else canny if p == "canny" else frame for p in self.processors]
        self.control = self.controls[0]
        return StreamOracle.__call__(self, x)
