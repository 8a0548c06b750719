"""fp32 restatement of controlnet_aux's `ControlNetHED_Apache2` and `HEDdetector` post-processing (the reference's default
ControlNet processor, lib/wrapper.py:40, 634-643).  [EXT] Recalled from the public upstream project, not verifiable offline;
the tests pin this restatement.

  * h = x - norm, x the RGB frame on the 0..255 scale (not / 255), norm a learned [1,3,1,1] offset (zero padding in h);
  * five DoubleConvBlocks, 3->64 (2 convs), 64->128 (2), 128->256 (3), 256->512 (3), 512->512 (3): 3x3 convs, pad 1, bias,
    ReLU; blocks 2-5 start with a 2x2/2 max-pool; each block's 1x1 `projection` to one channel is a side output;
  * HEDdetector: every side output resized to H x W with cv2.INTER_LINEAR (half-pixel centres: bilinear, align_corners=False),
    mean over the five, sigmoid, * 255, clip to [0, 255], truncation to u8 (safe=False, scribble=False);
  * the control image: the u8 map replicated to 3 channels, / 255.

Deviation: HEDdetector's own detect_resolution resampling (OpenCV area / cubic filters) is not reproduced; HED runs at the
engine's resolution on the frame after the encoder's nearest resize.  Test infrastructure only (see oracle/__init__)."""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.nn.functional as F

BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))   # (in, out, convs)


def side_outputs(sd: Dict[str, torch.Tensor], x255: torch.Tensor) -> List[torch.Tensor]:
    """x255: (1,3,H,W) on the 0..255 scale -> five (1,1,H/2^k,W/2^k) maps."""
    h = x255 - sd["norm"].reshape(1, 3, 1, 1)
    outs = []
    for b, (_, _, n) in enumerate(BLOCKS, start=1):
        if b > 1:
            h = F.max_pool2d(h, kernel_size=2, stride=2)
        for k in range(n):
            h = F.relu(F.conv2d(h, sd[f"block{b}.convs.{k}.weight"], sd[f"block{b}.convs.{k}.bias"], padding=1))
        outs.append(F.conv2d(h, sd[f"block{b}.projection.weight"].reshape(1, -1, 1, 1), sd[f"block{b}.projection.bias"]))
    return outs


def detect(sd: Dict[str, torch.Tensor], x255: torch.Tensor) -> torch.Tensor:
    """The u8 edge map (1,1,H,W)."""
    hh, ww = x255.shape[-2:]
    maps = [F.interpolate(o, size=(hh, ww), mode="bilinear", align_corners=False) for o in side_outputs(sd, x255)]
    e = torch.sigmoid(torch.stack(maps).mean(0))
    return (e * 255.0).clamp(0, 255).to(torch.uint8)


def control_image(sd: Dict[str, torch.Tensor], x01: torch.Tensor):
    """x01: (1,3,H,W) frame in [0,1] at the engine's size -> (1,3,H,W) control image in [0,1] and the u8 map."""
    u8 = detect(sd, x01 * 255.0)
    return (u8.float() / 255.0).repeat(1, 3, 1, 1), u8
