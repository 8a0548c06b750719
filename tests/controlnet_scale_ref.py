"""fp32 restatement of the ControlNet conditioning scale on top of oracle/controlnet.py (which it leaves as it is): each
stream-batch slot's residuals, every zero conv's output bias included, are multiplied by that slot's scale before the UNet adds
them to its skips, as diffusers' ControlNetModel.forward does with conditioning_scale."""
from typing import List, Optional

import torch

from oracle import controlnet as ocn


def controlnet_keep(n_steps: int, start: float, end: float) -> List[float]:
    """diffusers StableDiffusionControlNetPipeline.__call__'s controlnet_keep loop for one ControlNetModel, literally"""
    timesteps = list(range(n_steps))
    keep = []
    for i in range(len(timesteps)):
        keeps = [1.0 - float(i / len(timesteps) < s or (i + 1) / len(timesteps) > e) for s, e in zip([start], [end])]
        keep.append(keeps[0])
    return keep


class ScaledControlNetOracle(ocn.ControlNetStreamOracle):
    """ControlNetStreamOracle whose slot k's residuals are scaled by scales[k] (None: not scaled at all)"""

    scales: Optional[List[float]] = None

    def unet_step(self, x: torch.Tensor):
        cn_taps = {}
        res, mid = ocn.controlnet_forward(self.controlnet_sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds,
                                          self.control, cn_taps)
        if self.scales is not None:
            s = torch.tensor(self.scales, dtype=mid.dtype, device=mid.device).view(-1, 1, 1, 1)
            res, mid = [r * s for r in res], mid * s
        taps = {}
        eps = ocn.unet_forward(self.unet_sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds, res, mid, taps)
        self.last.update(cn_taps=cn_taps, unet_taps=taps)
        return self.scheduler_step_batch(eps, x), eps
