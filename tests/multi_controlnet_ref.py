"""fp32 restatement of several ControlNets conditioning one stream (diffusers' MultiControlNetModel) on top of
oracle/controlnet.py, which it leaves as it is: each net reads its own control image (the frame's HED edge map, computed once,
or the frame itself), computes its residuals with controlnet_forward, scales them per slot, and the nets' residuals are summed
before the UNet adds them to its skips, skip + (r_0 + r_1 + ...), as diffusers does.  The engine chains the sums instead,
((skip + r_0) + r_1) + ..., which differs in rounding only."""
from typing import Dict, List, Optional, Sequence

import torch

from oracle import controlnet as ocn
from oracle import hed
from oracle.stream import StreamOracle, image_preprocess


class MultiControlNetStreamOracle(ocn.ControlNetStreamOracle):
    """ControlNetStreamOracle with nets controlnet_sds[i], each on the control image of processors[i] ("hed" or None) and
    scaled per slot by scales[i] (None: not scaled at all).  With one net and no scales it computes what
    ControlNetStreamOracle computes."""

    def __init__(self, unet_sd, unet_cfg, vae_sd, controlnet_sds: Sequence[Dict[str, torch.Tensor]],
                 processors: Sequence[Optional[str]], t_index_list, width: int = 512, height: int = 512,
                 hed_sd: Optional[Dict[str, torch.Tensor]] = None, **kw):
        super().__init__(unet_sd, unet_cfg, vae_sd, controlnet_sds[0], t_index_list, width, height, hed_sd=hed_sd, **kw)
        assert len(controlnet_sds) == len(processors) and ("hed" in processors) == (hed_sd is not None)
        self.controlnet_sds = list(controlnet_sds)
        self.processors = list(processors)
        self.scales: List[Optional[List[float]]] = [None] * len(self.controlnet_sds)
        self.controls: List[torch.Tensor] = []

    def to(self, device, dtype: torch.dtype = torch.float32) -> "MultiControlNetStreamOracle":
        super().to(device, dtype)
        self.controlnet_sds = [{k: v.to(device=self.device, dtype=dtype) for k, v in sd.items()} for sd in self.controlnet_sds]
        return self

    def unet_step(self, x: torch.Tensor):
        res_sum, mid_sum, nets = None, None, []
        for i, sd in enumerate(self.controlnet_sds):
            cn_taps: Dict[str, torch.Tensor] = {}
            res, mid = ocn.controlnet_forward(sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds, self.controls[i],
                                              cn_taps)
            if self.scales[i] is not None:
                s = torch.tensor(self.scales[i], dtype=mid.dtype, device=mid.device).view(-1, 1, 1, 1)
                res, mid = [r * s for r in res], mid * s
            nets.append(dict(cn_taps=cn_taps, res=res, mid=mid))
            res_sum = res if res_sum is None else [a + b for a, b in zip(res_sum, res)]
            mid_sum = mid if mid_sum is None else mid_sum + mid
        taps: Dict[str, torch.Tensor] = {}
        eps = ocn.unet_forward(self.unet_sd, self.cfg, x, self.sub_timesteps_tensor, self.prompt_embeds, res_sum, mid_sum, taps)
        self.last.update(cn_taps=dict(nets[0]["cn_taps"]), nets=nets, unet_taps=taps)
        return self.scheduler_step_batch(eps, x), eps

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        img = image_preprocess(x.to(device=self.device, dtype=self.dtype), self.height, self.width, self.assume_unit_range)
        frame = (img + 1.0) * 0.5
        edge = None
        if "hed" in self.processors:   # once per frame, whichever nets read it
            edge, self.last["control"] = hed.control_image(self.hed_sd, frame)
        self.controls = [edge if p == "hed" else frame for p in self.processors]
        self.control = self.controls[0]
        return StreamOracle.__call__(self, x)
