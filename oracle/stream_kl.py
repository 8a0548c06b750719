"""StreamDiffusion with the model's own AutoencoderKL (use_tiny_vae=False): the StreamOracle of oracle/stream.py with the
TAESD encode / decode replaced by oracle/autoencoder_kl.py (the latent is scaling_factor times the mean of the encoder's
distribution; the decoder runs on x0 / scaling_factor), and the same on the GPU through torch's library kernels
(oracle/torch_gpu.py's `build`).  The VAE tensors of each frame are kept in `last` under the engine's tap names.  Test /
benchmark-baseline infrastructure only (see oracle/__init__)."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import autoencoder_kl as oakl
from . import controlnet as ocn
from . import unet as ounet
from .stream import StreamOracle, image_preprocess


class KLStreamOracle(StreamOracle):
    def __init__(self, *args, vae_kl: oakl.KLConfig = oakl.FULL, vae_scaling_factor: float = oakl.SCALING_FACTOR, **kw):
        super().__init__(*args, **kw)
        self.vae_kl, self.vae_scaling_factor = vae_kl, vae_scaling_factor

    def encode_image(self, image: torch.Tensor) -> torch.Tensor:
        z = oakl.encode_mean(self.vae_sd, image, self.vae_kl, self.last) * self.vae_scaling_factor
        return self.alpha_prod_t_sqrt[0] * z + self.beta_prod_t_sqrt[0] * self.init_noise[0]

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        img = image_preprocess(x.to(device=self.device, dtype=self.dtype), self.height, self.width, self.assume_unit_range)
        x_t = self.encode_image(img)
        x0 = self.predict_x0_batch(x_t)
        out = oakl.decode(self.vae_sd, x0 / self.vae_scaling_factor, self.vae_kl, self.last)
        self.last.update(x_t=x_t, x0=x0, image=out)
        return out


class KLControlNetStreamOracle(ocn.ControlNetStreamOracle, KLStreamOracle):
    """ControlNet conditioning (oracle/controlnet.py) with the AutoencoderKL: its __call__ derives the control image, then
    KLStreamOracle's runs the frame."""


def build(cfg: ounet.UNetConfig, unet_sd16: Dict[str, torch.Tensor], vae_sd16: Dict[str, torch.Tensor],
          t_index_list: List[int], hw: int, prompt_embeds: torch.Tensor, init_noise: Optional[torch.Tensor],
          dtype: torch.dtype = torch.float32, device: str = "cuda", width: Optional[int] = None,
          vae_kl: oakl.KLConfig = oakl.FULL) -> KLStreamOracle:
    """oracle/torch_gpu.py's `build` for a KLStreamOracle: on `device` in `dtype`, prepared like the engine (guidance 0.0, the
    engine's fp16-rounded noise); the frame is hw x hw, or hw high and `width` wide."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    orc = KLStreamOracle({k: v.float() for k, v in unet_sd16.items()}, cfg, {k: v.float() for k, v in vae_sd16.items()},
                         t_index_list, hw if width is None else width, hw, vae_kl=vae_kl)
    orc.prepare(prompt_embeds.float(), guidance_scale=0.0, init_noise=None if init_noise is None else init_noise.float())
    if init_noise is None:
        orc.init_noise = orc.init_noise.half().float()
    return orc.to(device, dtype)
