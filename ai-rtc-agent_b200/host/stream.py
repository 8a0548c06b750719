"""`StreamDiffusion` as the reference uses it (imported at lib/wrapper.py:20 from the un-vendored
yondonfu/StreamDiffusion@deepstream), re-implemented over libb200sd.so: the host-side bookkeeping
(LCM timestep table, per-slot scalars, seeded noise, prompt embedding, attributes that
lib/wrapper.py:389-407 pokes at) lives here in Python, everything per-frame runs in the engine.

Supported configuration = the one lib/pipeline.py:23-42 builds: img2img, use_denoising_batch=True,
frame_buffer_size=1, cfg_type "self"/"none" with guidance_scale <= 1.0 (no CFG arithmetic)."""
from __future__ import annotations

import ctypes as C
import math
import os
import weakref
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import capi
from .arch import UNetArch

NUM_TRAIN_TIMESTEPS = 1000
LCM_ORIGINAL_INFERENCE_STEPS = 50
LCM_TIMESTEP_SCALING = 10.0
LCM_SIGMA_DATA = 0.5


# ---- schedule tables (diffusers LCMScheduler with the SD scaled-linear betas) ---------------------------
def scaled_linear_alphas_cumprod(beta_start: float = 0.00085, beta_end: float = 0.012) -> torch.Tensor:
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, NUM_TRAIN_TIMESTEPS, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def lcm_timestep_table(num_inference_steps: int) -> List[int]:
    """LCMScheduler.set_timesteps(N): the 50 'origin' timesteps 19,39,..,999 walked backwards with stride
    50 // N.  N = 50 gives timesteps[i] = 999 - 20 i."""
    stride_train = NUM_TRAIN_TIMESTEPS // LCM_ORIGINAL_INFERENCE_STEPS
    origin = [(i + 1) * stride_train - 1 for i in range(LCM_ORIGINAL_INFERENCE_STEPS)]
    if num_inference_steps > LCM_ORIGINAL_INFERENCE_STEPS:
        raise ValueError("num_inference_steps cannot exceed the 50 LCM origin steps")
    step = LCM_ORIGINAL_INFERENCE_STEPS // num_inference_steps
    return list(reversed(origin))[::step][:num_inference_steps]


def lcm_boundary_scalings(timestep: int):
    scaled = timestep * LCM_TIMESTEP_SCALING
    denom = scaled * scaled + LCM_SIGMA_DATA * LCM_SIGMA_DATA
    return LCM_SIGMA_DATA * LCM_SIGMA_DATA / denom, scaled / denom ** 0.5


# ---- ControlNet conditioning scale and guidance window ----------------------------------------------------
DEFAULT_CONTROL = (1.0, 0.0, 1.0)   # (controlnet_conditioning_scale, control_guidance_start, control_guidance_end)


def check_control(scale: float, start: float = 0.0, end: float = 1.0) -> Tuple[float, float, float]:
    """(scale, start, end) as floats, with diffusers' checks (StableDiffusionControlNetPipeline.check_inputs): a finite
    scale (negative allowed), 0 <= start < end <= 1."""
    scale, start, end = float(scale), float(start), float(end)
    if not math.isfinite(scale):
        raise ValueError(f"controlnet_conditioning_scale must be finite (got {scale})")
    if start >= end:
        raise ValueError(f"control guidance start: {start} cannot be larger or equal to control guidance end: {end}")
    if start < 0.0:
        raise ValueError(f"control guidance start: {start} can't be smaller than 0")
    if end > 1.0:
        raise ValueError(f"control guidance end: {end} can't be larger than 1.0")
    return scale, start, end


def control_scales(control: Tuple[float, float, float], t_index_list: List[int], n_steps: int) -> List[float]:
    """The per-slot ControlNet scale of a stream batch: slot k stands for step t_index_list[k] of the n_steps-step timestep
    table, and is kept as diffusers' pipeline keeps step i of an n_steps-step run (controlnet_keep), times the scale."""
    scale, start, end = control
    return [scale * (0.0 if (i / n_steps < start or (i + 1) / n_steps > end) else 1.0) for i in t_index_list]


def check_controls(scale, start=0.0, end=1.0, nets: int = 1):
    """The settings of `nets` ControlNets, checked.  One net: check_control's (scale, start, end) floats.  Several: diffusers'
    MultiControlNetModel semantics (StableDiffusionControlNetPipeline.__call__ / check_inputs): a float scale applies to every
    net, a list has one per net; start / end may each be a float or a list, a float broadcast to the other's length (to
    `nets` when both are floats); then each (scale, start, end) is checked as for one net.  Returned as three tuples of
    length `nets`, (scales, starts, ends), so that set_control_scale(*settings) takes them back."""
    if nets == 1:
        return check_control(scale, start, end)
    seq = (list, tuple)
    if not isinstance(start, seq) and isinstance(end, seq):
        start = len(end) * [start]
    elif not isinstance(end, seq) and isinstance(start, seq):
        end = len(start) * [end]
    elif not isinstance(start, seq) and not isinstance(end, seq):
        start, end = nets * [start], nets * [end]
    if isinstance(scale, seq):
        if any(isinstance(v, seq) for v in scale):
            raise ValueError("A single batch of varying conditioning scale settings (e.g. [[1.0, 0.5], [0.2, 0.8]]) is not "
                             "supported at the moment. The conditioning scale must be fixed across the batch.")
        if len(scale) != nets:
            raise ValueError("For multiple controlnets: When `controlnet_conditioning_scale` is specified as `list`, it must "
                             "have the same length as the number of controlnets")
    else:
        scale = nets * [scale]
    if len(start) != len(end):
        raise ValueError(f"`control_guidance_start` has {len(start)} elements, but `control_guidance_end` has {len(end)} "
                         "elements. Make sure to provide the same number of elements to each list.")
    if len(start) != nets:
        raise ValueError(f"`control_guidance_start`: {list(start)} has {len(start)} elements but there are {nets} controlnets "
                         f"available. Make sure to provide {nets}.")
    return tuple(zip(*[check_control(v, a, b) for v, a, b in zip(scale, start, end)]))


DEFAULT_CANNY_THRESHOLDS = (100.0, 200.0)   # controlnet_aux CannyDetector's low_threshold / high_threshold


def check_canny_thresholds(low: float, high: float) -> Tuple[float, float]:
    """(low, high) as floats, finite (cv2.Canny swaps a reversed pair and floors both; so does the engine)"""
    low, high = float(low), float(high)
    if not (math.isfinite(low) and math.isfinite(high)):
        raise ValueError(f"Canny thresholds must be finite (got {low}, {high})")
    return low, high


def default_controls(nets: int):
    """The settings of `nets` ControlNets before any update: scale 1 over the whole run for each"""
    return DEFAULT_CONTROL if nets == 1 else tuple(nets * (v,) for v in DEFAULT_CONTROL)


def control_vector(control, t_index_list: List[int], n_steps: int) -> List[float]:
    """The per-slot scales of every net, [nets * batch], from settings as check_controls returns them: net i's row is
    control_scales of its own (scale, start, end)"""
    if isinstance(control[0], tuple):
        return [v for c in zip(*control) for v in control_scales(c, t_index_list, n_steps)]
    return control_scales(control, t_index_list, n_steps)


class ImageProcessor:
    """The part of diffusers' VaeImageProcessor the reference reaches (lib/wrapper.py:364)."""

    def __init__(self, vae_scale_factor: int = 8):
        self.vae_scale_factor = vae_scale_factor

    def preprocess(self, image, height: Optional[int] = None, width: Optional[int] = None) -> torch.Tensor:
        from PIL import Image
        if isinstance(image, Image.Image):
            if height and width and image.size != (width, height):
                image = image.resize((width, height), Image.LANCZOS)
            arr = np.asarray(image.convert("RGB"), dtype=np.float32) / 255.0
            image = torch.from_numpy(arr).permute(2, 0, 1)
        if isinstance(image, np.ndarray):
            image = torch.from_numpy(image)
        if image.dim() == 3:
            image = image.unsqueeze(0)
        if height and width and (image.shape[-2] != height or image.shape[-1] != width):
            image = torch.nn.functional.interpolate(image, size=(height, width))
        return image if image.min() < 0 else 2.0 * image - 1.0


class StreamDiffusion:
    styles = ()          # instances made by __init__ get a list (add_style)
    _is_style = False
    image_prompt = None  # the global image prompt: (host tokens [n_tok][D], scale) (set_image_tokens)
    control = DEFAULT_CONTROL   # the global ControlNet settings (check_controls; set_control_scale)
    has_controlnet = False      # built with a ControlNet (inherited by lanes and styles)
    control_nets = 1            # with has_controlnet: how many ControlNets (inherited by lanes and styles)
    has_canny = False           # a ControlNet's processor is "canny" (inherited by lanes and styles)
    canny_thresholds = DEFAULT_CANNY_THRESHOLDS   # the global Canny thresholds (set_canny_thresholds)

    def __init__(self, arch: UNetArch, unet_sd: Dict[str, torch.Tensor], vae_sd: Dict[str, torch.Tensor],
                 t_index_list: List[int], prompt_encoder: Callable[[str], torch.Tensor],
                 torch_dtype: torch.dtype = torch.float16, width: int = 512, height: int = 512,
                 do_add_noise: bool = True, use_denoising_batch: bool = True, frame_buffer_size: int = 1,
                 cfg_type: str = "self", device: str = "cuda", use_cuda_graph: bool = True,
                 packed_blob: Optional[str] = None, parent: Optional["StreamDiffusion"] = None,
                 controlnet_sd: Optional[Dict[str, torch.Tensor]] = None,
                 hed_sd: Optional[Dict[str, torch.Tensor]] = None, use_tiny_vae: bool = True,
                 vae_scaling_factor: float = 0.18215, live_lora: bool = False, style_of: Optional["StreamDiffusion"] = None,
                 ip_adapter=None, control_processors: Optional[List[Optional[str]]] = None):
        """vae_sd: TAESD (use_tiny_vae=True) or the model's own AutoencoderKL (use_tiny_vae=False: latents = vae_scaling_factor
        times the mean of the encoder's distribution, decoded from x0 / vae_scaling_factor).
        controlnet_sd: a diffusers ControlNetModel state dict (empty when the weights come from packed_blob); every
        stream-batch slot is then conditioned on the current frame's control image: the frame itself, or with hed_sd (a
        ControlNetHED.pth state dict, empty with packed_blob) its HED edge map.  Lanes inherit their parent's ControlNet.
        Several ControlNets (diffusers' MultiControlNetModel): controlnet_sd a list of 1..4 state dicts and control_processors
        one processor per net, "hed" (needs hed_sd; the edge map is computed once per frame), "canny" (cv2.Canny's edge map,
        computed once per frame; thresholds set_canny_thresholds) or None (the frame itself).  One state dict may take a
        control_processors list of one.
        live_lora: keep the base UNet weights on the device so that apply_lora() can switch LoRAs at run time (not with
        packed_blob; lanes inherit it).
        style_of: make a style of that live engine instead (add_style).
        ip_adapter: an image_prompt.IPAdapter (load_adapter): image prompts through the UNet's cross-attentions
        (set_image_tokens / update_image_prompt); lanes and styles inherit it."""
        if live_lora and packed_blob is not None:
            raise ValueError("live_lora needs the weights themselves: a packed blob does not carry the base weights")
        if hed_sd is not None and controlnet_sd is None:
            raise ValueError("the HED processor needs a ControlNet")
        nets_sd = controlnet_sd if isinstance(controlnet_sd, (list, tuple)) else None
        if nets_sd is not None or (controlnet_sd is not None and control_processors is not None):
            n = len(nets_sd) if nets_sd is not None else 1
            if not 1 <= n <= capi.MAX_CONTROLNETS:
                raise ValueError(f"1 to {capi.MAX_CONTROLNETS} ControlNets (got {n})")
            if control_processors is None or len(control_processors) != n:
                raise ValueError("control_processors needs one processor per ControlNet")
            for p in control_processors:
                if p not in capi.CONTROL_PROCESSORS:
                    raise NotImplementedError(f"ControlNet processor {p!r} (only 'hed', 'canny', or None: the frame itself)")
            if ("hed" in control_processors) != (hed_sd is not None):
                raise ValueError("hed_sd is needed exactly when a ControlNet's processor is 'hed'")
        elif control_processors is not None:
            raise ValueError("control_processors goes with a list of ControlNet state dicts")
        if frame_buffer_size != 1:
            raise NotImplementedError("frame_buffer_size > 1 is not on the reference's path (lib/pipeline.py:28)")
        if not use_denoising_batch:
            raise NotImplementedError("img2img mode must use denoising batch for now.")
        if torch_dtype != torch.float16:
            raise NotImplementedError("the sm_90a kernels compute in fp16 (fp32 accumulate) like the reference engines")
        self.arch = arch
        self.device = torch.device(device)
        self.dtype = torch_dtype
        self.generator = None
        self.height, self.width = height, width
        self.latent_height, self.latent_width = height // 8, width // 8
        self.frame_bff_size = frame_buffer_size
        self.denoising_steps_num = len(t_index_list)
        self.cfg_type = cfg_type
        self.use_denoising_batch = use_denoising_batch
        self.batch_size = self.denoising_steps_num * frame_buffer_size
        self.trt_unet_batch_size = self.batch_size  # cfg "self"/"none": no extra unconditional rows
        self.t_list = list(t_index_list)
        self.do_add_noise = do_add_noise
        self.similar_image_filter = False
        self.prev_image_result = None
        self.inference_time_ema = 0.0
        self._ev = None
        self.image_processor = ImageProcessor(8)
        self.prompt_encoder = prompt_encoder
        self.text_encoder = prompt_encoder
        self._handle = C.c_void_p()
        self._prepared = False
        self._lib = capi.lib()
        cfg = capi.EngineConfig()
        for i in range(4):
            cfg.block_out_channels[i] = arch.block_out_channels[i]
            cfg.heads[i] = arch.heads[i]
            cfg.down_attn[i] = arch.down_attn[i]
        cfg.cross_attention_dim = arch.cross_attention_dim
        cfg.layers_per_block = arch.layers_per_block
        cfg.norm_groups = arch.norm_groups
        cfg.ctx_tokens = arch.ctx_tokens
        cfg.batch = self.batch_size
        cfg.height, cfg.width = height, width
        cfg.do_add_noise = int(do_add_noise)
        cfg.use_cuda_graph = int(use_cuda_graph)
        cfg.controlnet = len(nets_sd) if nets_sd is not None else int(controlnet_sd is not None)
        self.has_controlnet = controlnet_sd is not None or (parent or style_of or self).has_controlnet
        self.control_nets = cfg.controlnet if controlnet_sd is not None else (parent or style_of or self).control_nets
        self.control = default_controls(self.control_nets)
        self.has_canny = "canny" in (control_processors or ()) or (parent or style_of or self).has_canny
        if control_processors is None:
            cfg.control_processor = capi.CONTROL_HED if hed_sd is not None else capi.CONTROL_FRAME
        else:
            procs = [capi.CONTROL_PROCESSORS[p] for p in control_processors]
            cfg.control_processor = procs[0]
            for i, p in enumerate(procs[1:]):
                cfg.control_processor_more[i] = p
        cfg.vae = capi.VAE_TINY if use_tiny_vae else capi.VAE_KL
        cfg.vae_scaling_factor = 0.0 if use_tiny_vae else float(vae_scaling_factor)
        cfg.ip_tokens = ip_adapter.n_tok if ip_adapter is not None else 0
        self.ip_adapter = ip_adapter   # with packed_blob its UNet weights come from the blob
        if not torch.cuda.is_available():
            raise capi.B2Error("no CUDA device: the H100 pipeline has no CPU fallback")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        torch.cuda.set_device(self.device)
        self._ctor = dict(torch_dtype=torch_dtype, width=width, height=height, do_add_noise=do_add_noise,
                          use_denoising_batch=use_denoising_batch, frame_buffer_size=frame_buffer_size, cfg_type=cfg_type,
                          device=device, use_cuda_graph=use_cuda_graph, use_tiny_vae=use_tiny_vae,
                          vae_scaling_factor=vae_scaling_factor, live_lora=live_lora, ip_adapter=ip_adapter)
        self.live_lora = bool(live_lora)
        # extra engines over this one's weights (add_lane).  A lane keeps no reference to its parent: an engine and its lanes then
        # form no reference cycle, so their device memory is released as soon as the last reference goes, not at the next
        # run of the garbage collector
        self.lanes: List["StreamDiffusion"] = []
        # styles of this engine's weights (add_style); like lanes they keep no reference to it
        self.styles: List["StreamDiffusion"] = []
        self._is_style = style_of is not None
        # live StreamStates of the engine, its lanes and its styles: any of them may step any of these states
        family = parent if parent is not None else style_of
        self._states = family._states if family is not None else weakref.WeakSet()
        if style_of is not None:
            # a style: the UNet weights of style_of's base plus LoRAs of its own (apply_lora), everything else shared
            capi.check(self._lib.b2sd_create_style(style_of._handle, C.byref(self._handle)), "b2sd_create_style")
            self._unet_shapes = style_of._unet_shapes
            return
        if parent is not None:
            # a lane: shares the parent's weights in HBM, owns its activations / stream state / CUDA graph
            capi.check(self._lib.b2sd_create_lane(parent._handle, C.byref(cfg), C.byref(self._handle)), "b2sd_create_lane")
            return
        capi.check(self._lib.b2sd_create(C.byref(cfg), C.byref(self._handle)), "b2sd_create")
        if live_lora:
            capi.check(self._lib.b2sd_set_live_params(self._handle, 1), "b2sd_set_live_params")
            self._unet_shapes = {k: tuple(v.shape) for k, v in unet_sd.items()}
        if packed_blob is not None:
            # kernel-native weights written by export_packed() / `python -m ai_rtc_agent_b200.pack`: no state dicts, no repacking
            capi.check(self._lib.b2sd_import_packed(self._handle, os.fsencode(packed_blob)), f"b2sd_import_packed({packed_blob})")
        else:
            self._load("", unet_sd)
            if ip_adapter is not None:
                self._load("", ip_adapter.unet)
            self._load("vae.", vae_sd)
            for i, sd in enumerate(nets_sd if nets_sd is not None else [controlnet_sd or {}]):
                self._load("controlnet." if i == 0 else f"controlnet{i}.", sd)
            self._load("hed.", hed_sd or {})

    # the reference reaches the UNet and the VAE as `stream.unet` / `stream.vae`; both are this engine.  Properties, not attributes
    # holding self: a self-reference would keep every engine's device memory until the garbage collector runs
    @property
    def unet(self) -> "StreamDiffusion":
        return self

    @property
    def vae(self) -> "StreamDiffusion":
        return self

    def set_concurrency(self, frames_in_flight: int) -> None:
        """Tell the engine how many frames will be in flight on this GPU (before prepare()): > 1 selects the throughput
        launch policy (b2sd_set_concurrency)."""
        capi.check(self._lib.b2sd_set_concurrency(self._handle, int(frames_in_flight)), "b2sd_set_concurrency")
        self._prepared = False

    def export_packed(self, path: str) -> None:
        """Write the packed-weight blob (after prepare()); the engine-file cache of lib/wrapper.py:593-597, 896-910."""
        self._check()
        tmp = f"{path}.tmp{os.getpid()}"
        capi.check(self._lib.b2sd_export_packed(self._handle, os.fsencode(tmp)), f"b2sd_export_packed({path})")
        os.replace(tmp, path)   # atomic: a concurrently starting replica never sees a half-written blob

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.b2sd_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass

    def _load(self, prefix: str, sd: Dict[str, torch.Tensor]) -> None:
        for key, t in sd.items():
            t = t.detach()
            if t.dtype not in (torch.float16, torch.float32):
                t = t.float()
            t = t.contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            capi.check(self._lib.b2sd_load_tensor(self._handle, (prefix + key).encode(), t.data_ptr(),
                                                  0 if t.dtype == torch.float16 else 1, shape, t.dim()),
                       f"b2sd_load_tensor({prefix + key})")

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ---- StreamDiffusion.prepare --------------------------------------------------------------------
    @torch.no_grad()
    def prepare(self, prompt: str, negative_prompt: str = "", num_inference_steps: int = 50,
                guidance_scale: float = 1.2, delta: float = 1.0,
                generator: Optional[torch.Generator] = None, seed: int = 2) -> None:
        self.generator = generator if generator is not None else torch.Generator()
        self.generator.manual_seed(seed)
        self.guidance_scale = 1.0 if self.cfg_type == "none" else guidance_scale
        if self.guidance_scale > 1.0:
            raise NotImplementedError("classifier-free guidance (guidance_scale > 1) is not on the reference's path "
                                      "(lib/pipeline.py:14 passes 0.0)")
        self.delta = delta
        T = self.denoising_steps_num
        self.prompt = prompt
        self.prompt_embeds = self._encode(prompt).repeat(self.batch_size, 1, 1)
        self.timesteps = lcm_timestep_table(num_inference_steps)
        self.sub_timesteps = [self.timesteps[t] for t in self.t_list]
        self.sub_timesteps_tensor = torch.tensor(self.sub_timesteps, dtype=torch.long, device=self.device)
        self.sub_timesteps_tensor = torch.repeat_interleave(self.sub_timesteps_tensor, repeats=self.frame_bff_size, dim=0)
        self.init_noise = torch.randn((self.batch_size, 4, self.latent_height, self.latent_width),
                                      generator=self.generator).to(dtype=self.dtype)
        self.stock_noise = torch.zeros_like(self.init_noise)
        scal = [lcm_boundary_scalings(t) for t in self.sub_timesteps]
        ac = scaled_linear_alphas_cumprod()
        f16 = lambda v: torch.tensor(v, dtype=torch.float32).to(self.dtype)  # the reference keeps these in fp16
        self.c_skip = f16([s[0] for s in scal]).view(T, 1, 1, 1)
        self.c_out = f16([s[1] for s in scal]).view(T, 1, 1, 1)
        self.alpha_prod_t_sqrt = torch.stack([ac[t].sqrt() for t in self.sub_timesteps]).to(self.dtype).view(T, 1, 1, 1)
        self.beta_prod_t_sqrt = torch.stack([(1 - ac[t]).sqrt() for t in self.sub_timesteps]).to(self.dtype).view(T, 1, 1, 1)
        self._engine_prepare()
        for lane in self._family()[1:]:
            lane._prepare_like(self)
        for state in list(self._states):   # as prepare zeroes the engines' own latent buffers, and follows its conditioning
            if not state.closed:
                state.reset()
                state.clear_overrides()

    _SCHEDULE_ATTRS = ("generator", "guidance_scale", "delta", "prompt", "prompt_embeds", "timesteps", "sub_timesteps", "sub_timesteps_tensor",
                       "init_noise", "stock_noise", "c_skip", "c_out", "alpha_prod_t_sqrt", "beta_prod_t_sqrt")

    def _engine_prepare(self) -> None:
        coef = torch.stack([self.alpha_prod_t_sqrt.flatten(), self.beta_prod_t_sqrt.flatten(),
                            self.c_skip.flatten(), self.c_out.flatten()]).float().contiguous()
        tsteps = torch.tensor(self.sub_timesteps, dtype=torch.float32)
        emb = self.prompt_embeds[0].to(torch.float16).cpu().contiguous()
        noise = self.init_noise.cpu().contiguous()
        capi.check(self._lib.b2sd_prepare(self._handle, emb.data_ptr(), tsteps.data_ptr(), coef.data_ptr(),
                                          noise.data_ptr(), self._stream()), "b2sd_prepare")
        self._push_control()
        self._prepared = True

    def _push_control(self) -> None:
        """This engine's global per-slot ControlNet scales from self.control and self.t_list (b2sd_set_control_scale, with
        several nets b2sd_set_control_scales)"""
        if self.has_controlnet:
            v = torch.tensor(control_vector(self.control, self.t_list, len(self.timesteps)), dtype=torch.float32)
            fn = "b2sd_set_control_scale" if self.control_nets == 1 else "b2sd_set_control_scales"
            capi.check(getattr(self._lib, fn)(self._handle, v.data_ptr(), self._stream()), fn)

    def _prepare_like(self, other: "StreamDiffusion") -> None:
        for name in self._SCHEDULE_ATTRS:
            setattr(self, name, getattr(other, name))
        self.t_list = list(other.t_list)
        self.control = other.control
        self._engine_prepare()
        if self.has_canny:   # a new lane or style starts with the family's global thresholds
            self.canny_thresholds = other.canny_thresholds
            capi.check(self._lib.b2sd_set_canny_thresholds(self._handle, *self.canny_thresholds), "b2sd_set_canny_thresholds")
        if other.image_prompt is not None:   # a new lane or style starts with the family's global image prompt
            tokens, scale = other.image_prompt
            capi.check(self._lib.b2sd_set_image_embeds(self._handle, tokens.data_ptr(), tokens.shape[0], scale, self._stream()),
                       "b2sd_set_image_embeds")
            self.image_prompt = other.image_prompt

    def add_lane(self) -> "StreamDiffusion":
        """Another engine over the same weights, prepared identically (same prompt embedding, schedule and seed-2 noise):
        frames may be alternated between this engine and its lanes on different CUDA streams.  Later prepare() /
        update_prompt() / timestep updates on this object reach every lane.  Stepped without a state, the lane is an
        independent temporal stream (or, for a 1-step stream batch, simply the next frame); to continue one stream with T > 1
        on several lanes, step one new_state() on each in turn."""
        self._check()
        lane = StreamDiffusion(self.arch, {}, {}, self.t_list, self.prompt_encoder, parent=self, **self._ctor)
        lane._prepare_like(self)
        self.lanes.append(lane)
        return lane

    def add_style(self) -> "StreamDiffusion":
        """A style of this live engine (b2sd_create_style): an engine whose UNet is this engine's base weights plus LoRAs of its
        own (its apply_lora), sharing every other weight with it, prepared like this engine on the current CUDA stream.  Give
        it lanes with its add_lane().  Later prepare() / update_prompt() / timestep updates on this object reach the style and
        its lanes; apply_lora() on this object does not.  Every state of this engine's weights may be stepped by the style's
        engines, but a state's own prompt / t_index_list must be set again on a style engine before it steps there.  Free the
        style with drop_style()."""
        self._check()
        if not self.live_lora or self._is_style:
            raise RuntimeError("add_style needs a live_lora engine that is not itself a style")
        style = StreamDiffusion(self.arch, {}, {}, self.t_list, self.prompt_encoder, style_of=self, **self._ctor)
        style._prepare_like(self)
        self.styles.append(style)
        return style

    def drop_style(self, style: "StreamDiffusion", after: "torch.cuda.Stream") -> None:
        """Free a style of this engine and its lanes after the work queued on `after` (which the caller makes wait for their
        last frames), stream-ordered: no host or device synchronisation (b2sd_release)."""
        self.styles.remove(style)
        for eng in [style] + style.lanes:
            if eng._handle.value:
                h, eng._handle = eng._handle, C.c_void_p()
                capi.check(self._lib.b2sd_release(h, after.cuda_stream), "b2sd_release")
        style.lanes = []

    def _family(self) -> List["StreamDiffusion"]:
        """this engine, its lanes, its styles and their lanes: every engine a global prompt / timestep update reaches"""
        return [self] + self.lanes + [e for st in self.styles for e in [st] + st.lanes]

    def new_state(self) -> "StreamState":
        """A fresh temporal stream (zeroed x_t_latent_buffer) that this engine and every lane of its weights can step:
        pass it as `state=` to step_u8 / step_u8_into / __call__.  prepare() resets it."""
        self._check()
        state = StreamState(self)
        self._states.add(state)
        return state

    _enc_stream = None

    def _encoder_stream(self):
        """the CUDA stream per-state prompts are encoded on (_encode_beside)"""
        if self._enc_stream is None:
            self._enc_stream = torch.cuda.Stream(self.device)
        return self._enc_stream

    def _encode(self, prompt: str) -> torch.Tensor:
        e = self.prompt_encoder(prompt)
        if e.dim() == 2:
            e = e.unsqueeze(0)
        if e.shape[-2] != self.arch.ctx_tokens or e.shape[-1] != self.arch.cross_attention_dim:
            raise ValueError(f"prompt embedding shape {tuple(e.shape)} != (1,{self.arch.ctx_tokens},{self.arch.cross_attention_dim})")
        return e.to(torch.float16)

    @torch.no_grad()
    def update_prompt(self, prompt: str) -> None:
        """The global prompt: this engine's, its lanes' and every live state's (a state's own prompt is dropped)."""
        self.prompt = prompt
        self.prompt_embeds = self._encode(prompt).repeat(self.batch_size, 1, 1)
        emb = self.prompt_embeds[0].cpu().contiguous()
        for eng in self._family():
            eng.prompt, eng.prompt_embeds = prompt, self.prompt_embeds
            capi.check(self._lib.b2sd_set_prompt_embeds(eng._handle, emb.data_ptr(), self._stream()), "b2sd_set_prompt_embeds")
        self.clear_overrides(prompt=True, t_index_list=False, image_prompt=False)

    def image_tokens(self, image) -> torch.Tensor:
        """(1, n_tok, D) fp16 image-prompt tokens of `image` (a PIL image or HWC uint8 array / tensor): the adapter's image encoder
        (set by the pipeline; a seeded synthetic one otherwise), then its projection"""
        if self.ip_adapter is None:
            raise RuntimeError("this engine was built without an IP-Adapter (ip_adapter=...)")
        enc = getattr(self, "image_encoder", None)
        if enc is None:
            from .image_prompt import SyntheticImageEncoder
            enc = self.image_encoder = SyntheticImageEncoder(self.ip_adapter.embed_dim)
        return self.ip_adapter.tokens(enc(image))

    @torch.no_grad()
    def set_image_tokens(self, tokens: Optional[torch.Tensor], scale: float = 1.0) -> None:
        """The global image prompt as (1, n_tok, D) fp16 tokens (image_tokens), None to clear: this engine's, its lanes' and its
        styles' (b2sd_set_image_embeds), and every live state's (a state's own image prompt is dropped, its own prompt kept)."""
        ptr, n = 0, 0
        if tokens is not None:
            tokens = tokens.reshape(-1, self.arch.cross_attention_dim).to(torch.float16).cpu().contiguous()
            ptr, n = tokens.data_ptr(), tokens.shape[0]
        for eng in self._family():
            capi.check(self._lib.b2sd_set_image_embeds(eng._handle, ptr or None, n, float(scale), self._stream()),
                       "b2sd_set_image_embeds")
        self.image_prompt = None if tokens is None else (tokens, float(scale))
        self.clear_overrides(prompt=False, t_index_list=False, image_prompt=True)

    def _timestep_tensor(self, sub_timesteps: List[int]) -> torch.Tensor:
        t = torch.tensor([float(v) for v in sub_timesteps], dtype=torch.float32)
        if t.numel() != self.batch_size:
            raise ValueError(f"t_index_list length {t.numel()} != stream batch {self.batch_size} (static batch, as the "
                             "reference's TensorRT engines)")
        return t

    def sync_timesteps(self) -> None:
        """Push self.sub_timesteps to the engine (called after lib/wrapper.py:389-407 style updates).  As in the
        reference only the timestep embedding changes; alpha/beta/c_skip/c_out keep their prepare() values.  Every live
        state's own t_index_list is dropped."""
        t = self._timestep_tensor(self.sub_timesteps)
        for eng in self._family():
            eng.t_list, eng.sub_timesteps, eng.sub_timesteps_tensor = self.t_list, self.sub_timesteps, self.sub_timesteps_tensor
            capi.check(self._lib.b2sd_set_timesteps(eng._handle, t.data_ptr(), self._stream()), "b2sd_set_timesteps")
            eng._push_control()   # the slots are masked with the new list
        self.clear_overrides(prompt=False, t_index_list=True)

    @torch.no_grad()
    def set_control_scale(self, scale: float, start: float = 0.0, end: float = 1.0) -> None:
        """The global ControlNet settings (diffusers' controlnet_conditioning_scale, control_guidance_start / _end): this
        engine's, its lanes' and its styles' (b2sd_set_control_scale), and every live state's (a state's own settings are
        dropped, its own t_index_list kept).  Slot k of the stream batch is conditioned with scale times diffusers'
        controlnet_keep of step t_index_list[k] of the len(self.timesteps)-step table (control_scales).  With several
        ControlNets each argument may be a float (every net) or a list (one per net), as check_controls takes them.  The
        settings are checked before anything changes; on the current CUDA stream, after the frames queued there."""
        if not self.has_controlnet:
            raise RuntimeError("this engine was built without a ControlNet")
        control = check_controls(scale, start, end, self.control_nets)
        for eng in self._family():
            eng.control = control
            eng._push_control()
        for state in list(self._states):
            if not state.closed:
                state.clear_overrides(prompt=False, t_index_list=False, control=True)

    def set_canny_thresholds(self, low: float = 100.0, high: float = 200.0) -> None:
        """The global Canny thresholds (cv2.Canny's threshold1 / threshold2): this engine's, its lanes' and its styles'
        (b2sd_set_canny_thresholds), and every live state's (a state's own thresholds are dropped).  Host values that the next
        steps pass to the Canny kernel: frames submitted before the call keep the old ones; no device work, no synchronisation."""
        if not self.has_canny:
            raise RuntimeError("this engine has no ControlNet with the 'canny' processor")
        low, high = check_canny_thresholds(low, high)
        for eng in self._family():
            capi.check(self._lib.b2sd_set_canny_thresholds(eng._handle, low, high), "b2sd_set_canny_thresholds")
            eng.canny_thresholds = (low, high)
        for state in list(self._states):
            if not state.closed:
                state.clear_canny_thresholds()

    def clear_overrides(self, prompt: bool = True, t_index_list: bool = True, image_prompt: Optional[bool] = None) -> None:
        """Every live state of this engine's weights follows the global prompt, t_index_list and / or image prompt again
        (image_prompt: default with the prompt)."""
        for state in list(self._states):
            if not state.closed:
                state.clear_overrides(prompt=prompt, t_index_list=t_index_list, image_prompt=image_prompt)

    @torch.no_grad()
    def apply_lora(self, lora_dict: Optional[Dict[str, float]]) -> None:
        """Switch the style LoRAs (live_lora engines): from now on the UNet computes with the base weights plus the LoRAs of
        lora_dict ({safetensors path: scale}, fused in order, as the constructor's lora_dict would have; None / {}: the base).
        The files are read and every pair checked before anything changes on the device.  The weights are re-fused on the
        device on the current CUDA stream, then the conditioning of this engine, its lanes and every live state (its own prompt
        / t_index_list included) is recomputed with them; the caller orders the stream after the frames in flight and before
        later ones.  No host synchronisation besides the upload of the factors and the prompt encoder's own."""
        from .weights import lora_factors
        if not self.live_lora:
            raise RuntimeError("apply_lora needs an engine built with live_lora=True (StreamDiffusionPipeline(live_lora=True) or "
                               "$B200SD_LIVE_LORA=1)")
        self._check()
        self.apply_factors(lora_factors(self._unet_shapes, lora_dict))

    @torch.no_grad()
    def apply_factors(self, factors) -> None:
        """apply_lora with the factors weights.lora_factors made from a lora_dict (checked already).  On a style only the style's
        engines are refreshed: the states stepped on it have their own prompt / t_index_list set again by whoever moves them."""
        keep = []   # the device factors stay referenced until the call has enqueued the work that reads them
        arr = (capi.LoraFactor * max(1, len(factors)))()
        for i, (key, up, down, scale) in enumerate(factors):
            up, down, scale = _factor_operands(up, down, scale)
            up, down = _on_device(up, self.device), _on_device(down, self.device)
            keep += [up, down]
            arr[i] = capi.LoraFactor(key.encode(), up.data_ptr(), down.data_ptr(), up.shape[1],
                                     0 if up.dtype == torch.float16 else 1, scale)
        capi.check(self._lib.b2sd_apply_lora(self._handle, len(factors), arr, self._stream()), "b2sd_apply_lora")
        for eng in [self] + self.lanes:
            capi.check(self._lib.b2sd_refresh_conditioning(eng._handle, self._stream()), "b2sd_refresh_conditioning")
        if self._is_style:
            return
        for state in list(self._states):
            if state.closed:
                continue
            if state.own_prompt is not None:
                state.set_prompt(state.own_prompt, engine=self)
            if state.own_image is not None:
                state.set_image_tokens(*state.own_image, engine=self)
            if state.own_t_index_list is not None:
                state.set_t_index_list(state.own_t_index_list, engine=self)
            elif state.own_control is not None:
                state.set_control_scale(*state.own_control, engine=self)

    def conditioning_binds(self) -> int:
        """How many conditioning block copies this engine's steps have issued (b2sd_conditioning_binds).  Test aid."""
        return self._lib.b2sd_conditioning_binds(self._handle)

    # ---- per frame ---------------------------------------------------------------------------------
    def _check(self):
        if not self._prepared:
            raise RuntimeError("StreamDiffusion.prepare() must be called before frames are processed")

    def _step(self, frame_ptr: int, in_kind: int, in_h: int, in_w: int, out_ptr: int, out_kind: int,
              state: Optional["StreamState"]) -> None:
        if state is None:
            capi.check(self._lib.b2sd_step_ex(self._handle, frame_ptr, in_kind, in_h, in_w, out_ptr, out_kind, self._stream()),
                       "b2sd_step_ex")
        else:
            capi.check(self._lib.b2sd_step_state(self._handle, state.handle, frame_ptr, in_kind, in_h, in_w, out_ptr, out_kind,
                                                 self._stream()), "b2sd_step_state")

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, state: Optional["StreamState"] = None) -> torch.Tensor:
        """x: (3,H',W') or (1,3,H',W') float tensor in [0,1] on the GPU -> (1,3,H,W) fp16 image in ~[-1,1].
        state: step that stream state (new_state) instead of this engine's own."""
        self._check()
        if x.dim() == 3:
            x = x.unsqueeze(0)
        if x.dtype == torch.float32:
            kind = capi.IN_F32_NCHW
        elif x.dtype == torch.float16:
            kind = capi.IN_F16_NCHW
        else:
            raise TypeError(f"unsupported image dtype {x.dtype}")
        x = x.to(self.device)
        # VaeImageProcessor.preprocess (re-run inside the reference's StreamDiffusion.__call__): an image that already has
        # negative values is taken as [-1,1] and NOT normalised again; the encoder's own (x+1)/2 then brings it to [0,1],
        # which is the range the engine's head expects.  Same host sync (`image.min()`) as the reference; the fused u8 entry
        # (step_u8, what lib/pipeline.py's __call__ uses) never comes through here.
        if bool(x.min() < 0):
            x = x * 0.5 + 0.5
        x = x.contiguous()
        out = torch.empty((1, 3, self.height, self.width), dtype=torch.float16, device=self.device)
        t0 = self._tick()
        self._step(x.data_ptr(), kind, x.shape[-2], x.shape[-1], out.data_ptr(), capi.OUT_F16_NCHW, state)
        self._tock(t0)
        self.prev_image_result = out
        return out

    # ---- inference_time_ema (StreamDiffusion.__call__ times every frame with CUDA events and keeps
    # ema = 0.9 ema + 0.1 dt; external code reads the attribute).  The reference pays a device-wide synchronize per frame for
    # it; here the events are read one frame late, so nothing on the path blocks.
    def _tick(self):
        if self._ev is None:
            self._ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(2)]
            self._ev_pending = None
            self._ev_idx = 0
        if self._ev_pending is not None:
            e0, e1 = self._ev_pending
            if e1.query():
                self.inference_time_ema = 0.9 * self.inference_time_ema + 0.1 * (e0.elapsed_time(e1) / 1000.0)
                self._ev_pending = None
        if self._ev_pending is not None:
            return None            # previous frame still in flight: skip this sample rather than wait
        pair = self._ev[self._ev_idx]
        self._ev_idx ^= 1
        pair[0].record(torch.cuda.current_stream(self.device))
        return pair

    def _tock(self, pair):
        if pair is not None:
            pair[1].record(torch.cuda.current_stream(self.device))
            self._ev_pending = pair

    @torch.no_grad()
    def step_u8(self, frame_nhwc: torch.Tensor, state: Optional["StreamState"] = None) -> torch.Tensor:
        """Fused fast path of lib/pipeline.py:76-96: u8 NHWC (1,H',W',3) CUDA tensor in, u8 NCHW (1,3,H,W) out,
        one engine call, no intermediate tensors.  state: step that stream state (new_state) instead of this engine's own."""
        self._check()
        if frame_nhwc.dtype != torch.uint8 or frame_nhwc.dim() != 4 or frame_nhwc.shape[-1] != 3 or not frame_nhwc.is_cuda:
            raise TypeError("expected a CUDA uint8 tensor shaped (1,H,W,3)")
        frame_nhwc = frame_nhwc.contiguous()
        out = torch.empty((1, 3, self.height, self.width), dtype=torch.uint8, device=self.device)
        t0 = self._tick()
        self._step(frame_nhwc.data_ptr(), capi.IN_U8_NHWC, frame_nhwc.shape[1], frame_nhwc.shape[2], out.data_ptr(),
                   capi.OUT_U8_NCHW, state)
        self._tock(t0)
        return out

    def step_u8_into(self, frame_nhwc: torch.Tensor, out: torch.Tensor, state: Optional["StreamState"] = None) -> torch.Tensor:
        self._step(frame_nhwc.data_ptr(), capi.IN_U8_NHWC, frame_nhwc.shape[1], frame_nhwc.shape[2], out.data_ptr(),
                   capi.OUT_U8_NCHW, state)
        return out

    def get_tensor(self, name: str) -> torch.Tensor:
        """Debug/parity tap of the last step as an fp16 NHWC CPU tensor."""
        n = C.c_int64()
        dims = (C.c_int * 4)()
        capi.check(self._lib.b2sd_get_tensor(self._handle, name.encode(), None, 0, C.byref(n), dims, self._stream()),
                   "b2sd_get_tensor")
        t = torch.empty(tuple(dims), dtype=torch.float16)
        capi.check(self._lib.b2sd_get_tensor(self._handle, name.encode(), t.data_ptr(), n.value, C.byref(n), dims,
                                             self._stream()), "b2sd_get_tensor")
        return t

    def profile(self, frame_nhwc: torch.Tensor, iters: int = 5):
        """Per-launch device times of one frame (eager replay, CUDA events): list of {"name", "ms"}."""
        import json
        self._check()
        out = torch.empty((1, 3, self.height, self.width), dtype=torch.uint8, device=self.device)
        buf = C.create_string_buffer(1 << 20)
        capi.check(self._lib.b2sd_profile(self._handle, frame_nhwc.data_ptr(), frame_nhwc.shape[1], frame_nhwc.shape[2],
                                          out.data_ptr(), iters, buf, len(buf), self._stream()), "b2sd_profile")
        return json.loads(buf.value.decode())

    def profile_kind(self, kind: str, iters: int = 20):
        """Device time of one launch class inside a CUDA graph (only those launches, program order):
        {"ms": per replay, "launches": n, "flops": algorithmic FLOPs per replay}."""
        self._check()
        ms, n, fl = C.c_double(), C.c_int(), C.c_double()
        capi.check(self._lib.b2sd_profile_kind(self._handle, kind.encode(), iters, C.byref(ms), C.byref(n), C.byref(fl),
                                               self._stream()), "b2sd_profile_kind")
        return {"ms": ms.value, "launches": n.value, "flops": fl.value}

    @torch.no_grad()
    def audit_step(self, frame_nhwc: torch.Tensor, fn: Callable[[int, bool, "capi.LaunchRecord"], None]) -> torch.Tensor:
        """step_u8 with the frame program run eagerly and fn(index, after, record) called before and after every kernel launch,
        with the stream synchronised (b2sd_audit_step): record describes the launch as the engine issues it.  An exception
        raised by fn aborts the step and is re-raised here.  Returns the u8 frame, as step_u8 does.  Test aid."""
        self._check()
        frame_nhwc = frame_nhwc.contiguous()
        out = torch.empty((1, 3, self.height, self.width), dtype=torch.uint8, device=self.device)
        failure = []

        def cb(_user, index, after, rec):
            try:
                fn(index, bool(after), rec.contents)
                return 0
            except BaseException as e:   # an exception cannot cross the C frames: keep it and abort the step
                failure.append(e)
                return 1

        cfn = capi.AUDIT_FN(cb)
        rc = self._lib.b2sd_audit_step(self._handle, frame_nhwc.data_ptr(), frame_nhwc.shape[1], frame_nhwc.shape[2],
                                       out.data_ptr(), cfn, None, self._stream())
        if failure:
            raise failure[0]
        capi.check(rc, "b2sd_audit_step")
        return out

    @torch.no_grad()
    def audit_refresh(self, fn: Callable[[int, bool, "capi.LaunchRecord"], None]) -> None:
        """The prompt / timestep refresh of prepare (cross-attention K / V^T of the prompt, time embeddings, every resnet's
        per-slot time bias) run eagerly, with fn called around every kernel launch as in audit_step (b2sd_audit_refresh).
        It recomputes what prepare computed.  Test aid."""
        self._check()
        failure = []

        def cb(_user, index, after, rec):
            try:
                fn(index, bool(after), rec.contents)
                return 0
            except BaseException as e:   # an exception cannot cross the C frames: keep it and abort the refresh
                failure.append(e)
                return 1

        rc = self._lib.b2sd_audit_refresh(self._handle, capi.AUDIT_FN(cb), None, self._stream())
        if failure:
            raise failure[0]
        capi.check(rc, "b2sd_audit_refresh")

    @property
    def launches_per_step(self) -> int:
        return self._lib.b2sd_launches_per_step(self._handle)


def _on_device(t: torch.Tensor, device: torch.device) -> torch.Tensor:
    """t on `device`, copied on the current stream without a host wait (a host tensor goes through pinned memory)"""
    if t.is_cuda:
        return t.to(device).contiguous()
    return t.contiguous().pin_memory().to(device, non_blocking=True)


def _factor_operands(up: torch.Tensor, down: torch.Tensor, scale: float):
    """A LoRA pair as the engine takes it: two fp16 factors as they are (exact operands), anything else as fp32 with each
    factor scaled by a power of two to a largest magnitude in [1, 2) and `scale` compensated (exact), so that the engine's
    fp16 hi / lo split of the factors keeps their small elements."""
    if up.dtype == torch.float16 and down.dtype == torch.float16:
        return up.contiguous(), down.contiguous(), float(scale)
    out = []
    for t in (up, down):
        t = t.float().contiguous()
        amax = float(t.abs().max()) if t.numel() else 0.0
        if amax > 0 and math.isfinite(amax):
            e = math.frexp(amax)[1] - 1        # amax in [2^e, 2^(e+1))
            t = t * 2.0 ** -e
            scale = scale * 2.0 ** e
        out.append(t)
    return out[0], out[1], float(scale)


def _encode_beside(eng: StreamDiffusion, prompt: str) -> torch.Tensor:
    """eng's embedding of `prompt`, [ctx_tokens][D] on the device, ready for the current stream's later work.  The encoder runs
    on a stream of its own: the current stream may have frames queued (a lane's), and an encoder that synchronises its stream
    (CLIP's blocking upload of the token ids) or launches kernels then waits only for earlier encodes, never for those frames."""
    cur = torch.cuda.current_stream(eng.device)
    side = eng._encoder_stream()
    with torch.cuda.stream(side):
        emb = _on_device(eng._encode(prompt)[0], eng.device)
        ready = torch.cuda.Event()
        ready.record(side)
    cur.wait_event(ready)
    emb.record_stream(cur)
    return emb


class StreamState:
    """One temporal stream's stream-batch state (x_t_latent_buffer), apart from the engines that step it (b2sd_state_*): any
    lane of the creating engine's weights steps it, so several video streams share a pool of lanes without mixing their
    frames.  (T-1)*(h/8)*(w/8)*4 fp16 values on the device; nothing at T = 1.  Made by StreamDiffusion.new_state().

    A state may also have its own prompt and its own t_index_list (set_prompt / set_t_index_list): a device copy of the
    conditioning blocks the engines compute from them (cross-attention K / V^T, resnet time biases), which a lane copies in
    before it steps the state.  Without them the state follows the engines' global prompt and t_index_list.  Likewise its own
    ControlNet settings (set_control_scale), which live in the time block beside the time biases: the per-slot scales follow
    the t_index_list the state is stepped with, its own or the global one."""

    own_prompt: Optional[str] = None               # None: the global prompt
    own_t_index_list: Optional[List[int]] = None   # None: the global t_index_list
    own_image: Optional[Tuple[torch.Tensor, float]] = None   # (device tokens [n_tok][D], scale); None: the global image prompt
    own_control: Optional[tuple] = None   # ControlNet settings (check_controls); None: the global settings
    own_canny: Optional[Tuple[float, float]] = None   # Canny thresholds; None: those of the engine that steps the state
    home: Optional[StreamDiffusion] = None   # where clear_overrides recomputes what it keeps (None: the creating engine)

    def __init__(self, engine: StreamDiffusion):
        self._engine = engine          # keeps the engine (and its stream / library) alive while the state exists
        self._lib = engine._lib
        self._handle = C.c_void_p()
        capi.check(self._lib.b2sd_state_create(engine._handle, C.byref(self._handle), engine._stream()), "b2sd_state_create")

    @torch.no_grad()
    def set_prompt(self, prompt: str, engine: Optional[StreamDiffusion] = None) -> None:
        """This stream's own prompt, for the steps submitted after the call.  Computed on `engine` (any lane of the creating
        engine's weights; default the creating engine) on the current CUDA stream, after the frames queued there, with no host
        synchronisation besides the prompt encoder's own, which runs on a stream of its own (_encode_beside) and so never waits
        for queued frames."""
        eng = engine or self._engine
        emb = _encode_beside(eng, prompt)
        capi.check(self._lib.b2sd_state_set_prompt_embeds(eng._handle, self.handle, emb.data_ptr(), eng._stream()),
                   "b2sd_state_set_prompt_embeds")
        self.own_prompt = prompt

    @torch.no_grad()
    def set_t_index_list(self, t_index_list: List[int], engine: Optional[StreamDiffusion] = None) -> None:
        """This stream's own t_index_list, as StreamDiffusion.sync_timesteps applies one: only the timesteps of the time
        embedding change (alpha / beta / c_skip / c_out keep their prepare() values).  Same stream and synchronisation rules as
        set_prompt."""
        eng = engine or self._engine
        t_index_list = list(t_index_list)
        t = _on_device(eng._timestep_tensor([eng.timesteps[i] for i in t_index_list]), eng.device)
        capi.check(self._lib.b2sd_state_set_timesteps(eng._handle, self.handle, t.data_ptr(), eng._stream()),
                   "b2sd_state_set_timesteps")
        self.own_t_index_list = t_index_list
        if eng.has_controlnet:   # the slots are masked with the state's own list
            self._push_control(eng)

    @torch.no_grad()
    def set_control_scale(self, scale: float, start: float = 0.0, end: float = 1.0,
                          engine: Optional[StreamDiffusion] = None) -> None:
        """This stream's own ControlNet settings (StreamDiffusion.set_control_scale's meaning), masked with the state's own
        t_index_list if it has one, else the global one.  The state's own t_index_list is kept.  Checked before anything
        changes; same stream and synchronisation rules as set_prompt."""
        eng = engine or self._engine
        if not eng.has_controlnet:
            raise RuntimeError("this engine was built without a ControlNet")
        control = check_controls(scale, start, end, eng.control_nets)
        self._push_control(eng, control)
        self.own_control = control

    def _push_control(self, eng: StreamDiffusion, control: Optional[tuple] = None) -> None:
        """The state's per-slot ControlNet scales (b2sd_state_set_control_scale, with several nets _scales) from `control`
        (default its own settings, else the global ones) and the t_index_list it is stepped with"""
        control = control or self.own_control or eng.control
        t_index_list = self.own_t_index_list if self.own_t_index_list is not None else eng.t_list
        v = _on_device(torch.tensor(control_vector(control, t_index_list, len(eng.timesteps)), dtype=torch.float32), eng.device)
        fn = "b2sd_state_set_control_scale" if eng.control_nets == 1 else "b2sd_state_set_control_scales"
        capi.check(getattr(self._lib, fn)(eng._handle, self.handle, v.data_ptr(), eng._stream()), fn)

    def set_canny_thresholds(self, low: float = 100.0, high: float = 200.0) -> None:
        """This stream's own Canny thresholds (b2sd_state_set_canny_thresholds): host values that every engine stepping the
        state passes to the Canny kernel, from the next step on.  Nothing else about the state (prompt, t_index_list,
        ControlNet settings, image prompt, the engine or style that steps it) changes them; a global set_canny_thresholds
        drops them."""
        low, high = check_canny_thresholds(low, high)
        capi.check(self._lib.b2sd_state_set_canny_thresholds(self.handle, low, high), "b2sd_state_set_canny_thresholds")
        self.own_canny = (low, high)

    def clear_canny_thresholds(self) -> None:
        """Follow the stepping engine's global Canny thresholds again (no-op for an engine without Canny)"""
        if self._engine.has_canny:
            capi.check(self._lib.b2sd_state_clear_canny_thresholds(self.handle), "b2sd_state_clear_canny_thresholds")
        self.own_canny = None

    @torch.no_grad()
    def set_image_tokens(self, tokens: Optional[torch.Tensor], scale: float = 1.0,
                         engine: Optional[StreamDiffusion] = None) -> None:
        """This stream's own image prompt as (1, n_tok, D) fp16 tokens (StreamDiffusion.image_tokens), None: the global one
        again.  The state's own prompt, if any, is kept.  Same stream and synchronisation rules as set_prompt."""
        eng = engine or self._engine
        if tokens is None:
            self.clear_overrides(prompt=False, t_index_list=False, image_prompt=True, engine=eng)
            return
        tokens = _on_device(tokens.reshape(-1, eng.arch.cross_attention_dim).to(torch.float16), eng.device)
        capi.check(self._lib.b2sd_state_set_image_embeds(eng._handle, self.handle, tokens.data_ptr(), tokens.shape[0],
                                                         float(scale), eng._stream()), "b2sd_state_set_image_embeds")
        self.own_image = (tokens, float(scale))

    def clear_overrides(self, prompt: bool = True, t_index_list: bool = True, image_prompt: Optional[bool] = None,
                        engine: Optional[StreamDiffusion] = None, control: bool = False) -> None:
        """Follow the global prompt, t_index_list, image prompt (default: with the prompt) and / or ControlNet settings again
        from the next step on.  The prompt and the image prompt share one conditioning block, and so do the t_index_list and
        the ControlNet settings: dropping one of a pair recomputes the block with the other on `engine` (default self.home);
        otherwise there is no device work."""
        engine = engine or self.home
        if image_prompt is None:
            image_prompt = prompt
        keep_prompt = None if prompt else self.own_prompt
        keep_image = None if image_prompt else self.own_image
        if prompt or image_prompt:
            capi.check(self._lib.b2sd_state_clear_conditioning(self.handle, capi.COND_PROMPT), "b2sd_state_clear_conditioning")
        if prompt or image_prompt:
            self.own_prompt = self.own_image = None
            if keep_prompt is not None:
                self.set_prompt(keep_prompt, engine=engine)
            if keep_image is not None:
                self.set_image_tokens(*keep_image, engine=engine)
        if t_index_list or control:
            keep_t = None if t_index_list else self.own_t_index_list
            keep_control = None if control else self.own_control
            capi.check(self._lib.b2sd_state_clear_conditioning(self.handle, capi.COND_TIME), "b2sd_state_clear_conditioning")
            self.own_t_index_list, self.own_control = None, keep_control
            if keep_t is not None:
                self.set_t_index_list(keep_t, engine=engine)   # with the settings kept
            elif keep_control is not None:
                self.set_control_scale(*keep_control, engine=engine)

    @property
    def handle(self) -> C.c_void_p:
        if not self._handle.value:
            raise RuntimeError("the stream state is closed")
        return self._handle

    @property
    def closed(self) -> bool:
        return not self._handle.value

    def reset(self) -> None:
        """Zero the state after its last step (stream-ordered, no host synchronisation)."""
        capi.check(self._lib.b2sd_state_reset(self.handle, self._engine._stream()), "b2sd_state_reset")

    def close(self) -> None:
        """Free the state after its last step, stream-ordered, without a host synchronisation.  Idempotent."""
        if self._handle.value:
            h, self._handle = self._handle, C.c_void_p()
            capi.check(self._lib.b2sd_state_destroy(h, self._engine._stream()), "b2sd_state_destroy")

    def __enter__(self) -> "StreamState":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
