"""Drop-in for the reference's `lib/pipeline.py:StreamDiffusionPipeline` (lib/pipeline.py:17-96): same
module constants, constructor, attributes and methods, so agent.py:23,423 and lib/tracks.py:24,38 run on
it unchanged.

Frames: the reference accepts `nvcv.Tensor` (NVDEC path) or `av.VideoFrame` (software decode).  Neither
package exists offline, so frames are recognised structurally: anything exposing
`__cuda_array_interface__` / `.cuda()` (nvcv.Tensor, torch.Tensor) is a GPU u8 NHWC frame, anything with
`.to_ndarray` is an av.VideoFrame; everything else raises Exception("invalid frame type") like
lib/pipeline.py:51-52.

Fast path: a GPU u8 frame goes through ONE engine call (pre + encode + UNet + decode + post fused,
u8 NHWC in -> u8 NCHW out, nothing leaves HBM).  preprocess / predict / postprocess remain callable
separately with the reference's tensor contracts."""
from __future__ import annotations

import collections
import os
import weakref
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .stream import check_controls
from .wrapper import LIVE_LORA_ENV, StreamDiffusionWrapper

DEFAULT_PROMPT = "fireworks in the night sky"
DEFAULT_T_INDEX_LIST = [18, 26, 35, 45]
DEFAULT_NUM_INFERENCE_STEPS = 50
DEFAULT_GUIDANCE_SCALE = 0.0
DEFAULT_LANES_ONE_STEP = 8    # frames in flight for a 1-step stream batch (measured with the throughput launch policy: 4 -> 409, 6 -> 470,
                              # 8 -> 483, 10 -> 481, 12 -> 486 fps; p50 submit -> result 10.4 / 13.5 / 16.8 / 17.8 / 18.7 ms; lanes=1: 241 fps, 4.2 ms)
DEFAULT_LANES_STATEFUL = 2    # T > 1: lanes stage-pipeline each stream state they step (SD-1.5 T=4 512x512, tools/bench_peers.py:
                              # 2 lanes 47.0 / 54.3 fps at 1 / 2+ peers, p50 42.5 / 36.8 ms; 3 lanes 47.1 / 56.1 fps at 1 / 4+
                              # peers but p50 63.7 / 53.4 ms and 3 GB more; 4 lanes no faster)
PER_PEER_STREAMS_ENV = "B200SD_PER_PEER_STREAMS"
CONTROLNET_ENV = "B200SD_CONTROLNET"
MAX_STYLES_ENV = "B200SD_MAX_STYLES"
DEFAULT_MAX_STYLES = 4        # viewers' own styles held at once (PeerStream.update_lora); each holds a UNet copy and its lanes
STYLE_LANES = DEFAULT_LANES_STATEFUL   # lanes of each such style


def env_flag(name: str) -> bool:
    """A boolean environment switch: unset, "", 0, false, no, off -> False; 1, true, yes, on -> True; anything else raises."""
    v = os.getenv(name, "").strip().lower()
    if v in ("", "0", "false", "no", "off"):
        return False
    if v in ("1", "true", "yes", "on"):
        return True
    raise ValueError(f"${name}={os.getenv(name)!r}: expected 1/0, true/false, yes/no or on/off")


def _is_video_frame(frame) -> bool:
    return hasattr(frame, "to_ndarray") and hasattr(frame, "pts")


def _is_gpu_frame(frame) -> bool:
    if isinstance(frame, torch.Tensor):
        return frame.is_cuda
    return hasattr(frame, "__cuda_array_interface__") or (hasattr(frame, "cuda") and hasattr(frame, "layout"))


def _as_torch_u8_nhwc(frame, device) -> torch.Tensor:
    if isinstance(frame, torch.Tensor):
        t = frame
    elif hasattr(frame, "cuda") and not hasattr(frame, "__cuda_array_interface__"):
        t = torch.as_tensor(frame.cuda(), device=device)  # nvcv.Tensor
    else:
        t = torch.as_tensor(frame, device=device)
    if t.dim() == 3:
        t = t.unsqueeze(0)
    if t.dtype != torch.uint8 or t.shape[-1] != 3:
        raise Exception("invalid frame type")
    return t


def _max_styles() -> int:
    return int(os.getenv(MAX_STYLES_ENV, "0")) or DEFAULT_MAX_STYLES


def style_key(lora_dict: Optional[Dict[str, float]]) -> Tuple[Tuple[str, int, int, float], ...]:
    """What a lora_dict means, for the style pool: its (real path, file size, mtime in ns, scale) in order, so that a replaced
    file or another order or scale is another style.  A missing file raises."""
    key = []
    for path, scale in (lora_dict or {}).items():
        st = os.stat(path)
        key.append((os.path.realpath(path), st.st_size, st.st_mtime_ns, float(scale)))
    return tuple(key)


class _Style:
    """A style of the pipeline's weights (StreamDiffusion.add_style) and its lanes, with their own streams: the lane pool of the
    viewers whose own lora_dict it is.  The same attributes as the pipeline's own lane pool, so _enqueue runs on either."""

    def __init__(self, key, lora_dict, engines, streams):
        self.key, self.lora_dict = key, dict(lora_dict or {})
        self._engines, self._lane_streams = engines, streams
        self._lane_done = [None] * len(engines)
        self._next_lane = 0
        self.users = 0   # open viewers on it


class StreamDiffusionPipeline:
    per_peer_streams = False
    _own_state = None   # the StreamState enqueue() steps (per-peer streams, or T > 1 on several lanes); None: the engines' own
    _lora = None        # the global lora_dict (update_lora)
    _lora_key = ()      # its style_key

    def __init__(self, model_id: str, t_index_list: Optional[List[int]] = None, width: int = 512, height: int = 512,
                 prompt: str = DEFAULT_PROMPT, lanes: Optional[int] = None, per_peer_streams: Optional[bool] = None,
                 live_lora: Optional[bool] = None, ip_adapter: Optional[str] = None,
                 controlnet: Optional[Union[str, List[str]]] = None,
                 controlnet_processor: Optional[Union[str, List[Optional[str]]]] = "hed"):
        """lanes: frames in flight for enqueue() ($B200SD_LANES overrides the default).  With a 1-step stream batch (SD-Turbo)
        consecutive frames are independent: DEFAULT_LANES_ONE_STEP lanes process frame n+1.. while frame n is still on the GPU.
        With T > 1 the stream batch carries state from frame to frame: the pipeline's stream is then a stream state that two lanes
        step in turn, stage-pipelined (TAESD encoder of frame n+1 and decoder of frame n-1 overlap the UNet of frame n).  Both
        are bit-identical to submitting the same frames one at a time.

        per_peer_streams (None: $B200SD_PER_PEER_STREAMS, default off): one pipeline serves several viewers, each with its own
        temporal stream.  open_stream() gives a viewer a PeerStream whose frames carry that viewer's stream-batch state only;
        pipeline(frame) / enqueue(frame) keep stepping the pipeline's own stream.  Any lane steps any viewer's state
        (DEFAULT_LANES_STATEFUL lanes for T > 1).  Off, every caller of the pipeline shares one temporal stream, as in the
        reference: with T > 1 a frame's output then mixes in frames of the other callers.

        live_lora (None: $B200SD_LIVE_LORA, default off): update_lora() switches style LoRAs while the pipeline runs.  The base
        weights stay on the device (more HBM, see README), and the packed-weight blob is neither read nor written.

        ip_adapter (None: $B200SD_IP_ADAPTER, default none): an IP-Adapter file (h94 ip-adapter_sd15.safetensors layout) or a
        directory holding one and its image_encoder/; "synthetic" for seeded weights with a synthetic model.
        update_image_prompt() then steers the video with an image, globally or per viewer (PeerStream.update_image_prompt).

        controlnet (None: $B200SD_CONTROLNET, default none): a diffusers ControlNetModel (id or path; "synthetic" with a
        synthetic model), conditioned on each frame's HED edge map (controlnet_processor="hed"), its Canny edge map
        (controlnet_processor="canny", thresholds update_canny_thresholds) or on the frame itself (controlnet_processor=None).  update_controlnet_scale() then sets its strength and guidance window, globally or per
        viewer (PeerStream.update_controlnet_scale).  A list of ids runs several ControlNets (diffusers'
        MultiControlNetModel), each with its own control image and settings; controlnet_processor is then one processor for
        every net or a list with one per net ($B200SD_CONTROLNET stays a single id)."""
        if per_peer_streams is None:
            per_peer_streams = env_flag(PER_PEER_STREAMS_ENV)
        self.per_peer_streams = bool(per_peer_streams)
        self._styles = collections.OrderedDict()   # style_key -> _Style of viewers' own styles, least recently used first
        self._peer_set = weakref.WeakSet()         # open PeerStreams
        self.prompt = prompt
        self.t_index_list = list(t_index_list) if t_index_list is not None else DEFAULT_T_INDEX_LIST
        self.device = "cuda"
        if live_lora is None:
            live_lora = env_flag(LIVE_LORA_ENV)
        self.model = StreamDiffusionWrapper.__new__(StreamDiffusionWrapper)
        self.model.live_lora = bool(live_lora)
        self.model.ip_adapter = ip_adapter
        self.model.canny_processor = True
        if controlnet is None:
            controlnet = os.getenv(CONTROLNET_ENV) or None
        self.model.__init__(
            model_id_or_path=model_id,
            device=self.device,
            dtype=torch.float16,
            t_index_list=self.t_index_list,
            frame_buffer_size=1,
            width=width,
            height=height,
            use_lcm_lora=True,
            output_type="pt",
            mode="img2img",
            use_denoising_batch=True,
            use_tiny_vae=True,
            cfg_type="self",
            engine_dir=os.getenv("TRT_ENGINES_CACHE", "./models/engines"),
            controlnet_id_or_path=controlnet,
            controlnet_processor_id=controlnet_processor,
        )
        stateful = len(self.t_index_list) > 1     # x_t_latent_buffer chains frame n+1 to frame n
        if lanes is None:
            lanes = int(os.getenv("B200SD_LANES", "0")) or (DEFAULT_LANES_STATEFUL if stateful else DEFAULT_LANES_ONE_STEP)
        if stateful and not self.per_peer_streams:
            lanes = min(lanes, 2)   # one stream in three stages, the middle one serial: a third lane has nothing to overlap
        # launch policy = number of frames in flight ($B200SD_POLICY_FRAMES overrides it for profiling: a single lane running the
        # throughput policy's launches gives ncu a clean one-frame launch list)
        self.model.stream.set_concurrency(max(1, int(os.environ.get("B200SD_POLICY_FRAMES", lanes))))
        self.model.prepare(prompt=self.prompt, num_inference_steps=DEFAULT_NUM_INFERENCE_STEPS,
                           guidance_scale=DEFAULT_GUIDANCE_SCALE)
        sd = self.model.stream
        self._engines = [sd] + [sd.add_lane() for _ in range(max(1, lanes) - 1)]
        # enqueue() steps this state: lanes take turns on one T > 1 stream, or the pipeline's stream is one more peer of the pool
        if self.per_peer_streams or (stateful and len(self._engines) > 1):
            self._own_state = sd.new_state()
        # one lane: frames run on the caller's stream, exactly as before.  Several lanes: every lane has its own stream (a lane on
        # the caller's stream would order the other lanes' "input ready" events behind its frames and serialise them)
        self._lane_streams = [None] if len(self._engines) == 1 else [torch.cuda.Stream(sd.device) for _ in self._engines]
        self._lane_done = [None] * len(self._engines)     # completion event of the last frame given to each lane
        self._next_lane = 0
        self._prime(self._lane_streams)

    @property
    def lanes(self) -> int:
        return len(self._engines)

    def _pools(self):
        """the pipeline's lane pool and every style's"""
        return [self] + list(self._styles.values())

    def _quiesce(self):
        """Every lane (the styles' too) finishes its queued frames before a prompt / timestep update touches the shared
        schedule."""
        cur = torch.cuda.current_stream(self.model.stream.device)
        for pool in self._pools():
            for ev in pool._lane_done:
                if ev is not None:
                    cur.wait_event(ev)
        return cur

    def _release(self, cur):
        done = torch.cuda.Event()
        done.record(cur)
        for pool in self._pools():
            for st in pool._lane_streams:
                if st is not None:
                    st.wait_event(done)

    def update_prompt(self, prompt: str):
        """The global prompt: every stream's, including open peer streams with a prompt of their own (PeerStream.update_prompt)."""
        cur = self._quiesce()
        self.model.stream.update_prompt(prompt)
        self._release(cur)

    def update_image_prompt(self, image, scale: float = 1.0):
        """The global image prompt (IP-Adapter): `image` is a PIL image or an HWC uint8 array / tensor, never a path; None clears
        it.  scale weighs the image attention against the text's.  Every stream's, including open peer streams with an image
        prompt of their own (PeerStream.update_image_prompt); each keeps its own prompt.  The image is encoded before anything
        changes; frames enqueued before the call use the old image prompt and frames enqueued after it the new one."""
        sd = self.model.stream
        tokens = None if image is None else sd.image_tokens(image)
        cur = self._quiesce()
        try:
            sd.set_image_tokens(tokens, scale)
        finally:
            self._release(cur)

    def update_lora(self, lora_dict: Optional[Dict[str, float]]):
        """The style LoRAs ({safetensors path: scale}, the wrapper's lora_dict form; None or {}: none) of every stream: the
        pipeline's own and every open peer stream, each keeping its own prompt / t_index_list.  Frames enqueued before the
        call use the old weights and frames enqueued after it the new ones.  Needs live_lora=True; errors are raised before
        anything changes."""
        if not self.model.live_lora:
            raise RuntimeError("update_lora needs StreamDiffusionPipeline(live_lora=True) (or $B200SD_LIVE_LORA=1)")
        cur = self._quiesce()
        try:
            self.model.update_lora(lora_dict)
            # every viewer follows the new global style, as a global prompt replaces viewers' own (the update above has set
            # their own prompt / t_index_list again on the pipeline's engines); cached styles stay valid for later requests
            for peer in list(self._peer_set):
                self._leave_style(peer)
            self._lora, self._lora_key = dict(lora_dict or {}), style_key(lora_dict)
        finally:
            self._release(cur)

    def update_controlnet_scale(self, scale: float, control_guidance_start: float = 0.0, control_guidance_end: float = 1.0):
        """The global ControlNet settings (diffusers' controlnet_conditioning_scale, control_guidance_start / _end): every
        stream's, including open peer streams with settings of their own (PeerStream.update_controlnet_scale); each keeps its
        own t_index_list, which masks its slots.  Checked before anything changes; frames enqueued before the call use the old
        settings and frames enqueued after it the new ones."""
        if not self.model.stream.has_controlnet:
            raise RuntimeError("update_controlnet_scale needs a pipeline with a ControlNet (controlnet=... or $B200SD_CONTROLNET)")
        check_controls(scale, control_guidance_start, control_guidance_end, self.model.stream.control_nets)
        cur = self._quiesce()
        try:
            self.model.update_controlnet_scale(scale, control_guidance_start, control_guidance_end)
        finally:
            self._release(cur)

    def update_canny_thresholds(self, low: float = 100.0, high: float = 200.0):
        """The global Canny thresholds (controlnet_aux CannyDetector's low_threshold / high_threshold): every stream's,
        including open peer streams with thresholds of their own (PeerStream.update_canny_thresholds).  Host values passed to
        the Canny kernel when a frame is enqueued: frames enqueued before the call use the old ones, frames enqueued after it
        the new ones, with no device work and no wait."""
        if not self.model.stream.has_canny:
            raise RuntimeError("update_canny_thresholds needs a pipeline with a ControlNet whose processor is 'canny' "
                               "(controlnet_processor='canny')")
        self.model.update_canny_thresholds(low, high)

    # ---- viewers' own styles (PeerStream.update_lora) ------------------------------------------------------------------
    def _leave_style(self, peer) -> None:
        if peer._style is not None:
            peer._style.users -= 1
            peer._style, peer._lora = None, None
            if peer._state is not None:
                peer._state.home = self.model.stream

    def _set_peer_style(self, peer, lora_dict: Optional[Dict[str, float]]) -> None:
        """Move `peer` to the lane pool of lora_dict's style (the pipeline's own when it is the global one), building the style
        when it is not cached.  Everything that can fail is checked before anything changes; unused styles beyond
        $B200SD_MAX_STYLES are evicted only once the switch has succeeded, so a build briefly holds one style more."""
        from .weights import lora_factors
        state = peer._live_state()
        if not self.model.live_lora:
            raise RuntimeError("PeerStream.update_lora needs StreamDiffusionPipeline(live_lora=True) (or $B200SD_LIVE_LORA=1)")
        key = style_key(lora_dict)
        if key == self._lora_key:
            target = None
        elif key in self._styles:
            target = self._styles[key]
        else:
            sd = self.model.stream
            factors = lora_factors(sd._unet_shapes, lora_dict)   # reads the files and checks every pair
            limit = _max_styles()
            unused = any(st.users == 0 for st in self._styles.values())
            leaving = peer._style is not None and peer._style.users == 1   # the viewer's style, which it alone uses
            if len(self._styles) >= limit and not unused and not leaving:
                raise RuntimeError(f"every one of the {limit} viewer styles (${MAX_STYLES_ENV}) is in use")
            target = self._build_style(key, lora_dict, factors)
        if target is peer._style:
            return
        if target is not None:
            self._styles[target.key] = self._styles.pop(target.key)   # most recently used
        # the viewer's own conditioning is computed again with the new weights, on the lane that takes its next frame
        pool = target or self
        image, control = getattr(state, "own_image", None), getattr(state, "own_control", None)
        if state.own_prompt is not None or state.own_t_index_list is not None or image is not None or control is not None:
            prompt, t_index_list = state.own_prompt, state.own_t_index_list

            def rebind(engine):
                if prompt is not None:
                    state.set_prompt(prompt, engine=engine)
                if t_index_list is not None:
                    state.set_t_index_list(t_index_list, engine=engine)   # with the viewer's ControlNet settings
                elif control is not None:
                    state.set_control_scale(*control, engine=engine)
                if image is not None:
                    state.set_image_tokens(*image, engine=engine)
            self._update_state(rebind, pool)
        self._leave_style(peer)
        if target is not None:
            target.users += 1
            peer._style, peer._lora = target, dict(lora_dict or {})
            state.home = target._engines[0]
        # back within the bound: unused styles, least recently used first, each freed after its last frames
        for k in [k for k, st in self._styles.items() if st.users == 0]:
            if len(self._styles) <= _max_styles():
                break
            self._evict(k)

    def _build_style(self, key, lora_dict, factors) -> _Style:
        """A style and its lanes, made, prepared and fused on a stream of their own: no wait for any queued frame."""
        sd = self.model.stream
        streams = [torch.cuda.Stream(sd.device) for _ in range(STYLE_LANES)]
        with torch.cuda.stream(streams[0]):
            style = sd.add_style()
            try:
                engines = [style] + [style.add_lane() for _ in range(STYLE_LANES - 1)]
                style.apply_factors(factors)
            except BaseException:
                sd.drop_style(style, streams[0])
                raise
        done = torch.cuda.Event()
        done.record(streams[0])
        for st in streams[1:]:
            st.wait_event(done)
        self._prime(streams)
        pool = self._styles[key] = _Style(key, lora_dict, engines, streams)
        return pool

    def _evict(self, key) -> None:
        """Free a cached style no viewer uses, after its lanes' last frames: stream-ordered, no host or device wait."""
        pool = self._styles.pop(key)
        after = torch.cuda.Stream(self.model.stream.device)
        for st in pool._lane_streams:   # the style's build and every frame given to it
            after.wait_stream(st)
        for ev in pool._lane_done:      # and their downloads
            if ev is not None:
                after.wait_event(ev)
        self.model.stream.drop_style(pool._engines[0], after)

    def _prime(self, streams) -> None:
        """Every frame's output is a fresh tensor allocated on its lane's stream (the caller owns it and may hold it across
        calls, SURVEY 8b "Ownership").  Give each lane stream's allocator pool a few output-sized blocks now: the first
        cudaMalloc a lane needed in the middle of a stream otherwise synchronises the device, i.e. stalls every frame in flight
        once (seen as a single 2x latency spike, 33 ms instead of 17 ms, some 50-80 frames into a run with 10 frames pending)."""
        for st in streams:
            if st is not None:
                with torch.cuda.stream(st):
                    prime = [torch.empty((1, 3, self.model.height, self.model.width), dtype=torch.uint8,
                                         device=self.model.stream.device) for _ in range(4)]
                    del prime

    @property
    def styles(self) -> int:
        """viewers' own styles held (PeerStream.update_lora), in use or cached"""
        return len(self._styles)

    def update_t_index_list(self, t_index_list: List[int]):
        """The global t_index_list: every stream's, including open peer streams with one of their own."""
        cur = self._quiesce()
        self.model.update_t_index_list(t_index_list)
        self.model.stream.clear_overrides(prompt=False, t_index_list=True)   # also when the global list was already this one
        self._release(cur)

    def _update_state(self, update, pool=None) -> None:
        """update(engine) refreshes one peer's conditioning on the lane of `pool` (a style's lanes, default the pipeline's) that
        takes the next submission, on that lane's stream: stream-ordered after the frames queued there, with no host wait and no
        wait on the other lanes."""
        pool = pool or self
        lane = pool._next_lane
        compute = pool._lane_streams[lane] or torch.cuda.current_stream(self.model.stream.device)
        with torch.cuda.stream(compute):
            update(pool._engines[lane])

    # ---- reference-shaped stages ----------------------------------------------------------------------
    def preprocess(self, frame) -> torch.Tensor:
        """-> (3,H,W) float32 in [0,1] on the GPU (lib/pipeline.py:50-67)."""
        if not _is_gpu_frame(frame) and not _is_video_frame(frame):
            raise Exception("invalid frame type")
        if _is_video_frame(frame):
            t = torch.from_numpy(frame.to_ndarray(format="rgb24")).unsqueeze(0).to(self.device)
        else:
            t = _as_torch_u8_nhwc(frame, self.device)
        return (t.to(torch.float32) * (1.0 / 255.0)).permute(0, 3, 1, 2).squeeze(0)

    def predict(self, frame: torch.Tensor) -> torch.Tensor:
        return self.model(image=frame)

    def postprocess(self, frame: torch.Tensor) -> torch.Tensor:
        """(3,H,W) in [0,1] -> (1,3,H,W) uint8; the cast truncates (lib/pipeline.py:72-74)."""
        return frame.mul(255.0).clamp_(0, 255).to(torch.uint8)[None]

    def __call__(self, frame):
        """lib/pipeline.py:76-96, blocking semantics preserved: the result is complete when the call returns only in the
        software-encode branch (`.cpu()`); with NVENC set the CUDA tensor is returned stream-ordered, like the reference."""
        return self._call(frame, self._own_state)

    def _call(self, frame, state, pool=None):
        ticket = self._enqueue(frame, state, pool)
        if os.getenv("NVENC"):
            ticket.wait(torch.cuda.current_stream(self.model.stream.device))   # stream-ordered result, whichever lane ran it
            return ticket.result(wait=False)
        return ticket.result()

    def open_stream(self) -> "PeerStream":
        """A new viewer's temporal stream (per_peer_streams only): its frames carry its own stream-batch state, starting from
        zeros, whatever other viewers submit in between."""
        if not self.per_peer_streams:
            raise RuntimeError("open_stream() needs per_peer_streams=True (or $B200SD_PER_PEER_STREAMS=1): without it every "
                               "caller of this pipeline shares one temporal stream")
        return PeerStream(self)

    # ---- non-blocking entry (SURVEY.md 8f-2): everything is queued on CUDA streams and a ticket comes back at once ------
    def enqueue(self, frame) -> "FrameTicket":
        """Queue one frame and return immediately.  GPU frames (NVDEC path) go straight to the engine on the current
        stream.  av.VideoFrame input is staged through a pinned ring and copied on a separate copy stream, so the upload of
        frame n+1 overlaps the compute of frame n; with NVENC unset the download of the result is queued the same way.
        Tickets complete in submission order (one temporal stream per pipeline, like the reference)."""
        return self._enqueue(frame, self._own_state)

    def _enqueue(self, frame, state, pool=None) -> "FrameTicket":
        """enqueue() on `state` (a StreamState, or None for the engines' own stream) on the lanes of `pool` (a viewer's
        style, default the pipeline's).  Lanes rotate over all submissions to the pool; frames of one state are ordered on the
        device by the state's event."""
        if not _is_gpu_frame(frame) and not _is_video_frame(frame):
            raise Exception("invalid frame type")
        pool = pool or self
        dev = self.model.stream.device
        caller = torch.cuda.current_stream(dev)
        lane = pool._next_lane
        pool._next_lane = (lane + 1) % len(pool._engines)
        engine = pool._engines[lane]
        compute = pool._lane_streams[lane] or caller
        if compute is not caller:
            ready = torch.cuda.Event()
            ready.record(caller)          # whatever produced the frame on the caller's stream
            compute.wait_event(ready)
        if _is_video_frame(frame):
            self._ensure_staging(dev)
            slot = self._slot
            self._slot = (slot + 1) % len(self._pinned_in)
            self._slot_free[slot].synchronize()          # the ring entry's previous upload has been consumed (depth-4 ring)
            arr = frame.to_ndarray(format="rgb24")
            host = self._pinned_in[slot]
            if tuple(arr.shape) != tuple(host.shape[1:]):
                host = self._pinned_in[slot] = torch.empty((1,) + tuple(arr.shape), dtype=torch.uint8).pin_memory()
            host[0].copy_(torch.from_numpy(arr))
            with torch.cuda.stream(self._copy_stream):
                rgb = host.to(dev, non_blocking=True)
                uploaded = torch.cuda.Event()
                uploaded.record(self._copy_stream)
            compute.wait_event(uploaded)
            rgb.record_stream(compute)
        else:
            slot = None
            rgb = _as_torch_u8_nhwc(frame, self.device)
            if compute is not caller:
                rgb.record_stream(compute)
        with torch.cuda.stream(compute):
            post_output = engine.step_u8(rgb, state=state)
        if compute is not caller:
            post_output.record_stream(caller)
        if slot is not None:
            self._slot_free[slot].record(compute)
        done = torch.cuda.Event()
        if os.getenv("NVENC"):
            done.record(compute)
            pool._lane_done[lane] = done
            return FrameTicket(post_output, done, None, None)
        # software-encode branch (lib/pipeline.py:83-94): hand back an av.VideoFrame with the input's timing
        assert _is_video_frame(frame)
        self._ensure_staging(dev)
        host_out = torch.empty((1, 3, self.model.height, self.model.width), dtype=torch.uint8).pin_memory()
        computed = torch.cuda.Event()
        computed.record(compute)
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(computed)
            host_out.copy_(post_output, non_blocking=True)
            post_output.record_stream(self._copy_stream)
            done.record(self._copy_stream)
        pool._lane_done[lane] = done
        return FrameTicket(post_output, done, host_out, frame)

    def _ensure_staging(self, dev) -> None:
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(dev)
            self._pinned_in = [torch.empty((1, self.model.height, self.model.width, 3), dtype=torch.uint8).pin_memory()
                               for _ in range(4)]
            self._slot_free = [torch.cuda.Event() for _ in range(4)]
            self._slot = 0


class FrameTicket:
    """Result handle of StreamDiffusionPipeline.enqueue()."""

    def __init__(self, tensor: torch.Tensor, done: "torch.cuda.Event", host_out: Optional[torch.Tensor], src_frame):
        self._tensor, self._done, self._host_out, self._src = tensor, done, host_out, src_frame

    def done(self) -> bool:
        """True once every GPU operation of this frame (and the download, if any) has finished; never blocks."""
        return self._done.query()

    def wait(self, stream) -> None:
        """Make `stream` wait for this frame (no host synchronisation): later work on it sees the finished tensor."""
        stream.wait_event(self._done)

    def result(self, wait: bool = True):
        """The (1,3,H,W) u8 CUDA tensor (NVENC set) or an av.VideoFrame carrying the input's pts/time_base."""
        if self._host_out is None:
            if wait:
                self._done.synchronize()
            return self._tensor
        try:
            import av
        except ImportError as exc:
            raise RuntimeError("NVENC is unset, so an av.VideoFrame must be returned, but PyAV is not installed; "
                               "set NVENC=1 to receive the CUDA tensor") from exc
        self._done.synchronize()
        hwc = self._host_out.permute(0, 2, 3, 1).squeeze(0).numpy()
        out = av.VideoFrame.from_ndarray(np.ascontiguousarray(hwc))
        out.pts = self._src.pts
        out.time_base = self._src.time_base
        return out


class PeerStream:
    """One viewer's temporal stream on a per-peer pipeline (StreamDiffusionPipeline.open_stream): enqueue() / __call__ behave
    as the pipeline's, with this viewer's own stream-batch state, and with this viewer's own prompt / t_index_list once it sets
    them (update_prompt / update_t_index_list; until then the pipeline's).  close() frees the state after its last frame,
    without a host synchronisation."""

    _style = None   # the pipeline's _Style this viewer's frames run on; None: the pipeline's lanes
    _lora = None    # this viewer's own lora_dict (update_lora), with _style

    def __init__(self, pipeline: StreamDiffusionPipeline):
        self._pipeline = pipeline
        self._state = pipeline.model.stream.new_state()
        pipeline._peer_set.add(self)

    @property
    def closed(self) -> bool:
        return self._state is None

    def _live_state(self):
        if self._state is None:
            raise RuntimeError("the peer stream is closed")
        return self._state

    def enqueue(self, frame) -> FrameTicket:
        return self._pipeline._enqueue(frame, self._live_state(), self._style)

    @property
    def prompt(self) -> str:
        """This viewer's prompt: its own (update_prompt) or the pipeline's global one"""
        own = self._live_state().own_prompt
        return own if own is not None else self._pipeline.model.stream.prompt

    @property
    def t_index_list(self) -> List[int]:
        own = self._live_state().own_t_index_list
        return list(own if own is not None else self._pipeline.model.stream.t_list)

    def update_prompt(self, prompt: str) -> None:
        """This viewer's own prompt: its frames enqueued after the call use it, whichever lane runs them; frames already
        queued, and every other viewer's frames, are unaffected.  Does not wait for queued frames.  A later global
        pipeline.update_prompt replaces it."""
        state = self._live_state()
        self._pipeline._update_state(lambda engine: state.set_prompt(prompt, engine=engine), self._style)

    @property
    def image_prompt(self):
        """(tokens, scale) of this viewer's image prompt: its own (update_image_prompt) or the pipeline's global one (None: none)"""
        own = self._live_state().own_image
        return own if own is not None else self._pipeline.model.stream.image_prompt

    def update_image_prompt(self, image, scale: float = 1.0) -> None:
        """This viewer's own image prompt (IP-Adapter): a PIL image or an HWC uint8 array / tensor, never a path; None: the
        pipeline's global one again.  update_prompt's ordering; the viewer keeps its own prompt.  A later global
        pipeline.update_image_prompt replaces it."""
        state = self._live_state()
        tokens = None if image is None else self._pipeline.model.stream.image_tokens(image)
        self._pipeline._update_state(lambda engine: state.set_image_tokens(tokens, scale, engine=engine), self._style)

    def update_t_index_list(self, t_index_list: List[int]) -> None:
        """This viewer's own t_index_list, with the semantics of the global update_t_index_list (only the time embedding's
        timesteps change) and update_prompt's ordering."""
        state = self._live_state()
        self._pipeline._update_state(lambda engine: state.set_t_index_list(t_index_list, engine=engine), self._style)

    @property
    def controlnet_scale(self) -> tuple:
        """This viewer's ControlNet (scale, start, end): its own (update_controlnet_scale) or the pipeline's global ones.  With
        several ControlNets each of the three is a list with one entry per net."""
        own = self._live_state().own_control
        control = own if own is not None else self._pipeline.model.stream.control
        return control if not isinstance(control[0], tuple) else tuple(list(v) for v in control)

    def update_controlnet_scale(self, scale: float, control_guidance_start: float = 0.0,
                                control_guidance_end: float = 1.0) -> None:
        """This viewer's own ControlNet settings (the pipeline's update_controlnet_scale), masked with its own t_index_list if
        it has one; update_prompt's ordering.  It keeps them through a global prompt / t_index_list / image prompt / LoRA
        update and a style move; a later global pipeline.update_controlnet_scale replaces them."""
        state = self._live_state()
        if not self._pipeline.model.stream.has_controlnet:
            raise RuntimeError("update_controlnet_scale needs a pipeline with a ControlNet (controlnet=... or $B200SD_CONTROLNET)")
        control = check_controls(scale, control_guidance_start, control_guidance_end,
                                 self._pipeline.model.stream.control_nets)
        self._pipeline._update_state(lambda engine: state.set_control_scale(*control, engine=engine), self._style)

    @property
    def canny_thresholds(self) -> tuple:
        """This viewer's Canny (low, high): its own (update_canny_thresholds) or the pipeline's global ones"""
        own = self._live_state().own_canny
        return own if own is not None else self._pipeline.model.stream.canny_thresholds

    def update_canny_thresholds(self, low: float = 100.0, high: float = 200.0) -> None:
        """This viewer's own Canny thresholds: its frames enqueued after the call use them, whichever lane or style runs them;
        frames already queued, and every other viewer's frames, are unaffected.  No device work, no wait.  It keeps them
        through prompt, t_index_list, image-prompt, ControlNet-scale and LoRA updates and style moves; a later global
        pipeline.update_canny_thresholds replaces them."""
        state = self._live_state()
        if not self._pipeline.model.stream.has_canny:
            raise RuntimeError("update_canny_thresholds needs a pipeline with a ControlNet whose processor is 'canny' "
                               "(controlnet_processor='canny')")
        state.set_canny_thresholds(low, high)

    @property
    def lora(self) -> Dict[str, float]:
        """This viewer's style LoRAs: its own (update_lora) or the pipeline's global ones"""
        self._live_state()
        return dict(self._lora if self._style is not None else (self._pipeline._lora or {}))

    def update_lora(self, lora_dict: Optional[Dict[str, float]]) -> None:
        """This viewer's own style: the base weights plus the LoRAs of lora_dict ({safetensors path: scale}, fused in order, the
        constructor's form; None or {}: the base weights).  Its frames enqueued after the call use it and frames already queued
        the old one; the stream state carries across, and the viewer keeps its own prompt / t_index_list.  Every other viewer
        is unaffected.  Viewers with the same lora_dict share one style; the global lora_dict is the pipeline's own lanes.  A
        style is built (on streams of its own, waiting for no queued frame) when no cached one matches; $B200SD_MAX_STYLES
        bounds how many are held, the least recently used unused one making room.  Needs live_lora=True.  Errors (a closed
        stream, a bad file, a pair that does not fit, a LoRA matching no module, every style in use) are raised before anything
        changes.  A later global pipeline.update_lora replaces it."""
        self._pipeline._set_peer_style(self, lora_dict)

    def __call__(self, frame):
        return self._pipeline._call(frame, self._live_state(), self._style)

    def close(self) -> None:
        if self._state is not None:
            state, self._state = self._state, None
            self._pipeline._leave_style(self)
            state.close()

    def __enter__(self) -> "PeerStream":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        # a viewer dropped without close(): its style is no longer in use, and its state is freed after its last frame
        try:
            self.close()
        except Exception:
            pass
