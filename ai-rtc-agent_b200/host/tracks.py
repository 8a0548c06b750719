"""Media-track adapter: the reference's `lib/tracks.py:VideoStreamTrack` (lib/tracks.py:9-38) with the one change
SURVEY.md 8f-2 asks for -- `pipeline(frame)` no longer blocks the asyncio event loop.

Same behaviour as the reference: the first `WARMUP_FRAMES` (default 10) source frames are run through the pipeline and
discarded on the first `recv()`, then `DROP_FRAMES` source frames are skipped before every processed frame, and every
`recv()` returns exactly one processed frame, in order.  Differences, both deliberate:
  * the frame is ENQUEUED (StreamDiffusionPipeline.enqueue: H2D copy, engine, D2H copy all stream-ordered) and the coroutine
    yields to the event loop until the CUDA event fires, so decoding / networking of neighbouring frames and other peers
    overlaps the GPU work instead of waiting behind a blocking call (lib/tracks.py:24,38 block the loop);
  * WARMUP_FRAMES is int-cast (in the reference a value set through the environment stays a str and `int < str` raises).
The reference's own lib/tracks.py also runs unmodified on lib.pipeline (tests/test_tracks.py); this adapter is the
non-blocking replacement.  aiortc is optional: with it installed the class derives from aiortc.MediaStreamTrack."""
from __future__ import annotations

import asyncio
import logging
import os

logger = logging.getLogger(__name__)

try:  # pragma: no cover - aiortc is not installable offline
    from aiortc import MediaStreamTrack as _Base
except ImportError:
    class _Base:  # minimal stand-in with the attributes aiortc's base class provides
        kind = "unknown"

        def __init__(self):
            self._ended = False

        def stop(self):
            self._ended = True


class VideoStreamTrack(_Base):
    kind = "video"

    def __init__(self, track, pipeline, poll_interval: float = 0.0):
        super().__init__()
        self.track = track
        self.pipeline = pipeline
        self.warmup_frame_idx = 0
        self.warmup_frames = int(os.getenv("WARMUP_FRAMES", 10))
        self.drop_frames = int(os.getenv("DROP_FRAMES", 0))
        self.poll_interval = poll_interval
        # a pipeline with per-peer streams gives this track its own temporal stream, opened at the first frame
        self._per_peer = bool(getattr(pipeline, "per_peer_streams", False))
        self._peer = None
        self._stopped = False

    def _target(self):
        if not self._per_peer:
            return self.pipeline
        if self._peer is None:
            self._peer = self.pipeline.open_stream()
        return self._peer

    def _close_stream(self):
        """Free this track's stream state (stream-ordered after its last frame: no device or host synchronisation)."""
        if self._peer is not None:
            peer, self._peer = self._peer, None
            peer.close()

    def stop(self):
        super().stop()
        self._stopped = True
        self._close_stream()

    def update_prompt(self, prompt: str) -> None:
        """A config message's prompt: this track's viewer only with per-peer streams (the stream is opened if no frame has
        arrived yet), else the pipeline's global prompt.  A no-op once the track is stopped."""
        if not self._stopped:
            self._target().update_prompt(prompt)

    def update_t_index_list(self, t_index_list) -> None:
        """As update_prompt, for the t_index_list"""
        if not self._stopped:
            self._target().update_t_index_list(t_index_list)

    def update_lora(self, lora_dict) -> None:
        """As update_prompt, for the style LoRAs ({safetensors path: scale}; None or {}: none): this viewer's own style with
        per-peer streams (PeerStream.update_lora), else the pipeline's global one"""
        if not self._stopped:
            self._target().update_lora(lora_dict)

    def update_image_prompt(self, image, scale: float = 1.0) -> None:
        """As update_prompt, for the IP-Adapter image prompt (a PIL image or an HWC uint8 array / tensor, never a path; None
        clears it): this viewer's own with per-peer streams (PeerStream.update_image_prompt), else the pipeline's global one"""
        if not self._stopped:
            self._target().update_image_prompt(image, scale)

    async def _recv_source(self):
        try:
            return await self.track.recv()
        except BaseException:   # the source ended (aiortc raises MediaStreamError) or the coroutine was cancelled
            self._close_stream()
            raise

    async def _process(self, frame):
        target = self._target()
        enqueue = getattr(target, "enqueue", None)
        if enqueue is None:                      # any callable pipeline works; it is then called synchronously like the reference
            return target(frame)
        ticket = enqueue(frame)
        while not ticket.done():
            await asyncio.sleep(self.poll_interval)   # let the event loop run while the GPU works
        return ticket.result()

    async def recv(self):
        while self.warmup_frame_idx < self.warmup_frames:
            logger.info(f"dropping warmup frames {self.warmup_frame_idx}")
            frame = await self._recv_source()
            await self._process(frame)
            self.warmup_frame_idx += 1

        # Frame dropping (lib/tracks.py:27-31): skipping source frames can help playback with some encoders
        for _ in range(self.drop_frames):
            await self._recv_source()

        frame = await self._recv_source()
        return await self._process(frame)
