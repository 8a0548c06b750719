"""Drop-in proof for the caller of the hot path (SURVEY.md 8 a-1 / f-2), CPU only.

The reference's own, unmodified lib/tracks.py (lib/tracks.py:9-38), loaded with `aiortc` stubbed and driven by the fake source
track and recording pipeline below, was run once per DROP_FRAMES setting; what it returned and the pipeline calls it made are
stored in tests/golden/reference_tracks.json (tests/golden/make_golden_tracks.py records them from a reference checkout).
This repo's non-blocking adapter (host/tracks.py) must make the same pipeline calls in the same order and return the same
frames through warm-up, frame dropping and steady state."""
import asyncio
import json
import os

import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_tracks.json")


class FakeSource:
    """aiortc-like source track: recv() is a coroutine handing out numbered frames."""

    def __init__(self):
        self.n = 0

    async def recv(self):
        await asyncio.sleep(0)
        self.n += 1
        return ("frame", self.n)


class RecordingPipeline:
    """Stands for StreamDiffusionPipeline: records the frames it is called with (lib/tracks.py:24,38 call `pipeline(frame)`)."""

    def __init__(self):
        self.calls = []

    def __call__(self, frame):
        self.calls.append(frame)
        return ("processed", frame[1])


class Ticket:
    def __init__(self, value, polls):
        self.value, self.polls = value, polls

    def done(self):
        self.polls -= 1
        return self.polls < 0

    def result(self):
        return self.value


class AsyncRecordingPipeline(RecordingPipeline):
    """Same, with the non-blocking enqueue() entry of host/pipeline.py; every ticket needs a few polls to complete."""

    def enqueue(self, frame):
        return Ticket(self(frame), polls=3)


def _drive(track, n):
    async def go():
        return [await track.recv() for _ in range(n)]
    return asyncio.run(go())


@pytest.mark.parametrize("drop", [0, 1])
def test_reference_tracks_py_runs_unchanged_and_adapter_matches_it(monkeypatch, drop):
    monkeypatch.delenv("WARMUP_FRAMES", raising=False)
    monkeypatch.setenv("DROP_FRAMES", str(drop))
    with open(GOLDEN) as f:
        ref = json.load(f)[str(drop)]
    ref_out = [tuple(o) for o in ref["outputs"]]
    ref_calls = [tuple(c) for c in ref["calls"]]
    our_pipe = AsyncRecordingPipeline()
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    our_track = VideoStreamTrack(FakeSource(), our_pipe)
    our_out = _drive(our_track, 5)
    # warm-up: 10 frames through the pipeline, discarded (lib/tracks.py:21-25); then `drop` source frames skipped per output
    first = 10 + drop + 1
    assert ref_out[0] == ("processed", first)
    assert [c[1] for c in ref_calls[:10]] == list(range(1, 11))
    assert our_out == ref_out
    assert our_pipe.calls == ref_calls
    assert ref["warmup_frame_idx"] == our_track.warmup_frame_idx == 10


def test_reference_tracks_py_imports_this_repos_pipeline_module(monkeypatch):
    """agent.py:23 does `from lib.pipeline import StreamDiffusionPipeline` next to `from lib.tracks import VideoStreamTrack`:
    both names must resolve in this repo's lib/ package, and the pipeline class must be callable with one frame argument."""
    import inspect
    import lib.pipeline as lp
    import lib.tracks as lt
    assert inspect.iscoroutinefunction(lt.VideoStreamTrack.recv)
    sig = inspect.signature(lp.StreamDiffusionPipeline.__call__)
    assert list(sig.parameters) == ["self", "frame"]
    assert hasattr(lp.StreamDiffusionPipeline, "enqueue")


def test_adapter_yields_to_the_event_loop_while_a_frame_is_in_flight(monkeypatch):
    """The point of 8f-2: while the GPU works on a frame the event loop keeps running other coroutines."""
    monkeypatch.setenv("WARMUP_FRAMES", "2")
    monkeypatch.setenv("DROP_FRAMES", "0")
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = AsyncRecordingPipeline()
    track = VideoStreamTrack(FakeSource(), pipe)
    assert track.warmup_frames == 2      # int-cast (the reference keeps the env string and would raise on `int < str`)
    ticks = []

    async def other_peer():
        for _ in range(50):
            ticks.append(len(pipe.calls))
            await asyncio.sleep(0)

    async def go():
        t = asyncio.create_task(other_peer())
        out = await track.recv()
        await t
        return out

    out = asyncio.run(go())
    assert out == ("processed", 3)
    assert len(set(ticks)) >= 3, "the other coroutine must have observed the pipeline at several stages"


def test_adapter_accepts_a_plain_callable_pipeline(monkeypatch):
    monkeypatch.setenv("WARMUP_FRAMES", "0")
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = RecordingPipeline()
    assert _drive(VideoStreamTrack(FakeSource(), pipe), 3) == [("processed", 1), ("processed", 2), ("processed", 3)]
