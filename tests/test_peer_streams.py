"""Per-peer temporal streams without a GPU: the pipeline's lane rotation and state routing over fake engines, the opt-in switch,
the track adapter's stream lifecycle, and the ctypes signatures of the stream-state calls."""
import asyncio
import contextlib
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- fake engines: record every step with its lane and state ----------------------------------------------------------------------
class FakeState:
    def __init__(self, n):
        self.n, self.closed, self.resets = n, False, 0

    def reset(self):
        self.resets += 1

    def close(self):
        self.closed = True


class FakeOut:
    def __init__(self, lane, state, frame):
        self.lane, self.state, self.frame = lane, state, frame

    def record_stream(self, stream):
        pass


class FakeEngine:
    """Stands for host.stream.StreamDiffusion: lanes share one log and one state counter, as lanes share one weight store."""

    def __init__(self, log, lane=0, states=None):
        self.log, self.lane = log, lane
        self.states = [] if states is None else states
        self.lanes, self.concurrency = [], None
        self.device = "cpu"

    def set_concurrency(self, n):
        self.concurrency = n

    def add_lane(self):   # as StreamDiffusion.add_lane: every lane is an independent engine
        lane = FakeEngine(self.log, len(self.lanes) + 1, self.states)
        self.lanes.append(lane)
        return lane

    def new_state(self):
        s = FakeState(len(self.states))
        self.states.append(s)
        return s

    def step_u8(self, rgb, state=None):
        self.log.append((self.lane, state, rgb.frame))
        return FakeOut(self.lane, state, rgb.frame)


class FakeFrame:
    def __init__(self, frame):
        self.frame = frame

    def record_stream(self, stream):
        pass


class FakeEvent:
    def record(self, stream=None):
        pass

    def query(self):
        return True

    def synchronize(self):
        pass


class FakeCudaStream:
    def __init__(self, *a, **k):
        pass

    def wait_event(self, ev):
        pass


@pytest.fixture
def fake_pipeline(monkeypatch):
    """make(t_index_list, **kw) -> (StreamDiffusionPipeline over fake engines, step log)"""
    from ai_rtc_agent_b200.host import pipeline as P
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    monkeypatch.delenv("B200SD_POLICY_FRAMES", raising=False)
    monkeypatch.delenv(P.PER_PEER_STREAMS_ENV, raising=False)
    monkeypatch.setattr(torch.cuda, "Stream", FakeCudaStream)
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    caller = FakeCudaStream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: caller)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(P, "_is_gpu_frame", lambda f: True)
    monkeypatch.setattr(P, "_as_torch_u8_nhwc", lambda f, d: FakeFrame(f))
    log = []

    class FakeWrapper:
        def __init__(self, t_index_list, width, height, **kw):
            self.stream = FakeEngine(log)
            self.height, self.width = height, width

        def prepare(self, **kw):
            pass

    monkeypatch.setattr(P, "StreamDiffusionWrapper", FakeWrapper)

    def make(t_index_list, **kw):
        return P.StreamDiffusionPipeline("tiny-sd15", t_index_list=t_index_list, width=64, height=64, **kw), log
    return make


def test_lanes_rotate_over_every_submission(fake_pipeline):
    pipe, log = fake_pipeline([18, 26, 35, 45], per_peer_streams=True, lanes=3)
    assert pipe.lanes == 3
    a, b = pipe.open_stream(), pipe.open_stream()
    for i, who in enumerate([a, b, pipe, b, a, a, b]):
        who.enqueue(("f", i))
    assert [lane for lane, _, _ in log] == [0, 1, 2, 0, 1, 2, 0]


def test_each_peer_steps_its_own_state(fake_pipeline):
    pipe, log = fake_pipeline([18, 26, 35, 45], per_peer_streams=True, lanes=2)
    own = pipe.model.stream.states[0]           # the pipeline's own stream
    a, b = pipe.open_stream(), pipe.open_stream()
    sa, sb = a._state, b._state
    assert len({id(own), id(sa), id(sb)}) == 3
    order = [("a", a), ("b", b), ("p", pipe), ("a", a), ("a", a), ("b", b), ("p", pipe)]
    outs = [who(("f", k, i)) for i, (k, who) in enumerate(order)]
    want = {"a": sa, "b": sb, "p": own}
    for (k, _), (_, state, frame), out in zip(order, log, outs):
        assert state is want[k] and frame[1] == k and out.state is want[k]
    a.close()
    assert sa.closed and not sb.closed and a.closed
    with pytest.raises(RuntimeError, match="closed"):
        a.enqueue(("f", "a", 99))
    with b:
        pass
    assert sb.closed


def test_mode_off_refuses_open_stream_and_lanes_step_one_own_state(fake_pipeline):
    pipe, log = fake_pipeline([18, 26, 35, 45], lanes=5)
    assert not pipe.per_peer_streams
    assert pipe.lanes == 2, "one stream: two stage-pipelined lanes"
    with pytest.raises(RuntimeError, match="per_peer_streams"):
        pipe.open_stream()
    for i in range(4):
        pipe.enqueue(("f", i))
    states = pipe.model.stream.states
    assert len(states) == 1, "the pipeline's own stream is one state"
    assert [(lane, state) for lane, state, _ in log] == [(0, states[0]), (1, states[0])] * 2, \
        "independent lanes step that state in turn"
    for tl, lanes in (([18, 26, 35, 45], 1), ([32], 8)):
        assert fake_pipeline(tl, lanes=lanes)[0]._own_state is None, "one lane, or T = 1: the engines' own latent buffers"


def test_lane_default_for_each_stream_batch(fake_pipeline):
    from ai_rtc_agent_b200.host import pipeline as P
    assert fake_pipeline([18, 26, 35, 45], per_peer_streams=True)[0].lanes == P.DEFAULT_LANES_STATEFUL
    assert fake_pipeline([18, 26, 35, 45])[0].lanes == P.DEFAULT_LANES_STATEFUL
    assert fake_pipeline([32], per_peer_streams=True)[0].lanes == P.DEFAULT_LANES_ONE_STEP
    assert fake_pipeline([32])[0].lanes == P.DEFAULT_LANES_ONE_STEP


@pytest.mark.parametrize("value,want", [(None, False), ("", False), ("0", False), ("false", False), ("Off", False),
                                        ("no", False), ("1", True), ("true", True), ("ON", True), (" yes ", True)])
def test_per_peer_streams_env_var(fake_pipeline, monkeypatch, value, want):
    from ai_rtc_agent_b200.host import pipeline as P
    if value is not None:
        monkeypatch.setenv(P.PER_PEER_STREAMS_ENV, value)
    assert P.env_flag(P.PER_PEER_STREAMS_ENV) is want
    assert fake_pipeline([18, 26, 35, 45])[0].per_peer_streams is want
    assert fake_pipeline([18, 26, 35, 45], per_peer_streams=not want)[0].per_peer_streams is (not want), "the argument wins"


def test_per_peer_streams_env_var_rejects_garbage(fake_pipeline, monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P
    monkeypatch.setenv(P.PER_PEER_STREAMS_ENV, "maybe")
    with pytest.raises(ValueError, match=P.PER_PEER_STREAMS_ENV):
        fake_pipeline([18, 26, 35, 45])


# ---- the track adapter ----------------------------------------------------------------------------------------------------------------
class EndOfSource(Exception):
    pass


class Source:
    def __init__(self, n):
        self.i, self.n = 0, n

    async def recv(self):
        await asyncio.sleep(0)
        if self.i >= self.n:
            raise EndOfSource()
        self.i += 1
        return ("frame", self.i)


class Ticket:
    def __init__(self, value):
        self.value, self.polls = value, 2

    def done(self):
        self.polls -= 1
        return self.polls < 0

    def result(self):
        return self.value


class RecordingPeer:
    def __init__(self, pipe):
        self.pipe, self.frames, self.closed = pipe, [], False

    def enqueue(self, frame):
        assert not self.closed
        self.frames.append(frame)
        return Ticket(("processed", frame[1]))

    def close(self):
        self.closed = True


class PerPeerPipeline:
    per_peer_streams = True

    def __init__(self):
        self.peers, self.direct = [], []

    def open_stream(self):
        self.peers.append(RecordingPeer(self))
        return self.peers[-1]

    def enqueue(self, frame):
        self.direct.append(frame)
        return Ticket(("processed", frame[1]))


def _drive(coro_fn):
    return asyncio.run(coro_fn())


def test_track_opens_one_stream_and_closes_it_on_stop(monkeypatch):
    monkeypatch.setenv("WARMUP_FRAMES", "2")
    monkeypatch.setenv("DROP_FRAMES", "0")
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = PerPeerPipeline()
    t1, t2 = VideoStreamTrack(Source(50), pipe), VideoStreamTrack(Source(50), pipe)

    async def go():
        return [await t1.recv() for _ in range(3)], [await t2.recv() for _ in range(2)]

    o1, o2 = _drive(go)
    assert o1 == [("processed", 3), ("processed", 4), ("processed", 5)] and o2 == [("processed", 3), ("processed", 4)]
    assert len(pipe.peers) == 2 and pipe.direct == [], "one stream per track; warm-up and later frames all go through it"
    assert [f[1] for f in pipe.peers[0].frames] == [1, 2, 3, 4, 5] and [f[1] for f in pipe.peers[1].frames] == [1, 2, 3, 4]
    t1.stop()
    assert pipe.peers[0].closed and not pipe.peers[1].closed
    t1.stop()                                   # idempotent
    t2.stop()
    assert pipe.peers[1].closed and len(pipe.peers) == 2


def test_track_closes_its_stream_when_the_source_ends(monkeypatch):
    monkeypatch.setenv("WARMUP_FRAMES", "1")
    monkeypatch.setenv("DROP_FRAMES", "0")
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = PerPeerPipeline()
    track = VideoStreamTrack(Source(3), pipe)

    async def go():
        outs = [await track.recv() for _ in range(2)]
        with pytest.raises(EndOfSource):
            await track.recv()
        return outs

    assert _drive(go) == [("processed", 2), ("processed", 3)]
    assert len(pipe.peers) == 1 and pipe.peers[0].closed


def test_track_without_per_peer_streams_uses_the_pipeline(monkeypatch):
    monkeypatch.setenv("WARMUP_FRAMES", "1")
    monkeypatch.setenv("DROP_FRAMES", "0")
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = PerPeerPipeline()
    pipe.per_peer_streams = False
    track = VideoStreamTrack(Source(5), pipe)

    async def go():
        return [await track.recv() for _ in range(2)]

    assert _drive(go) == [("processed", 2), ("processed", 3)]
    track.stop()
    assert pipe.peers == [] and [f[1] for f in pipe.direct] == [1, 2, 3]


# ---- C ABI ----------------------------------------------------------------------------------------------------------------------------
_C_TO_CTYPES = {"b2sd_handle": ctypes.c_void_p, "b2sd_state_handle": ctypes.c_void_p, "void*": ctypes.c_void_p,
                "const void*": ctypes.c_void_p, "int": ctypes.c_int, "b2sd_state_handle*": ctypes.POINTER(ctypes.c_void_p)}


@pytest.mark.parametrize("name", ["b2sd_state_create", "b2sd_state_reset", "b2sd_state_destroy", "b2sd_step_state"])
def test_state_call_ctypes_signatures_match_the_header(name):
    from ai_rtc_agent_b200.host import capi
    header = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared in include/b200sd.h"
    params = [re.sub(r"\s+", " ", p.strip()) for p in m.group(1).split(",")]
    want = []
    for p in params:
        ctype = re.sub(r"\s*\w+$", "", p).replace(" *", "*")   # drop the parameter name
        want.append(_C_TO_CTYPES[ctype])
    fn = getattr(capi.lib(), name)
    assert fn.restype is ctypes.c_int
    assert list(fn.argtypes) == want
    assert "typedef struct b2sd_state* b2sd_state_handle;" in header, "the state is an opaque handle, not a mirrored struct"


def test_state_calls_refuse_null_handles_without_a_device():
    from ai_rtc_agent_b200.host import capi
    lib = capi.lib()
    out = ctypes.c_void_p()
    assert lib.b2sd_state_create(None, ctypes.byref(out), None) != 0 and b"b2sd_prepare" in lib.b2sd_last_error()
    assert lib.b2sd_state_reset(None, None) != 0 and b"null state" in lib.b2sd_last_error()
    assert lib.b2sd_step_state(None, None, None, 0, 1, 1, None, 0, None) != 0
    assert lib.b2sd_state_destroy(None, None) == 0
