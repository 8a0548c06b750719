"""Per-peer prompts and t_index_lists without a GPU: the host bookkeeping of StreamDiffusion / StreamState over a recording fake
of the C library (per-key global updates, prepare, the t_index_list checks), the pipeline's routing of a peer's update to one
lane over fake engines, the track adapter's update methods, and the ctypes signatures and null-handle refusals of the calls."""
import contextlib
import ctypes
import os
import re
import types
import weakref

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T4 = [18, 26, 35, 45]


# ---- the real host classes over a recording fake of libb200sd -------------------------------------------------------------------
class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("b2sd_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name[5:],) + tuple(a.value if isinstance(a, ctypes.c_void_p) else a for a in args))
            return 0
        return call

    def named(self, name):
        return [c for c in self.calls if c[0] == name]


@pytest.fixture
def host(monkeypatch):
    """(root engine, new_state(), fake library): a StreamDiffusion and StreamStates built around FakeLib, no device"""
    from ai_rtc_agent_b200.host import stream as S
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    monkeypatch.setattr(S, "_on_device", lambda t, device: t.contiguous())   # pinned memory needs a driver
    monkeypatch.setattr(S, "_encode_beside", lambda eng, prompt: eng._encode(prompt)[0])   # streams need one too
    lib = FakeLib()
    eng = object.__new__(S.StreamDiffusion)
    eng.__dict__.update(
        _lib=lib, _handle=ctypes.c_void_p(1), lanes=[], _states=weakref.WeakSet(), _prepared=True, _ev=None,
        arch=types.SimpleNamespace(ctx_tokens=77, cross_attention_dim=8), prompt_encoder=SyntheticPromptEncoder(8),
        device=torch.device("cpu"), dtype=torch.float16, t_list=list(T4), denoising_steps_num=4, batch_size=4, frame_bff_size=1,
        cfg_type="self", latent_height=2, latent_width=2, generator=None)
    eng._stream = lambda: 0
    eng.prepare("global", guidance_scale=0.0)
    lane = object.__new__(S.StreamDiffusion)
    lane.__dict__.update(eng.__dict__, _handle=ctypes.c_void_p(2), lanes=[])
    lane._stream = lambda: 0
    eng.lanes.append(lane)
    states = []

    def new_state():
        st = object.__new__(S.StreamState)
        st.__dict__.update(_engine=eng, _lib=lib, _handle=ctypes.c_void_p(100 + len(states)))
        states.append(st)
        eng._states.add(st)
        return st
    lib.calls.clear()
    return eng, new_state, lib


def test_state_update_runs_on_the_given_engine_only(host):
    eng, new_state, lib = host
    a = new_state()
    a.set_prompt("a prompt", engine=eng.lanes[0])
    a.set_t_index_list([10, 20, 30, 40])
    assert [c[:3] for c in lib.calls] == [("state_set_prompt_embeds", 2, 100), ("state_set_timesteps", 1, 100)]
    assert not lib.named("set_prompt_embeds") and not lib.named("set_timesteps"), "the global conditioning is left alone"
    assert a.own_prompt == "a prompt" and a.own_t_index_list == [10, 20, 30, 40]


def test_state_prompt_is_encoded_beside_the_lane_stream(monkeypatch):
    """The encoder runs on the engine's encoder stream, never on the (lane) stream current at the call, which may have frames
    queued: an encoder that synchronises its stream would wait for them.  The current stream then waits for the embedding only."""
    from ai_rtc_agent_b200.host import stream as S
    log, cur = [], []

    class Stream:
        def __init__(self, *a, name="encoder", **k):
            self.name = name

        def wait_event(self, ev):
            log.append(("wait", self.name, ev.on))

    class Event:
        def record(self, stream):
            self.on = stream.name
            log.append(("record", stream.name))

    class Emb:
        def record_stream(self, stream):
            log.append(("record_stream", stream.name))

    @contextlib.contextmanager
    def on(stream):
        cur.append(stream)
        try:
            yield
        finally:
            cur.pop()
    cur.append(Stream(name="lane"))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: cur[-1])
    monkeypatch.setattr(torch.cuda, "Stream", Stream)
    monkeypatch.setattr(torch.cuda, "Event", Event)
    monkeypatch.setattr(torch.cuda, "stream", on)
    monkeypatch.setattr(S, "_on_device", lambda t, device: Emb())
    eng = object.__new__(S.StreamDiffusion)
    eng.device = "cpu"
    eng._encode = lambda prompt: log.append(("encode", cur[-1].name)) or [prompt]
    S._encode_beside(eng, "x")
    S._encode_beside(eng, "y")
    once = [("encode", "encoder"), ("record", "encoder"), ("wait", "lane", "encoder"), ("record_stream", "lane")]
    assert log == once + once and eng._encoder_stream() is eng._encoder_stream()


def test_state_t_index_list_is_checked_like_the_global_one(host):
    eng, new_state, lib = host
    a = new_state()
    eng.sub_timesteps = [eng.timesteps[t] for t in [10, 20, 30]]
    with pytest.raises(ValueError) as glob:
        eng.sync_timesteps()
    with pytest.raises(ValueError) as own:
        a.set_t_index_list([10, 20, 30])
    assert str(own.value) == str(glob.value)
    with pytest.raises(IndexError):
        a.set_t_index_list([10, 20, 30, 99])
    assert a.own_t_index_list is None and not lib.named("state_set_timesteps")


def test_global_updates_clear_only_their_own_key(host):
    from ai_rtc_agent_b200.host import capi
    eng, new_state, lib = host
    a, b, c = new_state(), new_state(), new_state()
    a.set_prompt("a")
    b.set_t_index_list([10, 20, 30, 40])
    lib.calls.clear()
    eng.update_prompt("new global")
    assert [x[1] for x in lib.named("set_prompt_embeds")] == [1, 2], "the root and its lane"
    assert sorted(x[1:] for x in lib.named("state_clear_conditioning")) == [(100, capi.COND_PROMPT), (101, capi.COND_PROMPT),
                                                                             (102, capi.COND_PROMPT)]
    assert a.own_prompt is None and b.own_t_index_list == [10, 20, 30, 40] and eng.prompt == eng.lanes[0].prompt == "new global"
    lib.calls.clear()
    eng.sync_timesteps()
    assert sorted(x[1:] for x in lib.named("state_clear_conditioning")) == [(100, capi.COND_TIME), (101, capi.COND_TIME),
                                                                             (102, capi.COND_TIME)]
    assert b.own_t_index_list is None


def test_prepare_clears_every_override(host):
    eng, new_state, lib = host
    a, b = new_state(), new_state()
    a.set_prompt("a")
    a.set_t_index_list([10, 20, 30, 40])
    b.set_prompt("b")
    b.close()
    lib.calls.clear()
    eng.prepare("fresh", guidance_scale=0.0)
    assert sorted(x[1:] for x in lib.named("state_clear_conditioning")) == [(100, 0), (100, 1)], "live states only"
    assert lib.named("state_reset") == [("state_reset", 100, 0)]
    assert a.own_prompt is None and a.own_t_index_list is None and eng.prompt == "fresh"


def test_closed_state_refuses_updates(host):
    _, new_state, lib = host
    a = new_state()
    a.close()
    for fn in (lambda: a.set_prompt("x"), lambda: a.set_t_index_list(T4), lambda: a.clear_overrides()):
        with pytest.raises(RuntimeError, match="closed"):
            fn()
    assert not lib.named("state_set_prompt_embeds")


# ---- the pipeline over fake engines ------------------------------------------------------------------------------------------
class FakeStream:
    def __init__(self, *a, **k):
        self.waits = 0

    def wait_event(self, ev):
        self.waits += 1


class FakeEvent:
    def record(self, stream=None):
        pass

    def query(self):
        return True

    def synchronize(self):
        pass


class FakeState:
    def __init__(self, log, n):
        self.log, self.n, self.closed = log, n, False
        self.own_prompt = self.own_t_index_list = None

    def reset(self):
        pass

    def close(self):
        self.closed = True

    def set_prompt(self, prompt, engine):
        self.log.append(("prompt", self.n, prompt, engine.lane, CURRENT[0]))
        self.own_prompt = prompt

    def set_t_index_list(self, t_index_list, engine):
        self.log.append(("t_index_list", self.n, list(t_index_list), engine.lane, CURRENT[0]))
        self.own_t_index_list = list(t_index_list)

    def clear_overrides(self, prompt=True, t_index_list=True):
        if prompt:
            self.own_prompt = None
        if t_index_list:
            self.own_t_index_list = None


class FakeOut:
    def record_stream(self, stream):
        pass


class FakeEngine:
    def __init__(self, log, lane=0, states=None):
        self.log, self.lane, self.lanes, self.device = log, lane, [], "cpu"
        self.states = [] if states is None else states
        self.prompt, self.t_list = "global", list(T4)

    def set_concurrency(self, n):
        pass

    def add_lane(self):
        self.lanes.append(FakeEngine(self.log, len(self.lanes) + 1, self.states))
        return self.lanes[-1]

    def new_state(self):
        self.states.append(FakeState(self.log, len(self.states)))
        return self.states[-1]

    def step_u8(self, rgb, state=None):
        self.log.append(("step", state.n if state else None, rgb, self.lane, CURRENT[0]))
        return FakeOut()

    def update_prompt(self, prompt):          # StreamDiffusion.update_prompt's effect on the states
        self.prompt = prompt
        self.clear_overrides(prompt=True, t_index_list=False)

    def clear_overrides(self, prompt=True, t_index_list=True):
        for s in self.states:
            if not s.closed:
                s.clear_overrides(prompt=prompt, t_index_list=t_index_list)


CURRENT = [None]


@pytest.fixture
def fake_pipeline(monkeypatch):
    """make(t_index_list, **kw) -> (pipeline over fake engines, log); torch.cuda.stream(s) makes s current in CURRENT"""
    from ai_rtc_agent_b200.host import pipeline as P
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    monkeypatch.delenv("B200SD_POLICY_FRAMES", raising=False)
    monkeypatch.delenv(P.PER_PEER_STREAMS_ENV, raising=False)
    monkeypatch.setattr(torch.cuda, "Stream", FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    caller = FakeStream()
    CURRENT[0] = caller
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: CURRENT[0])

    @contextlib.contextmanager
    def on(stream):
        prev, CURRENT[0] = CURRENT[0], stream
        try:
            yield
        finally:
            CURRENT[0] = prev
    monkeypatch.setattr(torch.cuda, "stream", on)
    monkeypatch.setattr(P, "_is_gpu_frame", lambda f: True)

    class Frame:
        def __init__(self, f):
            self.f = f

        def record_stream(self, stream):
            pass
    monkeypatch.setattr(P, "_as_torch_u8_nhwc", lambda f, d: f if isinstance(f, Frame) else Frame(f))
    log = []

    class FakeWrapper:
        def __init__(self, t_index_list, width, height, **kw):
            self.stream = FakeEngine(log)
            self.height, self.width = height, width

        def prepare(self, **kw):
            pass

        def update_t_index_list(self, t_index_list):   # the wrapper returns early when the list is unchanged
            if t_index_list != self.stream.t_list:
                self.stream.t_list = list(t_index_list)
                self.stream.clear_overrides(prompt=False, t_index_list=True)

    monkeypatch.setattr(P, "StreamDiffusionWrapper", FakeWrapper)

    def make(t_index_list, **kw):
        return P.StreamDiffusionPipeline("tiny-sd15", t_index_list=t_index_list, width=64, height=64, **kw), log
    return make


def test_peer_update_runs_on_the_next_lane_and_waits_on_no_other(fake_pipeline):
    pipe, log = fake_pipeline(T4, per_peer_streams=True, lanes=3)
    a, b = pipe.open_stream(), pipe.open_stream()
    for who in (a, b, a, b):
        who.enqueue("f")
    waits = [s.waits for s in pipe._lane_streams]
    log.clear()
    a.update_prompt("mine")                 # the next submission goes to lane 1
    b.update_t_index_list([10, 20, 30, 40])
    assert log == [("prompt", a._state.n, "mine", 1, pipe._lane_streams[1]),
                   ("t_index_list", b._state.n, [10, 20, 30, 40], 1, pipe._lane_streams[1])]
    assert [s.waits for s in pipe._lane_streams] == waits, "no lane stream waits on another"
    assert pipe._next_lane == 1, "an update is not a submission"
    b.enqueue("f")
    assert log[-1][3] == 1
    assert (a.prompt, a.t_index_list, b.prompt, b.t_index_list) == ("mine", T4, "global", [10, 20, 30, 40])


def test_one_lane_updates_on_the_callers_stream(fake_pipeline):
    pipe, log = fake_pipeline([32], per_peer_streams=True, lanes=1)
    a = pipe.open_stream()
    a.update_prompt("mine")
    assert log == [("prompt", a._state.n, "mine", 0, CURRENT[0])]


def test_new_stream_starts_from_the_global_values(fake_pipeline):
    pipe, _ = fake_pipeline(T4, per_peer_streams=True, lanes=2)
    pipe.update_prompt("later global")
    pipe.update_t_index_list([10, 20, 30, 40])
    s = pipe.open_stream()
    assert s.prompt == "later global" and s.t_index_list == [10, 20, 30, 40]
    assert s._state.own_prompt is None and s._state.own_t_index_list is None


def test_global_updates_are_per_key(fake_pipeline):
    pipe, _ = fake_pipeline(T4, per_peer_streams=True, lanes=2)
    a, b, c = pipe.open_stream(), pipe.open_stream(), pipe.open_stream()
    a.update_prompt("a")
    b.update_t_index_list([10, 20, 30, 40])
    pipe.update_prompt("g")
    assert [s.prompt for s in (a, b, c)] == ["g"] * 3
    assert b.t_index_list == [10, 20, 30, 40] and a.t_index_list == T4
    a.update_prompt("a2")
    pipe.update_t_index_list(T4)                 # unchanged global list: still every stream's from now on
    assert [s.t_index_list for s in (a, b, c)] == [T4] * 3 and a.prompt == "a2"


def test_closed_peer_stream_refuses_updates(fake_pipeline):
    pipe, log = fake_pipeline(T4, per_peer_streams=True, lanes=2)
    a = pipe.open_stream()
    a.close()
    for fn in (lambda: a.update_prompt("x"), lambda: a.update_t_index_list(T4)):
        with pytest.raises(RuntimeError, match="the peer stream is closed"):
            fn()
    assert log == []


# ---- the track adapter ----------------------------------------------------------------------------------------------------------
class RecordingTarget:
    def __init__(self):
        self.updates, self.closed = [], False

    def update_prompt(self, prompt):
        self.updates.append(("prompt", prompt))

    def update_t_index_list(self, t_index_list):
        self.updates.append(("t_index_list", t_index_list))

    def close(self):
        self.closed = True


class Pipeline(RecordingTarget):
    def __init__(self, per_peer):
        super().__init__()
        self.per_peer_streams, self.peers = per_peer, []

    def open_stream(self):
        self.peers.append(RecordingTarget())
        return self.peers[-1]


def test_track_updates_its_own_stream_before_any_frame():
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = Pipeline(True)
    t1, t2 = VideoStreamTrack(None, pipe), VideoStreamTrack(None, pipe)
    t1.update_prompt("one")
    t1.update_t_index_list([10, 20, 30, 40])
    t2.update_prompt("two")
    assert len(pipe.peers) == 2 and pipe.updates == []
    assert pipe.peers[0].updates == [("prompt", "one"), ("t_index_list", [10, 20, 30, 40])]
    assert pipe.peers[1].updates == [("prompt", "two")]
    assert t1._target() is pipe.peers[0], "frames then use the stream the update opened"


def test_track_without_per_peer_streams_updates_the_pipeline():
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = Pipeline(False)
    t = VideoStreamTrack(None, pipe)
    t.update_prompt("all")
    t.update_t_index_list([10, 20, 30, 40])
    assert pipe.updates == [("prompt", "all"), ("t_index_list", [10, 20, 30, 40])] and pipe.peers == []


@pytest.mark.parametrize("per_peer", [True, False])
def test_track_updates_after_stop_are_ignored(per_peer):
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack
    pipe = Pipeline(per_peer)
    t = VideoStreamTrack(None, pipe)
    if per_peer:
        t.update_prompt("before")
    t.stop()
    t.update_prompt("late")
    t.update_t_index_list([10, 20, 30, 40])
    assert pipe.updates == [] and len(pipe.peers) == (1 if per_peer else 0)
    if per_peer:
        assert pipe.peers[0].updates == [("prompt", "before")] and pipe.peers[0].closed


# ---- C ABI ----------------------------------------------------------------------------------------------------------------------
_C_TO_CTYPES = {"b2sd_handle": ctypes.c_void_p, "b2sd_state_handle": ctypes.c_void_p, "void*": ctypes.c_void_p,
                "const void*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "int": ctypes.c_int}


@pytest.mark.parametrize("name,restype", [("b2sd_state_set_prompt_embeds", ctypes.c_int), ("b2sd_state_set_timesteps", ctypes.c_int),
                                          ("b2sd_state_clear_conditioning", ctypes.c_int),
                                          ("b2sd_conditioning_binds", ctypes.c_int64)])
def test_conditioning_call_ctypes_signatures_match_the_header(name, restype):
    from ai_rtc_agent_b200.host import capi
    header = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    m = re.search(r"\b(int|int64_t)\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared in include/b200sd.h"
    assert {"int": ctypes.c_int, "int64_t": ctypes.c_int64}[m.group(1)] is restype
    want = []
    for p in (re.sub(r"\s+", " ", p.strip()) for p in m.group(2).split(",")):
        want.append(_C_TO_CTYPES[re.sub(r"\s*\w+$", "", p).replace(" *", "*")])
    fn = getattr(capi.lib(), name)
    assert fn.restype is restype and list(fn.argtypes) == want


def test_conditioning_calls_refuse_null_handles_without_a_device():
    from ai_rtc_agent_b200.host import capi
    lib = capi.lib()
    assert lib.b2sd_state_set_prompt_embeds(None, None, None, None) != 0 and b"b2sd_prepare" in lib.b2sd_last_error()
    assert lib.b2sd_state_set_timesteps(None, None, None, None) != 0 and b"b2sd_prepare" in lib.b2sd_last_error()
    assert lib.b2sd_state_clear_conditioning(None, 0) != 0 and b"null state" in lib.b2sd_last_error()
    assert lib.b2sd_conditioning_binds(None) == -1
