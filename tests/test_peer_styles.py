"""Per-viewer style LoRAs without a GPU: the pipeline's style pool over fake engines (style keys, routing of each viewer's frames
to its style's lanes, sharing, LRU eviction and the capacity refusal, global updates), the track adapter's update_lora, and
the ctypes signatures and null-handle refusals of b2sd_create_style / b2sd_release."""
import contextlib
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T4 = [18, 26, 35, 45]
CURRENT = [None]


class FakeStream:
    def __init__(self, *a, **k):
        self.waits = 0

    def wait_event(self, ev):
        self.waits += 1

    def wait_stream(self, other):
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

    def close(self):
        self.closed = True

    def set_prompt(self, prompt, engine):
        self.log.append(("prompt", self.n, prompt, engine.name))
        self.own_prompt = prompt

    def set_t_index_list(self, t_index_list, engine):
        self.log.append(("t_index_list", self.n, list(t_index_list), engine.name))
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
    """StreamDiffusion's style / lane / global-update surface, recording into log"""

    def __init__(self, log, name, states):
        self.log, self.name, self.states = log, name, states
        self.lanes, self.styles, self.device = [], [], "cpu"
        self.prompt, self.t_list, self.live_lora, self._unet_shapes = "global", list(T4), True, {}
        self.lora = None

    def set_concurrency(self, n):
        pass

    def add_lane(self):
        self.lanes.append(FakeEngine(self.log, f"{self.name}.{len(self.lanes) + 1}", self.states))
        self.lanes[-1].lora = self.lora
        return self.lanes[-1]

    def add_style(self):
        self.made = getattr(self, "made", 0) + 1
        self.styles.append(FakeEngine(self.log, f"style{self.made - 1}", self.states))
        self.styles[-1].prompt, self.styles[-1].t_list = self.prompt, list(self.t_list)
        self.log.append(("add_style", self.styles[-1].name))
        return self.styles[-1]

    def drop_style(self, style, after):
        self.styles.remove(style)
        self.log.append(("drop_style", style.name))

    def apply_factors(self, factors):
        for e in [self] + self.lanes:
            e.lora = factors

    def new_state(self):
        self.states.append(FakeState(self.log, len(self.states)))
        return self.states[-1]

    def step_u8(self, rgb, state=None):
        self.log.append(("step", state.n if state else None, self.name, self.lora))
        return FakeOut()

    def _family(self):
        return [self] + self.lanes + [e for st in self.styles for e in [st] + st.lanes]

    def update_prompt(self, prompt):          # StreamDiffusion.update_prompt: every engine of the family, every state
        for e in self._family():
            e.prompt = prompt
        self.clear_overrides(prompt=True, t_index_list=False)

    def clear_overrides(self, prompt=True, t_index_list=True):
        for s in self.states:
            if not s.closed:
                s.clear_overrides(prompt=prompt, t_index_list=t_index_list)


@pytest.fixture
def styles(monkeypatch, tmp_path):
    """make(t_index_list, **kw) -> (per-peer live-LoRA pipeline over fake engines, log, lora file paths a, b, c)"""
    from ai_rtc_agent_b200.host import pipeline as P
    from ai_rtc_agent_b200.host import weights as W
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.setenv("B200SD_LIVE_LORA", "1")
    for v in ("B200SD_LANES", "B200SD_POLICY_FRAMES", P.MAX_STYLES_ENV):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setattr(torch.cuda, "Stream", FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    CURRENT[0] = FakeStream()
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
    monkeypatch.setattr(P, "_as_torch_u8_nhwc", lambda f, d: FakeOut())
    log = []

    def factors(shapes, lora_dict):          # what lora_factors checks: readable files
        for path in lora_dict or {}:
            if open(path).read() == "bad":
                raise ValueError(f"{path}: not a safetensors file")
        return tuple((os.path.basename(p), s) for p, s in (lora_dict or {}).items())
    monkeypatch.setattr(W, "lora_factors", factors)

    class FakeWrapper:
        live_lora = True

        def __init__(self, t_index_list, width, height, **kw):
            self.stream = FakeEngine(log, "pipe", [])
            self.height, self.width = height, width

        def prepare(self, **kw):
            pass

        def update_lora(self, lora_dict):
            self.stream.apply_factors(factors(None, lora_dict))

        def update_t_index_list(self, t_index_list):
            for e in self.stream._family():
                e.t_list = list(t_index_list)
            self.stream.clear_overrides(prompt=False, t_index_list=True)

    monkeypatch.setattr(P, "StreamDiffusionWrapper", FakeWrapper)
    paths = []
    for name in "abc":
        paths.append(str(tmp_path / f"{name}.safetensors"))
        open(paths[-1], "w").write(name)

    def make(t_index_list=T4, **kw):
        kw.setdefault("per_peer_streams", True)
        return P.StreamDiffusionPipeline("tiny-sd15", t_index_list=t_index_list, width=64, height=64, **kw), log
    return make, paths


def test_style_key_follows_order_scale_and_file(tmp_path):
    from ai_rtc_agent_b200.host.pipeline import style_key
    a, b = str(tmp_path / "a.safetensors"), str(tmp_path / "b.safetensors")
    open(a, "w").write("a")
    open(b, "w").write("b")
    k = style_key({a: 1.0, b: 0.5})
    assert style_key({a: 1, b: 0.5}) == k and style_key(dict([(a, 1.0), (b, 0.5)])) == k
    assert style_key({b: 0.5, a: 1.0}) != k, "LoRAs fuse in order: another order is another style"
    assert style_key({a: 1.0, b: 0.25}) != k
    os.symlink(a, str(tmp_path / "link.safetensors"))
    assert style_key({str(tmp_path / "link.safetensors"): 1.0, b: 0.5}) == k, "a path is its real path"
    st = os.stat(a)
    os.utime(a, ns=(st.st_atime_ns, st.st_mtime_ns + 10 ** 9))
    assert style_key({a: 1.0, b: 0.5}) != k, "a replaced file is another style"
    assert style_key(None) == style_key({}) == ()
    with pytest.raises(FileNotFoundError):
        style_key({str(tmp_path / "missing.safetensors"): 1.0})


def test_frames_go_to_their_styles_lanes_only(styles):
    make, (a, b, _) = styles
    pipe, log = make()
    v0, v1, v2, v3 = (pipe.open_stream() for _ in range(4))
    v1.update_lora({a: 1.0})
    v2.update_lora({b: 1.0})
    v3.update_lora({a: 1.0})
    assert pipe.styles == 2, "two viewers with one dict share one style"
    assert v1._style is v3._style and v1._style is not v2._style
    log.clear()
    for _ in range(3):
        for v in (v0, v1, v2, v3):
            v.enqueue("f")
    steps = [c for c in log if c[0] == "step"]
    by_state = {}
    for _, n, engine, lora in steps:
        by_state.setdefault(n, set()).add((engine.split(".")[0], lora))
    assert by_state[v0._state.n] == {("pipe", None)}
    assert by_state[v1._state.n] == by_state[v3._state.n] == {("style0", (("a.safetensors", 1.0),))}
    assert by_state[v2._state.n] == {("style1", (("b.safetensors", 1.0),))}
    lanes = {engine for _, n, engine, _ in steps if n in (v1._state.n, v3._state.n)}
    assert lanes == {"style0", "style0.1"}, "a style's viewers rotate over its lanes"
    assert v1.lora == {a: 1.0} and v0.lora == {}


def test_switch_carries_own_conditioning_to_the_new_lanes(styles):
    make, (a, _, _) = styles
    pipe, log = make()
    v = pipe.open_stream()
    v.update_prompt("mine")
    v.update_t_index_list([10, 20, 30, 40])
    log.clear()
    v.update_lora({a: 1.0})
    assert [c for c in log if c[0] in ("prompt", "t_index_list")] == [
        ("prompt", v._state.n, "mine", "style0"), ("t_index_list", v._state.n, [10, 20, 30, 40], "style0")]
    log.clear()
    v.update_prompt("mine2")                     # later own updates run on the style's lanes
    assert log == [("prompt", v._state.n, "mine2", "style0")]
    log.clear()
    v.update_lora(None)                          # the global dict: back on the pipeline's lanes
    assert v._style is None and [c[3] for c in log if c[0] == "prompt"] == ["pipe"]
    assert pipe.styles == 1, "an unused style stays cached"


def test_the_global_dict_makes_no_style(styles):
    make, (a, _, _) = styles
    pipe, log = make()
    pipe.update_lora({a: 1.0})
    v = pipe.open_stream()
    v.update_lora({a: 1.0})
    assert pipe.styles == 0 and v._style is None and v.lora == {a: 1.0}
    v.update_lora({})                            # the base weights are a style once the global dict is not empty
    assert pipe.styles == 1 and v.lora == {}


def test_lru_eviction_and_capacity_refusal(styles, monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P
    make, (a, b, c) = styles
    monkeypatch.setenv(P.MAX_STYLES_ENV, "2")
    pipe, log = make()
    v1, v2 = pipe.open_stream(), pipe.open_stream()
    v1.update_lora({a: 1.0})
    v2.update_lora({b: 1.0})
    v1.update_lora(None)                         # style a unused, cached
    v2.update_lora({a: 1.0})                     # a again: a cache hit, b now unused and least recently used
    assert [c for c in log if c[0] == "add_style"] == [("add_style", "style0"), ("add_style", "style1")]
    v1.update_lora({c: 1.0})                     # room for c: b goes
    assert ("drop_style", "style1") in log and pipe.styles == 2
    assert {s.lora_dict == {c: 1.0} or s.lora_dict == {a: 1.0} for s in pipe._styles.values()} == {True}
    before = (list(pipe._styles), v1._style, v2._style, len(log))
    v3 = pipe.open_stream()
    with pytest.raises(RuntimeError, match="in use"):
        v3.update_lora({b: 1.0})
    assert (list(pipe._styles), v1._style, v2._style, len(log)) == before and v3._style is None
    v1.close()                                   # closing frees its style for eviction
    v3.update_lora({b: 1.0})
    assert pipe.styles == 2 and v3._style.lora_dict == {b: 1.0}
    v3.update_lora({c: 1.0})                     # v3 alone uses b: leaving it makes the room, b goes after the switch
    assert pipe.styles == 2 and v3._style.lora_dict == {c: 1.0} and ("drop_style", "style3") in log


def test_eviction_waits_for_a_successful_build(styles, monkeypatch):
    """a build that fails on the device leaves the cached styles as they were; a successful one evicts only afterwards, so
    the pool holds one style more during the build"""
    from ai_rtc_agent_b200.host import pipeline as P
    make, (a, b, c) = styles
    monkeypatch.setenv(P.MAX_STYLES_ENV, "1")
    pipe, log = make()
    v = pipe.open_stream()
    v.update_lora({a: 1.0})
    v.update_lora(None)                          # a: unused, cached
    held = []
    real = FakeEngine.add_style

    def failing(self):
        raise RuntimeError("device allocation failed")
    monkeypatch.setattr(FakeEngine, "add_style", failing)
    with pytest.raises(RuntimeError, match="allocation"):
        v.update_lora({b: 1.0})
    assert list(pipe._styles) and [s.lora_dict for s in pipe._styles.values()] == [{a: 1.0}] and v._style is None

    def counting(self):
        held.append(len(pipe._styles))
        return real(self)
    monkeypatch.setattr(FakeEngine, "add_style", counting)
    v.update_lora({b: 1.0})
    assert held == [1] and [s.lora_dict for s in pipe._styles.values()] == [{b: 1.0}]
    assert log.index(("drop_style", "style0")) > log.index(("add_style", "style1"))


def test_a_dropped_viewer_frees_its_style(styles, monkeypatch):
    import gc
    from ai_rtc_agent_b200.host import pipeline as P
    make, (a, b, _) = styles
    monkeypatch.setenv(P.MAX_STYLES_ENV, "1")
    pipe, log = make()
    v = pipe.open_stream()
    v.update_lora({a: 1.0})
    state = v._state
    del v                                        # never closed
    gc.collect()
    assert state.closed and next(iter(pipe._styles.values())).users == 0
    w = pipe.open_stream()
    w.update_lora({b: 1.0})                      # room: a is unused
    assert [s.lora_dict for s in pipe._styles.values()] == [{b: 1.0}]


def test_refusals_change_nothing(styles):
    make, (a, b, _) = styles
    pipe, log = make()
    v = pipe.open_stream()
    v.update_lora({a: 1.0})
    open(b, "w").write("bad")
    before = (list(pipe._styles), v._style, len(log))
    with pytest.raises(ValueError, match="not a safetensors"):
        v.update_lora({b: 1.0})
    with pytest.raises(FileNotFoundError):
        v.update_lora({b + ".missing": 1.0})
    assert (list(pipe._styles), v._style, len(log)) == before
    v.close()
    with pytest.raises(RuntimeError, match="the peer stream is closed"):
        v.update_lora({a: 1.0})
    off, _ = make(live_lora=False)
    with pytest.raises(RuntimeError, match="live_lora=True"):
        off.open_stream().update_lora({a: 1.0})


def test_global_updates_reach_styles(styles):
    make, (a, b, _) = styles
    pipe, log = make()
    v1, v2 = pipe.open_stream(), pipe.open_stream()
    v1.update_lora({a: 1.0})
    v1.update_prompt("own")
    pipe.update_prompt("g")
    assert {e.prompt for e in pipe.model.stream._family()} == {"g"} and v1.prompt == "g"
    pipe.update_t_index_list([10, 20, 30, 40])
    assert {tuple(e.t_list) for e in pipe.model.stream._family()} == {(10, 20, 30, 40)}
    waits = [s.waits for s in v1._style._lane_streams]
    pipe.update_prompt("g2")
    assert all(w2 > w1 for w1, w2 in zip(waits, [s.waits for s in v1._style._lane_streams])), \
        "style lanes are released after a global update"
    pipe.update_lora({b: 1.0})                   # drops every viewer's own style; the styles stay cached
    assert v1._style is None and v1.lora == {b: 1.0} and pipe.styles == 1 and pipe._styles[next(iter(pipe._styles))].users == 0
    log.clear()
    v1.enqueue("f")
    assert log[-1][2].startswith("pipe")


def test_track_routes_update_lora():
    from ai_rtc_agent_b200.host.tracks import VideoStreamTrack

    class Target:
        def __init__(self):
            self.updates, self.closed, self.peers = [], False, []

        def update_lora(self, d):
            self.updates.append(d)

        def close(self):
            self.closed = True

    class Pipe(Target):
        def __init__(self, per_peer):
            super().__init__()
            self.per_peer_streams = per_peer

        def open_stream(self):
            self.peers.append(Target())
            return self.peers[-1]
    pipe = Pipe(True)
    t = VideoStreamTrack(None, pipe)
    t.update_lora({"a": 1.0})
    assert pipe.updates == [] and pipe.peers[0].updates == [{"a": 1.0}]
    t.stop()
    t.update_lora({"b": 1.0})
    assert pipe.peers[0].updates == [{"a": 1.0}]
    g = Pipe(False)
    VideoStreamTrack(None, g).update_lora(None)
    assert g.updates == [None] and g.peers == []


_C_TO_CTYPES = {"b2sd_handle": ctypes.c_void_p, "b2sd_handle*": ctypes.POINTER(ctypes.c_void_p), "void*": ctypes.c_void_p}


@pytest.mark.parametrize("name", ["b2sd_create_style", "b2sd_release"])
def test_style_call_ctypes_signatures_match_the_header(name):
    from ai_rtc_agent_b200.host import capi
    header = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared in include/b200sd.h"
    want = [_C_TO_CTYPES[re.sub(r"\s*\w+$", "", re.sub(r"\s+", " ", p.strip())).replace(" *", "*")] for p in m.group(1).split(",")]
    fn = getattr(capi.lib(), name)
    assert fn.restype is ctypes.c_int and list(fn.argtypes) == want


def test_style_calls_refuse_null_handles_without_a_device():
    from ai_rtc_agent_b200.host import capi
    lib = capi.lib()
    out = ctypes.c_void_p()
    assert lib.b2sd_create_style(None, ctypes.byref(out)) != 0 and b"null argument" in lib.b2sd_last_error()
    assert not out.value
    assert lib.b2sd_release(None, None) == 0, "releasing nothing is a no-op, like b2sd_destroy"
