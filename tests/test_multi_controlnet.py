"""Several ControlNets (diffusers' MultiControlNetModel), without a GPU: the per-net slot masks against diffusers'
controlnet_keep loop, the broadcasting and checks with diffusers' messages, the wrapper's and the pipeline's list arguments, the
blob keys and synthetic seeds, the extended b2sd_config layout, which per-net settings the host layer gives every viewer through
a random sequence of updates, and the multi-net restatement against the single-net one."""
import ctypes
import random
import types
import weakref

import pytest
import torch

T4 = [18, 26, 35, 45]


def diffusers_cond_scales(scales, starts, ends, n_steps):
    """StableDiffusionControlNetPipeline.__call__ with a MultiControlNetModel: controlnet_keep, then step i's cond_scale per
    net, restated from upstream"""
    timesteps = list(range(n_steps))
    controlnet_keep = []
    for i in range(len(timesteps)):
        keeps = [1.0 - float(i / len(timesteps) < s or (i + 1) / len(timesteps) > e) for s, e in zip(starts, ends)]
        controlnet_keep.append(keeps)
    return [[c * s for c, s in zip(scales, controlnet_keep[i])] for i in range(n_steps)]


def test_per_net_masks_are_diffusers_controlnet_keep():
    from ai_rtc_agent_b200.host.stream import check_controls, control_vector
    rng = random.Random(3)
    windows = [(0.0, 1.0), (0.0, 0.5), (0.5, 1.0), (0.2, 0.8), (0.98, 1.0), (0.0, 0.02), (0.36, 0.72)]
    for n in range(1, 51):
        for nets in range(1, 5):
            for _ in range(4):
                w = [rng.choice(windows) for _ in range(nets)]
                scales = [rng.choice([1.0, 0.6, -0.5, 0.0, 1.3]) for _ in range(nets)]
                t = sorted(rng.sample(range(n), min(n, rng.randint(1, 4))))
                want = diffusers_cond_scales(scales, [a for a, _ in w], [b for _, b in w], n)
                if nets == 1:
                    control = check_controls(scales[0], w[0][0], w[0][1], 1)
                else:
                    control = check_controls(scales, [a for a, _ in w], [b for _, b in w], nets)
                got = control_vector(control, t, n)
                assert got == [want[i][k] for k in range(nets) for i in t], (n, nets, w, scales, t)


def test_broadcasting():
    from ai_rtc_agent_b200.host.stream import check_controls
    assert check_controls(0.5, 0.0, 1.0, 1) == (0.5, 0.0, 1.0)
    assert check_controls(0.5, 0.0, 1.0, 3) == ((0.5,) * 3, (0.0,) * 3, (1.0,) * 3)
    assert check_controls([0.5, 1.0], 0.2, [0.6, 0.9], 2) == ((0.5, 1.0), (0.2, 0.2), (0.6, 0.9))
    assert check_controls(1.0, [0.1, 0.3], 0.8, 2) == ((1.0, 1.0), (0.1, 0.3), (0.8, 0.8))
    # taken back by set_control_scale(*settings)
    s = check_controls([0.5, 1.0], [0.0, 0.5], 1.0, 2)
    assert check_controls(*s, nets=2) == s


@pytest.mark.parametrize("args,match", [
    (([1.0, 0.5, 0.2], 0.0, 1.0), "must have the same length as the number of controlnets"),
    (([[1.0, 0.5], [0.2, 0.8]], 0.0, 1.0), "A single batch of varying conditioning scale settings"),
    ((1.0, [0.0, 0.1], [1.0]), "`control_guidance_start` has 2 elements, but `control_guidance_end` has 1 elements"),
    ((1.0, [0.0, 0.1, 0.2], 1.0), r"has 3 elements but there are 2 controlnets available. Make sure to provide 2."),
    ((1.0, [0.0, 0.6], [1.0, 0.4]), "cannot be larger or equal to control guidance end"),
    ((1.0, [-0.1, 0.0], 1.0), "can't be smaller than 0"),
    ((1.0, 0.0, [1.0, 1.1]), "can't be larger than 1.0"),
    (([1.0, float("nan")], 0.0, 1.0), "finite"),
])
def test_checks_use_diffusers_messages(args, match):
    from ai_rtc_agent_b200.host.stream import check_controls
    with pytest.raises(ValueError, match=match):
        check_controls(*args, nets=2)


# ---- wrapper and pipeline arguments -------------------------------------------------------------------------------------------
def _load_model_calls(monkeypatch, **kw):
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    calls = []
    monkeypatch.setattr(StreamDiffusionWrapper, "_load_model", lambda self, **a: calls.append(a) or None)
    StreamDiffusionWrapper("tiny-turbo", [32], **kw)
    return calls[-1]


def test_a_list_of_one_is_the_plain_value(monkeypatch):
    plain = _load_model_calls(monkeypatch, controlnet_id_or_path="cn", controlnet_processor_id="hed")
    for kw in (dict(controlnet_id_or_path=["cn"]), dict(controlnet_id_or_path=["cn"], controlnet_processor_id=["hed"]),
               dict(controlnet_id_or_path="cn", controlnet_processor_id=["hed"])):
        assert _load_model_calls(monkeypatch, **kw) == plain, kw
    frame = _load_model_calls(monkeypatch, controlnet_id_or_path=["cn"], controlnet_processor_id=[None])
    assert (frame["controlnet_id_or_path"], frame["controlnet_processor_id"]) == ("cn", None)


def test_lists_and_a_shared_processor(monkeypatch):
    got = _load_model_calls(monkeypatch, controlnet_id_or_path=["a", "b"], controlnet_processor_id=[None, "hed"])
    assert (got["controlnet_id_or_path"], got["controlnet_processor_id"]) == (["a", "b"], [None, "hed"])
    got = _load_model_calls(monkeypatch, controlnet_id_or_path=("a", "b", "c"))   # the default "hed" for every net
    assert (got["controlnet_id_or_path"], got["controlnet_processor_id"]) == (["a", "b", "c"], ["hed"] * 3)
    with pytest.raises(ValueError, match="3 entries for 2"):
        _load_model_calls(monkeypatch, controlnet_id_or_path=["a", "b"], controlnet_processor_id=["hed", None, None])


@pytest.mark.parametrize("proc", ["canny", "depth", "openpose"])
def test_an_unknown_processor_inside_a_list_is_refused_by_name(proc):
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    with pytest.raises(NotImplementedError, match=repr(proc)):
        StreamDiffusionWrapper("tiny-turbo", [32], controlnet_id_or_path=["a", "b"], controlnet_processor_id=["hed", proc])
    with pytest.raises(NotImplementedError, match=repr(proc)):
        StreamDiffusionWrapper("tiny-turbo", [32], controlnet_id_or_path=["a"], controlnet_processor_id=[proc])


def test_pipeline_lists_reach_the_wrapper(monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P

    class Stop(Exception):
        pass
    seen = []

    def init(self, **kw):
        seen.append(kw)
        raise Stop
    monkeypatch.setattr(P.StreamDiffusionWrapper, "__init__", init)
    monkeypatch.delenv("B200SD_CONTROLNET", raising=False)
    with pytest.raises(Stop):
        P.StreamDiffusionPipeline("model", controlnet=["a", "b"], controlnet_processor=[None, "hed"])
    assert (seen[-1]["controlnet_id_or_path"], seen[-1]["controlnet_processor_id"]) == (["a", "b"], [None, "hed"])


def test_blob_keys_by_order_and_processor(tmp_path):
    from ai_rtc_agent_b200.host import weights as W

    def key(cn, proc):
        return W.packed_blob_path(tmp_path, "m", "sd15", True, None, None, None, synthetic=True, controlnet=cn,
                                  control_processor=proc)
    keys = [key(["a", "b"], [None, "hed"]), key(["b", "a"], [None, "hed"]), key(["a", "b"], ["hed", None]),
            key(["a", "b"], ["hed", "hed"]), key("a", None), key(["a", "b", "c"], [None, "hed", None])]
    assert len(set(keys)) == len(keys)
    assert key("a", "hed") == key("a", "hed")


def test_synthetic_seeds_by_position():
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    arch = A.TINY_TURBO
    single = W.resolve_controlnet("synthetic-cn", arch, True)
    nets = [W.resolve_controlnet("synthetic-cn", arch, True, net=i) for i in range(3)]
    assert all(torch.equal(single[k], nets[0][k]) for k in single), "net 0 keeps the single net's seed"
    key = "controlnet_mid_block.weight"
    assert not torch.equal(nets[0][key], nets[1][key]) and not torch.equal(nets[1][key], nets[2][key])


def test_config_layout_extends_the_old_one():
    """control_processor_more is appended: every earlier field keeps its offset, so a version-4 blob's config is a prefix"""
    from ai_rtc_agent_b200.host import capi
    C = capi.EngineConfig
    assert C.control_processor_more.offset == C.ip_tokens.offset + 4
    assert ctypes.sizeof(C) == C.control_processor_more.offset + 4 * (capi.MAX_CONTROLNETS - 1)
    assert [f[0] for f in C._fields_][-2:] == ["ip_tokens", "control_processor_more"]


def test_header_declares_the_same_layout():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "b200sd.h")).read()
    body = src[src.index("typedef struct {\n    int block_out_channels[4];"):]
    body = body[:body.index("} b2sd_config;")]
    assert body.rstrip().endswith("Inherited by lanes and styles. */") and "int control_processor_more[B2SD_MAX_CONTROLNETS - 1];" in body
    assert body.index("int ip_tokens;") < body.index("int control_processor_more[")
    from ai_rtc_agent_b200.host import capi
    assert re.search(r"#define B2SD_MAX_CONTROLNETS (\d+)", src).group(1) == str(capi.MAX_CONTROLNETS)
    for fn in ("b2sd_set_control_scales", "b2sd_state_set_control_scales"):
        assert fn + "(" in src


# ---- host bookkeeping of per-net settings over a recording fake of libb200sd ---------------------------------------------------
class FakeLib:
    """Records every call; scale vectors are read at the call (host memory here), [nets * batch] for the plural calls"""

    def __init__(self, batch, nets):
        self.calls, self.batch, self.nets = [], batch, nets

    def __getattr__(self, name):
        if not name.startswith("b2sd_"):
            raise AttributeError(name)

        def call(*args):
            a = [x.value if isinstance(x, ctypes.c_void_p) else x for x in args]
            if name in ("b2sd_set_control_scale", "b2sd_state_set_control_scale"):
                raise AssertionError(f"{name} with {self.nets} nets")
            if name in ("b2sd_set_control_scales", "b2sd_state_set_control_scales"):
                a[-2] = list((ctypes.c_float * (self.batch * self.nets)).from_address(a[-2]))
            self.calls.append((name[5:],) + tuple(a))
            return 0
        return call


@pytest.fixture
def host(monkeypatch):
    from ai_rtc_agent_b200.host import stream as S
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    monkeypatch.setattr(S, "_on_device", lambda t, device: t.contiguous())
    monkeypatch.setattr(S, "_encode_beside", lambda eng, prompt: eng._encode(prompt)[0])
    lib = FakeLib(4, 2)
    eng = object.__new__(S.StreamDiffusion)
    eng.__dict__.update(
        _lib=lib, _handle=ctypes.c_void_p(1), lanes=[], _states=weakref.WeakSet(), _prepared=True, _ev=None,
        arch=types.SimpleNamespace(ctx_tokens=77, cross_attention_dim=8), prompt_encoder=SyntheticPromptEncoder(8),
        device=torch.device("cpu"), dtype=torch.float16, t_list=list(T4), denoising_steps_num=4, batch_size=4, frame_bff_size=1,
        cfg_type="self", latent_height=2, latent_width=2, generator=None, has_controlnet=True, control_nets=2,
        control=S.default_controls(2), live_lora=True, _is_style=False, use_denoising_batch=True)
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
    return eng, new_state, lib


def f32(xs):
    return torch.tensor(xs, dtype=torch.float32).tolist()


def test_prepare_pushes_every_nets_scales(host):
    eng, _, lib = host
    assert [c[:3] for c in lib.calls if c[0] == "set_control_scales"] == [("set_control_scales", 1, [1.0] * 8)]


def test_refused_updates_change_nothing(host):
    eng, new_state, lib = host
    a = new_state()
    lib.calls.clear()
    for bad in (([1.0, 0.5, 0.2],), (1.0, [0.7, 0.0], [0.3, 1.0]), ([float("nan"), 1.0],), (1.0, [0.0, 0.1, 0.2])):
        with pytest.raises(ValueError):
            eng.set_control_scale(*bad)
        with pytest.raises(ValueError):
            a.set_control_scale(*bad)
    assert lib.calls == [] and eng.control == ((1.0, 1.0), (0.0, 0.0), (1.0, 1.0)) and a.own_control is None


def test_random_updates_match_a_model_of_every_viewer(host):
    """A seeded sequence of global and per-viewer prompt, t_index_list, per-net ControlNet and LoRA updates.  After each,
    every viewer is stepped with the per-net scales of (its own settings or the global ones) masked by (its own t_index_list or
    the global one)."""
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import check_controls, control_vector
    eng, new_state, lib = host
    states = [new_state() for _ in range(3)]
    model = {"control": check_controls(1.0, 0.0, 1.0, 2), "t": list(T4), "own_c": [None] * 3, "own_t": [None] * 3}
    rng = random.Random(11)
    eng.set_control_scale(1.0)   # the defaults, on the root and its lane
    lists = [[10, 20, 30, 40], [0, 16, 32, 45], [18, 26, 35, 45], [5, 24, 25, 49]]
    settings = [([0.6, 1.2], 0.0, 1.0), (1.0, [0.5, 0.0], 1.0), ([-0.5, 0.3], 0.0, [0.5, 1.0]), (0.37, 0.2, 0.8),
                ([0.0, 1.0], 0.0, 1.0), (1.0, 0.0, 1.0)]
    for step in range(60):
        op = rng.choice(["g_prompt", "g_t", "g_control", "g_lora", "v_prompt", "v_t", "v_control"])
        v = rng.randrange(3)
        if op == "g_prompt":
            eng.update_prompt(f"p{step}")
        elif op == "g_t":
            t = rng.choice(lists)
            eng.t_list, eng.sub_timesteps = t, [eng.timesteps[i] for i in t]
            eng.sync_timesteps()
            model["t"], model["own_t"] = list(t), [None] * 3
        elif op == "g_control":
            c = rng.choice(settings)
            eng.set_control_scale(*c)
            model["control"], model["own_c"] = check_controls(*c, nets=2), [None] * 3
        elif op == "g_lora":
            eng.apply_factors([])
        elif op == "v_prompt":
            states[v].set_prompt(f"v{step}")
        elif op == "v_t":
            t = rng.choice(lists)
            states[v].set_t_index_list(t)
            model["own_t"][v] = list(t)
        else:
            c = rng.choice(settings)
            states[v].set_control_scale(*c)
            model["own_c"][v] = check_controls(*c, nets=2)
        glob = [c for c in lib.calls if c[0] == "set_control_scales"]
        assert {c[1] for c in glob[-2:]} == {1, 2} and glob[-1][2] == glob[-2][2], "the root and its lane agree"
        assert glob[-1][2] == f32(control_vector(model["control"], model["t"], 50))
        for k, st in enumerate(states):
            assert st.own_control == model["own_c"][k] and st.own_t_index_list == model["own_t"][k], (step, op, k)
            mine = [c for c in lib.calls if (c[0] == "state_set_control_scales" and c[2] == 100 + k) or
                    (c[0] == "state_clear_conditioning" and c[1] == 100 + k and c[2] == capi.COND_TIME) or
                    (c[0] == "state_set_timesteps" and c[2] == 100 + k)]
            if model["own_c"][k] is None and model["own_t"][k] is None:
                assert not mine or mine[-1][0] == "state_clear_conditioning", (step, op, k)
            else:
                want = control_vector(model["own_c"][k] or model["control"], model["own_t"][k] or model["t"], 50)
                assert mine[-1][0] == "state_set_control_scales" and mine[-1][3] == f32(want), (step, op, k)


# ---- the same bookkeeping through the pipeline, viewers and style moves --------------------------------------------------------
@pytest.fixture
def peers(host, monkeypatch, tmp_path):
    """(per-peer pipeline over the host fixture's two-net engines, a cached style of one LoRA file, that file's lora_dict,
    FakeLib)"""
    import contextlib
    from ai_rtc_agent_b200.host import pipeline as P
    from ai_rtc_agent_b200.host import stream as S
    from ai_rtc_agent_b200.host import wrapper as Wm
    eng, _, lib = host

    class Stream:
        def wait_event(self, ev):
            pass

    class Event:
        def record(self, stream=None):
            pass
    cur = Stream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: cur)
    monkeypatch.setattr(torch.cuda, "Event", Event)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())

    def new_state(self):
        st = object.__new__(S.StreamState)
        st.__dict__.update(_engine=self, _lib=lib, _handle=ctypes.c_void_p(200 + len(self._states)))
        self._states.add(st)
        return st
    eng.new_state = types.MethodType(new_state, eng)
    style = object.__new__(S.StreamDiffusion)
    style.__dict__.update(eng.__dict__, _handle=ctypes.c_void_p(3), lanes=[], _is_style=True)
    style._stream = lambda: 0
    eng.styles = [style]
    path = str(tmp_path / "a.safetensors")
    open(path, "w").write("a")
    lora = {path: 1.0}
    model = object.__new__(Wm.StreamDiffusionWrapper)
    model.__dict__.update(stream=eng, live_lora=True, _ext_stream=None, device="cpu")
    p = object.__new__(P.StreamDiffusionPipeline)
    p.__dict__.update(model=model, per_peer_streams=True, _peer_set=weakref.WeakSet(), _engines=[eng] + eng.lanes,
                      _lane_streams=[None, None], _lane_done=[None, None], _next_lane=0, _lora=None, _lora_key=())
    p._styles = {P.style_key(lora): P._Style(P.style_key(lora), lora, [style], [None])}
    p._styles[P.style_key(lora)].users = 1   # never evicted here
    return p, style, lora, lib


def test_pipeline_viewers_and_style_moves_match_a_model(peers):
    """A seeded sequence of the public calls with two nets: StreamDiffusionPipeline.update_controlnet_scale /
    update_t_index_list / update_prompt, PeerStream.update_controlnet_scale (floats and per-net lists) / update_t_index_list /
    update_lora (moves to and from a style).  After each, every viewer's controlnet_scale is its own or the global settings as
    three lists of one entry per net, and its time block holds both nets' scales of those settings masked by its own or the
    global t_index_list, computed on an engine of the store it runs on (the style's after a move there)."""
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import check_controls, control_vector
    p, style, lora, lib = peers
    views = [p.open_stream() for _ in range(3)]
    handles = {id(v): v._state.handle.value for v in views}
    model = {"control": check_controls(1.0, 0.0, 1.0, 2), "t": list(T4), "own_c": [None] * 3, "own_t": [None] * 3,
             "style": [False] * 3}
    rng = random.Random(5)
    lists = [[10, 20, 30, 40], [0, 16, 32, 45], [5, 24, 25, 49]]
    settings = [([0.6, 1.2], 0.0, 1.0), (1.0, [0.5, 0.0], 1.0), ([-0.5, 0.3], 0.0, [0.5, 1.0]), (0.37, 0.2, 0.8)]
    for step in range(60):
        op = rng.choice(["g_control", "g_t", "g_prompt", "v_control", "v_t", "v_style", "v_unstyle"])
        k = rng.randrange(3)
        v = views[k]
        if op == "g_control":
            c = rng.choice(settings)
            p.update_controlnet_scale(*c)
            model["control"], model["own_c"] = check_controls(*c, nets=2), [None] * 3
        elif op == "g_t":
            t = rng.choice(lists)
            p.update_t_index_list(t)
            model["t"], model["own_t"] = list(t), [None] * 3
        elif op == "g_prompt":
            p.update_prompt(f"p{step}")
        elif op == "v_control":
            c = rng.choice(settings)
            v.update_controlnet_scale(*c)
            model["own_c"][k] = check_controls(*c, nets=2)
        elif op == "v_t":
            t = rng.choice(lists)
            v.update_t_index_list(t)
            model["own_t"][k] = list(t)
        elif op == "v_style":
            v.update_lora(lora)
            model["style"][k] = True
        else:
            v.update_lora(None)
            model["style"][k] = False
        for j, w in enumerate(views):
            settings_j = model["own_c"][j] or model["control"]
            assert w.controlnet_scale == tuple(list(x) for x in settings_j), (step, op, j)
            assert all(isinstance(x, list) and len(x) == 2 for x in w.controlnet_scale)
            h = handles[id(w)]
            mine = [c for c in lib.calls if (c[0] == "state_set_control_scales" and c[2] == h) or
                    (c[0] == "state_clear_conditioning" and c[1] == h and c[2] == capi.COND_TIME)]
            if model["own_c"][j] is None and model["own_t"][j] is None:
                assert not mine or mine[-1][0] == "state_clear_conditioning", (step, op, j)
            else:
                want = control_vector(settings_j, model["own_t"][j] or model["t"], 50)
                assert mine[-1][0] == "state_set_control_scales" and mine[-1][3] == f32(want), (step, op, j)
                assert (mine[-1][1] == 3) == model["style"][j], (step, op, j, "computed on the store the viewer runs on")
    assert any(c[0] == "state_set_control_scales" and c[1] == 3 for c in lib.calls), "a viewer's settings moved to the style"


def test_pipeline_refuses_bad_per_net_settings_before_anything_changes(peers):
    p, style, lora, lib = peers
    v = p.open_stream()
    lib.calls.clear()
    for bad in (([1.0, 0.5, 0.2],), (1.0, [0.0, 0.1, 0.2]), (1.0, [0.6, 0.0], [0.4, 1.0])):
        with pytest.raises(ValueError):
            p.update_controlnet_scale(*bad)
        with pytest.raises(ValueError):
            v.update_controlnet_scale(*bad)
    assert not [c for c in lib.calls if "control_scale" in c[0]]
    assert v.controlnet_scale == ([1.0, 1.0], [0.0, 0.0], [1.0, 1.0])


# ---- the multi-net restatement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("processor", [None, "hed"])
def test_one_net_restatement_is_the_single_net_oracle(processor):
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import unet as ounet
    from oracle import weights as ow
    from ai_rtc_agent_b200.host import arch as A
    from tests.multi_controlnet_ref import MultiControlNetStreamOracle
    cfg = ounet.tiny_config(True)
    usd, vsd = ow.to_float(ow.make_unet_weights(cfg)), ow.to_float(ow.make_taesd_weights())
    cn = ow.to_float(ocn.make_weights(cfg))
    hed = {k: v.half().float() for k, v in A.synthetic_hed().items()} if processor else None
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim).float()
    noise = torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(3))
    single = ocn.ControlNetStreamOracle(usd, cfg, vsd, cn, [20, 40], 64, 64, hed_sd=hed)
    multi = MultiControlNetStreamOracle(usd, cfg, vsd, [cn], [processor], [20, 40], 64, 64, hed_sd=hed)
    for o in (single, multi):
        o.prepare(emb, guidance_scale=0.0, init_noise=noise)
    for i in range(2):
        frame = ow.make_frame(64, 64, seed=i)
        assert torch.equal(opipe.frame_to_u8(single, frame), opipe.frame_to_u8(multi, frame)), f"frame {i}"
