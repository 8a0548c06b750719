"""ControlNet conditioning scale and guidance window, without a GPU: the per-slot mask against diffusers' controlnet_keep, the
checks, the fp32 restatement, and which settings the host layer gives every viewer through a random sequence of updates."""
import ctypes
import random
import types
import weakref

import pytest
import torch

from tests.controlnet_scale_ref import ScaledControlNetOracle, controlnet_keep

T_LISTS = [[0], [10], [20], [25], [45], [49], [20, 40], [0, 49], [32, 45], [18, 26, 35, 45], [0, 16, 32, 45],
           [10, 20, 30, 40], [18, 26, 35], [5, 15, 25, 35, 45], [0, 1, 2, 3, 4, 5, 6, 7]]
WINDOWS = [(0.0, 1.0), (0.0, 0.5), (0.5, 1.0), (0.2, 0.8), (0.36, 0.72), (0.0, 0.02), (0.98, 1.0), (0.5, 0.52), (0.25, 0.75)]


def test_slot_mask_is_diffusers_controlnet_keep_at_every_table_length():
    from ai_rtc_agent_b200.host.stream import control_scales
    for n in range(1, 51):
        lists = [t for t in T_LISTS if max(t) < n] + [list(range(n))]
        for start, end in WINDOWS:
            keep = controlnet_keep(n, start, end)
            for t in lists:
                for scale in (1.0, 0.6, -0.5, 0.0):
                    assert control_scales((scale, start, end), t, n) == [scale * keep[i] for i in t], (n, t, start, end)


def test_slot_mask_boundaries():
    """`<` and `>` as diffusers writes them: a step whose fraction equals start is kept, one ending exactly at end is kept"""
    from ai_rtc_agent_b200.host.stream import control_scales
    assert control_scales((1.0, 0.5, 1.0), [24, 25, 26], 50) == [0.0, 1.0, 1.0]
    assert control_scales((1.0, 0.0, 0.5), [23, 24, 25], 50) == [1.0, 1.0, 0.0]
    assert control_scales((2.0, 0.0, 1.0), [0, 49], 50) == [2.0, 2.0]
    assert control_scales((1.0, 0.0, 0.02), [0, 1], 50) == [1.0, 0.0]


@pytest.mark.parametrize("args,match", [((1.0, 0.5, 0.5), "larger or equal"), ((1.0, 0.6, 0.4), "larger or equal"),
                                        ((1.0, -0.1, 0.5), "smaller than 0"), ((1.0, 0.0, 1.01), "larger than 1.0"),
                                        ((float("nan"), 0.0, 1.0), "finite"), ((float("inf"), 0.0, 1.0), "finite")])
def test_settings_are_checked_like_diffusers(args, match):
    from ai_rtc_agent_b200.host.stream import check_control
    with pytest.raises(ValueError, match=match):
        check_control(*args)
    assert check_control(-0.5, 0.0, 1.0) == (-0.5, 0.0, 1.0)   # negative scales are allowed, as in diffusers


# ---- the fp32 restatement ---------------------------------------------------------------------------------------------------
def _oracles(scales_list):
    from oracle import controlnet as ocn
    from oracle import stream as ostream
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(False)
    usd, vsd = ow.to_float(ow.make_unet_weights(cfg)), ow.to_float(ow.make_taesd_weights())
    cn = ow.to_float(ocn.make_weights(cfg))
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim).float()
    t = [18, 26, 35, 45]
    plain = ostream.StreamOracle(usd, cfg, vsd, t, 64, 64)
    ref = ocn.ControlNetStreamOracle(usd, cfg, vsd, cn, t, 64, 64)
    scaled = []
    for s in scales_list:
        o = ScaledControlNetOracle(usd, cfg, vsd, cn, t, 64, 64)
        o.scales = s
        scaled.append(o)
    for o in [plain, ref] + scaled:
        o.prepare(emb, guidance_scale=0.0, seed=3)
    return plain, ref, scaled


def test_oracle_scale_one_and_zero():
    from oracle import pipeline as opipe
    from oracle import weights as ow
    plain, ref, (one, zero) = _oracles([[1.0] * 4, [0.0] * 4])
    for i in range(3):
        frame = ow.make_frame(64, 64, seed=i)
        f_plain, f_ref, f_one, f_zero = (opipe.frame_to_u8(o, frame) for o in (plain, ref, one, zero))
        assert torch.equal(f_one, f_ref), "scale 1 is the ControlNet as it was"
        assert torch.equal(f_zero, f_plain), "scale 0 on every slot is the UNet without a ControlNet"
        assert not torch.equal(f_ref, f_plain)


def test_oracle_residuals_are_linear_in_the_scale():
    """residual(s) - skip = s * (residual(1) - skip), per slot, in float64"""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(False)
    usd = {k: v.double() for k, v in ow.to_float(ow.make_unet_weights(cfg)).items()}
    cn = {k: v.double() for k, v in ow.to_float(ocn.make_weights(cfg)).items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 4, 8, 8, generator=g, dtype=torch.float64)
    ts = torch.tensor([999.0, 659.0, 479.0, 99.0], dtype=torch.float64)
    ctx = ow.make_prompt_embeds(cfg.cross_attention_dim).double().expand(4, -1, -1)
    control = torch.rand(1, 3, 64, 64, generator=g, dtype=torch.float64)
    res, mid = ocn.controlnet_forward(cn, cfg, x, ts, ctx, control)
    s = torch.tensor([0.0, 1.0, -0.5, 0.37], dtype=torch.float64).view(-1, 1, 1, 1)
    base, one, scaled = {}, {}, {}
    ocn.unet_forward(usd, cfg, x, ts, ctx, [torch.zeros_like(r) for r in res], torch.zeros_like(mid), base)
    ocn.unet_forward(usd, cfg, x, ts, ctx, res, mid, one)
    ocn.unet_forward(usd, cfg, x, ts, ctx, [r * s for r in res], mid * s, scaled)
    keys = [k for k in one if k.startswith("res.")] + ["cn_mid"]
    for k in keys:
        torch.testing.assert_close(scaled[k] - base[k], s * (one[k] - base[k]), rtol=1e-12, atol=1e-12)


# ---- host bookkeeping over a recording fake of libb200sd ----------------------------------------------------------------------
class FakeLib:
    """Records every call; the scale vectors are read at the call (host memory here)"""

    def __init__(self, batch):
        self.calls, self.batch = [], batch

    def __getattr__(self, name):
        if not name.startswith("b2sd_"):
            raise AttributeError(name)

        def call(*args):
            a = [x.value if isinstance(x, ctypes.c_void_p) else x for x in args]
            if name in ("b2sd_set_control_scale", "b2sd_state_set_control_scale"):
                a[-2] = list((ctypes.c_float * self.batch).from_address(a[-2]))
            self.calls.append((name[5:],) + tuple(a))
            return 0
        return call


T4 = [18, 26, 35, 45]


def f32(xs):
    return torch.tensor(xs, dtype=torch.float32).tolist()


@pytest.fixture
def host(monkeypatch):
    from ai_rtc_agent_b200.host import stream as S
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    monkeypatch.setattr(S, "_on_device", lambda t, device: t.contiguous())
    monkeypatch.setattr(S, "_encode_beside", lambda eng, prompt: eng._encode(prompt)[0])
    lib = FakeLib(4)
    eng = object.__new__(S.StreamDiffusion)
    eng.__dict__.update(
        _lib=lib, _handle=ctypes.c_void_p(1), lanes=[], _states=weakref.WeakSet(), _prepared=True, _ev=None,
        arch=types.SimpleNamespace(ctx_tokens=77, cross_attention_dim=8), prompt_encoder=SyntheticPromptEncoder(8),
        device=torch.device("cpu"), dtype=torch.float16, t_list=list(T4), denoising_steps_num=4, batch_size=4, frame_bff_size=1,
        cfg_type="self", latent_height=2, latent_width=2, generator=None, has_controlnet=True, live_lora=True, _is_style=False,
        use_denoising_batch=True)
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


def test_prepare_pushes_the_global_scales(host):
    eng, _, lib = host
    assert [c[:3] for c in lib.calls if c[0] == "set_control_scale"] == [("set_control_scale", 1, [1.0] * 4)]


def test_engine_without_a_controlnet_refuses():
    from ai_rtc_agent_b200.host import stream as S
    eng = object.__new__(S.StreamDiffusion)
    st = object.__new__(S.StreamState)
    st.__dict__.update(_engine=eng, _lib=None, _handle=ctypes.c_void_p(5))
    with pytest.raises(RuntimeError, match="without a ControlNet"):
        eng.set_control_scale(0.5)
    with pytest.raises(RuntimeError, match="without a ControlNet"):
        st.set_control_scale(0.5)


def test_bad_settings_change_nothing(host):
    eng, new_state, lib = host
    a = new_state()
    lib.calls.clear()
    for bad in ((1.0, 0.7, 0.3), (float("nan"), 0.0, 1.0)):
        with pytest.raises(ValueError):
            eng.set_control_scale(*bad)
        with pytest.raises(ValueError):
            a.set_control_scale(*bad)
    assert lib.calls == [] and eng.control == (1.0, 0.0, 1.0) and a.own_control is None


def test_random_updates_match_a_model_of_every_viewer(host):
    """A seeded sequence of global and per-viewer prompt, t_index_list, ControlNet and LoRA updates.  After each, every viewer
    is stepped with the scales of (its own settings or the global ones) masked by (its own t_index_list or the global one):
    a state with either of its own carries those scales in its own time block (its latest state_set_control_scale since its
    time block was last cleared); the others have no time block of their own and read the engines' global scales."""
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import control_scales
    eng, new_state, lib = host
    states = [new_state() for _ in range(4)]
    model = {"control": (1.0, 0.0, 1.0), "t": list(T4), "own_c": [None] * 4, "own_t": [None] * 4}
    rng = random.Random(7)
    lists = [[10, 20, 30, 40], [0, 16, 32, 45], [18, 26, 35, 45], [5, 24, 25, 49]]
    settings = [(0.6, 0.0, 1.0), (1.0, 0.5, 1.0), (-0.5, 0.0, 0.5), (0.37, 0.2, 0.8), (0.0, 0.0, 1.0), (1.0, 0.0, 1.0)]
    for step in range(60):
        op = rng.choice(["g_prompt", "g_t", "g_control", "g_lora", "v_prompt", "v_t", "v_control"])
        v = rng.randrange(4)
        if op == "g_prompt":
            eng.update_prompt(f"p{step}")
        elif op == "g_t":
            t = rng.choice(lists)
            eng.t_list, eng.sub_timesteps = t, [eng.timesteps[i] for i in t]
            eng.sync_timesteps()
            model["t"], model["own_t"] = list(t), [None] * 4
        elif op == "g_control":
            c = rng.choice(settings)
            eng.set_control_scale(*c)
            model["control"], model["own_c"] = c, [None] * 4
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
            model["own_c"][v] = c
        glob = [c for c in lib.calls if c[0] == "set_control_scale"]
        assert {c[1] for c in glob[-2:]} == {1, 2} and glob[-1][2] == glob[-2][2], "the root and its lane agree"
        assert glob[-1][2] == f32(control_scales(model["control"], model["t"], 50))
        for k, st in enumerate(states):
            assert st.own_control == model["own_c"][k] and st.own_t_index_list == model["own_t"][k], (step, op, k)
            mine = [c for c in lib.calls if (c[0] == "state_set_control_scale" and c[2] == 100 + k) or
                    (c[0] == "state_clear_conditioning" and c[1] == 100 + k and c[2] == capi.COND_TIME) or
                    (c[0] == "state_set_timesteps" and c[2] == 100 + k)]
            if model["own_c"][k] is None and model["own_t"][k] is None:
                assert not mine or mine[-1][0] == "state_clear_conditioning", (step, op, k)
            else:
                want = control_scales(model["own_c"][k] or model["control"], model["own_t"][k] or model["t"], 50)
                assert mine[-1][0] == "state_set_control_scale" and mine[-1][3] == f32(want), (step, op, k)


def test_pipeline_keywords_reach_the_wrapper(monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P

    class Stop(Exception):
        pass
    seen = []

    def init(self, **kw):
        seen.append(kw)
        raise Stop
    monkeypatch.setattr(P.StreamDiffusionWrapper, "__init__", init)
    monkeypatch.delenv("B200SD_CONTROLNET", raising=False)
    for kw, want in (({}, (None, "hed")), ({"controlnet": "cn", "controlnet_processor": None}, ("cn", None)),
                     ({"controlnet": "x"}, ("x", "hed"))):
        with pytest.raises(Stop):
            P.StreamDiffusionPipeline("model", **kw)
        assert (seen[-1]["controlnet_id_or_path"], seen[-1]["controlnet_processor_id"]) == want
    monkeypatch.setenv("B200SD_CONTROLNET", "from-env")
    with pytest.raises(Stop):
        P.StreamDiffusionPipeline("model")
    assert seen[-1]["controlnet_id_or_path"] == "from-env"
    with pytest.raises(Stop):
        P.StreamDiffusionPipeline("model", controlnet="given")
    assert seen[-1]["controlnet_id_or_path"] == "given"


# ---- the same bookkeeping through the pipeline, viewers and style moves --------------------------------------------------------
@pytest.fixture
def peers(host, monkeypatch, tmp_path):
    """(per-peer pipeline over the host fixture's engines, a cached style of one LoRA file, that file's lora_dict, FakeLib)"""
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
    eng.new_state = types.MethodType(lambda self: _new_state(self, lib), eng)
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


def _new_state(eng, lib):
    from ai_rtc_agent_b200.host import stream as S
    st = object.__new__(S.StreamState)
    st.__dict__.update(_engine=eng, _lib=lib, _handle=ctypes.c_void_p(200 + len(eng._states)))
    eng._states.add(st)
    return st


def test_pipeline_viewers_and_style_moves_match_a_model(peers):
    """A seeded sequence of the public calls: StreamDiffusionPipeline.update_controlnet_scale / update_t_index_list /
    update_prompt, PeerStream.update_controlnet_scale / update_t_index_list / update_lora (moves to and from a style).  After
    each, every viewer's controlnet_scale is (its own or the global settings), and its time block holds the scales of those
    settings masked by (its own or the global t_index_list), computed on an engine of the store it runs on (the style's after a
    move there); a viewer with neither of its own has no time block of its own."""
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import control_scales
    p, style, lora, lib = peers
    views = [p.open_stream() for _ in range(3)]
    handles = {id(v): v._state.handle.value for v in views}
    model = {"control": (1.0, 0.0, 1.0), "t": list(T4), "own_c": [None] * 3, "own_t": [None] * 3, "style": [False] * 3}
    rng = random.Random(11)
    lists = [[10, 20, 30, 40], [0, 16, 32, 45], [5, 24, 25, 49]]
    settings = [(0.6, 0.0, 1.0), (1.0, 0.5, 1.0), (-0.5, 0.0, 0.5), (0.37, 0.2, 0.8)]
    for step in range(50):
        op = rng.choice(["g_control", "g_t", "g_prompt", "v_control", "v_t", "v_style", "v_unstyle"])
        k = rng.randrange(3)
        v = views[k]
        if op == "g_control":
            c = rng.choice(settings)
            p.update_controlnet_scale(*c)
            model["control"], model["own_c"] = c, [None] * 3
        elif op == "g_t":
            t = rng.choice(lists)
            p.update_t_index_list(t)
            model["t"], model["own_t"] = list(t), [None] * 3
        elif op == "g_prompt":
            p.update_prompt(f"p{step}")
        elif op == "v_control":
            c = rng.choice(settings)
            v.update_controlnet_scale(*c)
            model["own_c"][k] = c
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
            assert w.controlnet_scale == (model["own_c"][j] or model["control"]), (step, op, j)
            h = handles[id(w)]
            mine = [c for c in lib.calls if (c[0] == "state_set_control_scale" and c[2] == h) or
                    (c[0] == "state_clear_conditioning" and c[1] == h and c[2] == capi.COND_TIME)]
            if model["own_c"][j] is None and model["own_t"][j] is None:
                assert not mine or mine[-1][0] == "state_clear_conditioning", (step, op, j)
            else:
                want = control_scales(model["own_c"][j] or model["control"], model["own_t"][j] or model["t"], 50)
                assert mine[-1][0] == "state_set_control_scale" and mine[-1][3] == f32(want), (step, op, j)
                assert (mine[-1][1] == 3) == model["style"][j], (step, op, j, "computed on the store the viewer runs on")


def test_wrapper_update_controlnet_scale_reaches_the_engines(host):
    from ai_rtc_agent_b200.host import wrapper as Wm
    eng, _, lib = host
    model = object.__new__(Wm.StreamDiffusionWrapper)
    model.__dict__.update(stream=eng, _ext_stream=None)
    lib.calls.clear()
    model.update_controlnet_scale(0.5, control_guidance_start=0.4, control_guidance_end=1.0)
    assert [c[1:3] for c in lib.calls if c[0] == "set_control_scale"] == [(1, [0.0, 0.5, 0.5, 0.5]), (2, [0.0, 0.5, 0.5, 0.5])]
    with pytest.raises(ValueError):
        model.update_controlnet_scale(1.0, 0.5, 0.2)
