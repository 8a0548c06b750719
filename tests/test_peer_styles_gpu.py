"""Per-viewer style LoRAs on the GPU: a style's weights against a fresh live engine's, viewers' frames against pipelines whose
global style is theirs (bit for bit), a switch between queued frames, own prompts with own styles, memory across style
cycles, refusals, and a switch that does not wait for another viewer's queued frames."""
import ctypes
import os
import struct
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]
TT = "transformer_blocks.0."
MODS_A = ["down_blocks.0.attentions.0." + TT + "attn2.to_k", "down_blocks.0.attentions.0." + TT + "attn2.to_v",
          "up_blocks.3.attentions.2." + TT + "attn2.to_k", "mid_block.attentions.0." + TT + "attn2.to_v",
          "down_blocks.1.resnets.0.time_emb_proj", "up_blocks.1.resnets.0.time_emb_proj",
          "down_blocks.1.attentions.0." + TT + "attn1.to_q", "mid_block.attentions.0." + TT + "ff.net.0.proj",
          "down_blocks.0.attentions.0.proj_in", "up_blocks.2.attentions.1." + TT + "ff.net.2",
          "up_blocks.1.resnets.0.conv2", "up_blocks.1.resnets.0.conv_shortcut", "conv_in"]
MODS_B = ["down_blocks.0.attentions.1." + TT + "attn2.to_k", "up_blocks.3.attentions.2." + TT + "attn2.to_v",
          "up_blocks.3.attentions.2." + TT + "attn2.to_k", "mid_block.resnets.1.time_emb_proj",
          "down_blocks.1.resnets.0.time_emb_proj", "up_blocks.2.attentions.0." + TT + "attn1.to_out.0",
          "down_blocks.2.resnets.0.conv1", "up_blocks.0.resnets.2.conv2", "conv_out"]


# ---- LoRA writers, weights and pipelines (as in test_lora_switch_gpu.py) ---------------------------------------------------------
def _write_lora(path, usd, mods, rank, dtype, seed, gain=0.3):
    """A peft-style LoRA on `mods` whose deltas are about `gain` times the weights' spread"""
    from safetensors.torch import save_file
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for m in mods:
        w = usd[m + ".weight"]
        rows, cols = w.shape[0], w[0].numel()
        down = torch.randn(rank, cols, generator=g) / cols ** 0.5
        up = torch.randn(rows, rank, generator=g) * (gain * float(w.float().std()) / rank ** 0.5)
        if w.dim() == 4:
            down, up = down.reshape(rank, *w.shape[1:]), up.reshape(rows, rank, 1, 1)
        sd[f"unet.{m}.lora_A.weight"] = down.to(dtype).contiguous()
        sd[f"unet.{m}.lora_B.weight"] = up.to(dtype).contiguous()
    save_file(sd, str(path))
    return str(path)


def _loras(tmp_path, usd):
    """A: fp16 factors (rank 4) and fp32 factors (rank 8) in two files; B: other modules, fp16, rank 16"""
    a1 = _write_lora(tmp_path / "a1.safetensors", usd, MODS_A[:7], 4, torch.float16, 1)
    a2 = _write_lora(tmp_path / "a2.safetensors", usd, MODS_A[4:], 8, torch.float32, 2)
    b = _write_lora(tmp_path / "b.safetensors", usd, MODS_B, 16, torch.float16, 3)
    return {a1: 0.8, a2: 1.25}, {b: 1.0}


def _weights(turbo):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(turbo)
    return (A.TINY_TURBO if turbo else A.TINY_SD15), cfg, ow.make_unet_weights(cfg), ow.make_taesd_weights(), \
        ow.make_prompt_embeds(cfg.cross_attention_dim)


def _engine(arch, usd, vsd, emb, tl, cn=None, hw=128):
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, width=hw, height=hw, live_lora=True, controlnet_sd=cn)
    sd.prepare("p", guidance_scale=0.0)
    return sd


def _blob(sd, path):
    from ai_rtc_agent_b200.host import capi
    sd.export_packed(str(path))
    data = open(path, "rb").read()
    (count,) = struct.unpack_from("<I", data, 8 + 4 + ctypes.sizeof(capi.EngineConfig))
    return data, count


def _pipe(model_id, tl, monkeypatch, lanes=None, hw=128, live=True):
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    if "tiny" in model_id:
        arch, _, usd, vsd, _ = _weights("turbo" in model_id)
        W.register_preloaded(model_id, arch, usd, vsd)
    try:
        return StreamDiffusionPipeline(model_id, t_index_list=tl, width=hw, height=hw, lanes=lanes, live_lora=live,
                                       per_peer_streams=True)
    finally:
        W._PRELOADED.pop(model_id, None)


def _frame(i, hw=128):
    from oracle import weights as ow
    return ow.make_frame(hw, hw, seed=300 + i).cuda()


def _equal(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"{what}: frame {i} differs (max |d| {(g.int() - w.int()).abs().max().item()})"


def _single(model_id, tl, monkeypatch, lanes, lora, idx, prompt=None, t_index_list=None):
    """One viewer alone on a pipeline whose global style is `lora`, with its own prompt / t_index_list"""
    p = _pipe(model_id, tl, monkeypatch, lanes)
    if lora:
        p.update_lora(lora)
    with p.open_stream() as v:
        if prompt is not None:
            v.update_prompt(prompt)
        if t_index_list is not None:
            v.update_t_index_list(t_index_list)
        return [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in idx]]


@pytest.fixture
def env(monkeypatch):
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.setenv("B200SD_SYNTHETIC_WEIGHTS", "1")
    for v in ("B200SD_LANES", "B200SD_MAX_STYLES", "B200SD_POLICY_FRAMES"):
        monkeypatch.delenv(v, raising=False)
    return monkeypatch


@pytest.mark.parametrize("controlnet", [False, True])
def test_style_weights_equal_a_fresh_engine(cuda, tmp_path, controlnet):
    from oracle import controlnet as ocn
    arch, cfg, usd, vsd, emb = _weights(False)
    cn = ocn.make_weights(cfg) if controlnet else None
    A_, B_ = _loras(tmp_path, usd)
    root = _engine(arch, usd, vsd, emb, T4, cn)
    root.apply_lora(B_)                               # the parent's own style does not reach its styles
    style = root.add_style()
    style.apply_lora(A_)
    fresh = _engine(arch, usd, vsd, emb, T4, cn)
    fresh.apply_lora(A_)
    got, n = _blob(style, tmp_path / "s.b2pack")
    want, _ = _blob(fresh, tmp_path / "f.b2pack")
    assert got == want, "a style's weights must equal a fresh live engine's with the same LoRAs, byte for byte"
    base = root.add_style()
    fresh_base = _engine(arch, usd, vsd, emb, T4, cn)
    assert _blob(base, tmp_path / "b.b2pack")[0] == _blob(fresh_base, tmp_path / "fb.b2pack")[0]
    print(f"style blob: {n} entries, {len(got)} bytes")


@pytest.mark.parametrize("model_id,tl,lanes", [("tiny-turbo", [32], 8), ("tiny-sd15", T4, 2)], ids=["T1-8lanes", "T4-2lanes"])
def test_viewers_frames_equal_single_viewer_pipelines(cuda, tmp_path, env, model_id, tl, lanes):
    _, _, usd, _, _ = _weights("turbo" in model_id)
    A_, B_ = _loras(tmp_path, usd)
    n = 6
    p = _pipe(model_id, tl, env, lanes)
    launches = p.model.stream.launches_per_step
    views = [p.open_stream() for _ in range(4)]
    for v, d in zip(views, (None, A_, B_, A_)):
        if d is not None:
            v.update_lora(d)
    assert p.styles == 2
    tickets = {k: [] for k in range(4)}
    for i in range(n):
        for k, v in enumerate(views):
            tickets[k].append(v.enqueue(_frame(10 * k + i)))
    got = {k: [t.result().cpu() for t in ts] for k, ts in tickets.items()}
    for k, d in enumerate((None, A_, B_, A_)):
        _equal(got[k], _single(model_id, tl, env, lanes, d, [10 * k + i for i in range(n)]), f"viewer {k}")
    assert not torch.equal(got[1][0], _single(model_id, tl, env, lanes, None, [10])[0]), "style A must change the frames"
    assert p.model.stream.launches_per_step == launches and all(e.launches_per_step == launches for e in p._engines)


def test_switch_is_ordered_between_queued_frames(cuda, tmp_path, env):
    """T = 4: frames of a viewer queued before its update_lora use the old style, those after it the new one, with the
    stream state carried across.  The reference is one viewer on a pipeline whose global style switches from A to B with
    the device idle between the two halves (the global update_lora of test_lora_switch_gpu.py)."""
    _, _, usd, _, _ = _weights(False)
    A_, B_ = _loras(tmp_path, usd)
    sync = _pipe("tiny-sd15", T4, env)
    with sync.open_stream() as v:
        sync.update_lora(A_)
        want = [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(4)]]
        torch.cuda.synchronize()
        sync.update_lora(B_)
        torch.cuda.synchronize()
        want += [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(4, 8)]]
    p = _pipe("tiny-sd15", T4, env)
    other = p.open_stream()
    other.update_lora(B_)                            # B exists already: the switch below is a cache hit
    v = p.open_stream()
    v.update_lora(A_)
    first = [v.enqueue(_frame(i)) for i in range(4)]
    v.update_lora(B_)
    second = [v.enqueue(_frame(i)) for i in range(4, 8)]
    _equal([t.result().cpu() for t in first + second], want, "frames around a queued switch")
    no_switch = _single("tiny-sd15", T4, env, None, A_, range(8))
    assert all(not torch.equal(a, b) for a, b in zip(want[4:], no_switch[4:]))


@pytest.mark.parametrize("order", ["style-first", "conditioning-first"])
def test_own_prompt_and_t_index_list_with_own_style(cuda, tmp_path, env, order):
    _, _, usd, _, _ = _weights(False)
    A_, B_ = _loras(tmp_path, usd)
    own_tl, tl2 = [10, 20, 30, 40], [5, 15, 25, 40]
    # the reference: one viewer on a pipeline whose global style is A, with the same conditioning as its own, then B globally
    ref = _pipe("tiny-sd15", T4, env)
    ref.update_lora(A_)
    with ref.open_stream() as r:
        r.update_prompt("my own")
        r.update_t_index_list(own_tl)
        want = [t.result().cpu() for t in [r.enqueue(_frame(i)) for i in range(3)]]
        r.update_prompt("global 2")
        r.update_t_index_list(tl2)
        want += [t.result().cpu() for t in [r.enqueue(_frame(i)) for i in range(3, 5)]]
        ref.update_lora(B_)
        want += [t.result().cpu() for t in [r.enqueue(_frame(i)) for i in range(5, 7)]]
    p = _pipe("tiny-sd15", T4, env)
    v, w = p.open_stream(), p.open_stream()
    steps = [lambda: v.update_lora(A_), lambda: v.update_prompt("my own"), lambda: v.update_t_index_list(own_tl)]
    for s in (steps if order == "style-first" else steps[1:] + steps[:1]):
        s()
    w.update_lora(A_)
    got = [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(3)]]
    _equal(got, want[:3], "own style, prompt and t_index_list")
    # global updates: the prompt and t_index_list reach the style's engines and replace the viewer's own; update_lora drops
    # every viewer's own style (a global t_index_list changes only the time embedding's timesteps, as a viewer's own one does)
    p.update_prompt("global 2")
    p.update_t_index_list(tl2)
    assert v.prompt == "global 2" and v.t_index_list == tl2 and v.lora == A_ and v._style is not None
    got += [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(3, 5)]]
    p.update_lora(B_)
    assert v.lora == B_ and w.lora == B_ and v._style is None and p.styles == 1
    got += [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(5, 7)]]
    _equal(got, want, "a styled viewer across global updates")
    v.close()
    w.close()


@pytest.mark.parametrize("tl", [T4, [32]], ids=["T4", "T1"])
def test_controlnet_hed_with_two_styles(cuda, tmp_path, tl):
    """A ControlNet + HED engine (the style shares the ControlNet, HED and their K / V blocks): viewers stepped in rotation on
    the root's lanes and on two styles' lanes, on lanes' own streams, equal fresh live engines with the same LoRAs"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    _, cfg, usd, vsd, _ = _weights(False)
    cn = ocn.make_weights(cfg)
    hed_sd = {k: v.half().float() for k, v in A.synthetic_hed().items()}
    A_, B_ = _loras(tmp_path, usd)

    def engine():
        sd = StreamDiffusion(A.TINY_SD15, usd, vsd, tl, SyntheticPromptEncoder(cfg.cross_attention_dim), width=128, height=128,
                             controlnet_sd=cn, hed_sd=hed_sd, live_lora=True)
        sd.set_concurrency(2)
        sd.prepare("p", guidance_scale=0.0)
        return sd
    root = engine()
    pools = [[root, root.add_lane()]]
    for d in (A_, B_):
        style = root.add_style()
        pools.append([style, style.add_lane()])
        style.apply_lora(d)
    streams = [[torch.cuda.Stream() for _ in pool] for pool in pools]
    ready = torch.cuda.Event()
    ready.record()
    states = [root.new_state() for _ in pools]
    n = 5
    outs = [[] for _ in pools]
    for i in range(n):
        for k, pool in enumerate(pools):
            st = streams[k][i % 2]
            with torch.cuda.stream(st):
                st.wait_event(ready)
                outs[k].append(pool[i % 2].step_u8(_frame(10 * k + i), state=states[k]))
    torch.cuda.synchronize()
    got = [[o.cpu() for o in v] for v in outs]
    for s in states:
        s.close()

    def alone(d, idx):
        """the frames of one viewer on a fresh live engine after apply_lora(d)"""
        fresh = engine()
        if d is not None:
            fresh.apply_lora(d)
        with fresh.new_state() as st:
            return [fresh.step_u8(_frame(i), state=st).cpu() for i in idx]
    for k, d in enumerate((None, A_, B_)):
        idx = [10 * k + i for i in range(n)]
        _equal(got[k], alone(d, idx), f"pool {k} (ControlNet + HED)")
        if d is not None:
            assert any(not torch.equal(g, b) for g, b in zip(got[k], alone(None, idx))), f"style {k} must change the frames"


def test_memory_and_frame_programs_across_style_cycles(cuda, tmp_path, env):
    _, _, usd, _, _ = _weights(False)
    A_, B_ = _loras(tmp_path, usd)
    env.setenv("B200SD_MAX_STYLES", "1")
    p = _pipe("tiny-sd15", T4, env)
    launches = [e.launches_per_step for e in p._engines]
    v = p.open_stream()
    v.update_lora(A_)                                 # a first cycle: the override pool and allocator warm up
    v.enqueue(_frame(0)).result()
    v.update_lora(B_)
    v.enqueue(_frame(1)).result()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(20):
        v.update_lora(A_ if k % 2 == 0 else B_)       # each evicts the other
        v.enqueue(_frame(k)).result()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    print(f"20 style cycles: free device memory {free0 / 2**20:.1f} -> {free1 / 2**20:.1f} MiB")
    assert abs(free1 - free0) <= 64 << 20, "style cycles must return their memory (up to what the override pool keeps)"
    assert [e.launches_per_step for e in p._engines] == launches and p.styles == 1


def test_refusals(cuda, tmp_path, env):
    from ai_rtc_agent_b200.host import capi
    _, _, usd, _, _ = _weights(False)
    A_, B_ = _loras(tmp_path, usd)
    off = _pipe("tiny-sd15", T4, env, live=False)
    with off.open_stream() as v, pytest.raises(RuntimeError, match="live_lora=True"):
        v.update_lora(A_)
    env.setenv("B200SD_MAX_STYLES", "1")
    p = _pipe("tiny-sd15", T4, env)
    v, w = p.open_stream(), p.open_stream()
    v.update_lora(A_)
    before = [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(2)]]
    bad = tmp_path / "bad.safetensors"
    bad.write_bytes(b"not a safetensors file")
    with pytest.raises(Exception):
        w.update_lora({str(bad): 1.0})
    with pytest.raises(RuntimeError, match="in use"):
        w.update_lora(B_)
    c = p.open_stream()
    c.close()
    with pytest.raises(RuntimeError, match="closed"):
        c.update_lora(A_)
    assert p.styles == 1 and w._style is None
    ref = _single("tiny-sd15", T4, env, None, A_, range(4))
    _equal(before + [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in range(2, 4)]], ref, "frames after refusals")
    # a state of another store's family is still refused with the old message; an override of another store is refused
    other = _pipe("tiny-sd15", T4, env)
    lib = capi.lib()
    foreign = other.model.stream.new_state()
    out = torch.empty((1, 3, 128, 128), dtype=torch.uint8, device="cuda")
    f = _frame(0).contiguous()
    style_eng = v._style._engines[0]
    rc = lib.b2sd_step_state(style_eng._handle, foreign.handle, f.data_ptr(), capi.IN_U8_NHWC, 128, 128, out.data_ptr(),
                             capi.OUT_U8_NCHW, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"another weight store, batch or size" in lib.b2sd_last_error()
    w.update_prompt("computed on the pipeline's store")
    rc = lib.b2sd_step_state(style_eng._handle, w._state.handle, f.data_ptr(), capi.IN_U8_NHWC, 128, 128, out.data_ptr(),
                             capi.OUT_U8_NCHW, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"another weight store's parameters" in lib.b2sd_last_error()
    torch.cuda.synchronize()


def test_switch_to_a_cached_style_does_not_wait(cuda, tmp_path, env):
    """Viewer B has 8 full-size 512x512 T=4 frames queued when viewer A switches to a style that is already built: the call
    returns while B's last frames are still pending."""
    p = _pipe("runwayml/stable-diffusion-v1-5", T4, env, hw=512)
    usd_shapes = p.model.stream._unet_shapes
    fake = {k: torch.zeros(s) for k, s in usd_shapes.items() if k.endswith(".weight") and any(m in k for m in MODS_A[:2])}
    A_ = {_write_lora(tmp_path / "a.safetensors", {k: v + 1.0 for k, v in fake.items()}, [k[:-7] for k in fake], 4,
                      torch.float16, 1): 1.0}
    a, b, c = p.open_stream(), p.open_stream(), p.open_stream()
    c.update_lora(A_)                                  # builds the style
    for i in range(2):
        c.enqueue(_frame(i, 512))
        b.enqueue(_frame(i, 512))
    torch.cuda.synchronize()
    tb = [b.enqueue(_frame(i, 512)) for i in range(8)]
    t0 = time.perf_counter()
    a.update_lora(A_)
    host_ms = (time.perf_counter() - t0) * 1e3
    pending = not tb[-1].done() and not tb[-2].done()
    ta = a.enqueue(_frame(0, 512))
    print(f"switch to a cached style: {host_ms:.2f} ms on the host; B's last frames pending after it: {pending}")
    assert pending, f"the switch waited for queued frames ({host_ms:.1f} ms)"
    ta.result()
    for t in tb:
        t.result()
