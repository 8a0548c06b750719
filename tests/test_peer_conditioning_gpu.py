"""Per-peer prompts and t_index_lists on the GPU.  Viewers with their own conditioning, interleaved through one per-peer
pipeline, each get bit for bit what a dedicated one-lane pipeline gives when it is prepared with the global values and then
given that viewer's update_prompt / update_t_index_list at the same frame; and every check also asserts that the overridden
viewer's frames differ from the global conditioning's, so that a build ignoring the overrides fails.  Also: mid-stream updates
with frames pending, the per-key interplay with global updates, ControlNet + HED and the AutoencoderKL at the engine level, no
conditioning copies without overrides, an update that does not wait for queued frames, the refusals, and the memory."""
import gc
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]
SCHEDULE = {2: [0, 0, 1, 0, 1, 1, 0, 1, 0], 3: [0, 0, 1, 0, 1, 2, 1, 0, 2, 0, 1, 2]}
PROMPTS = {1: "a red fox in the snow", 2: "a city street at night"}   # peer 0 keeps the global conditioning
TLISTS = {4: {1: [10, 20, 30, 40], 2: [5, 15, 25, 45]}, 2: {1: [10, 30], 2: [25, 45]}, 1: {1: [20], 2: [45]}}


def _weights(model_id):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config("turbo" in model_id) if model_id.startswith("tiny") else ounet.config_for(model_id)
    return A.arch_for(model_id), cfg, ow.make_unet_weights(cfg), ow.make_taesd_weights()


def _pipelines(model_id, tl, hw, specs, monkeypatch):
    """One StreamDiffusionPipeline per entry of `specs` over one set of seeded weights ("policy": the launch policy's frames in
    flight, so that a one-lane reference runs the same launches as a pool of lanes).  Prompts go through the synthetic encoder."""
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import PER_PEER_STREAMS_ENV, StreamDiffusionPipeline
    height, width = (hw, hw) if isinstance(hw, int) else hw
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    monkeypatch.delenv(PER_PEER_STREAMS_ENV, raising=False)
    arch, _, usd, vsd = _weights(model_id)
    W.register_preloaded(model_id, arch, usd, vsd)
    out = []
    try:
        for kw in specs:
            kw = dict(kw)
            policy = kw.pop("policy", None)
            if policy:
                monkeypatch.setenv("B200SD_POLICY_FRAMES", str(policy))
            else:
                monkeypatch.delenv("B200SD_POLICY_FRAMES", raising=False)
            out.append(StreamDiffusionPipeline(model_id, t_index_list=tl, width=width, height=height, **kw))
    finally:
        W._PRELOADED.pop(model_id, None)
        monkeypatch.delenv("B200SD_POLICY_FRAMES", raising=False)
    return out


def _frames(peers, counts, height, width, base=0):
    from oracle import weights as ow
    return {p: [ow.make_frame(height, width, seed=base + 1000 * p + i).cuda() for i in range(counts[p])] for p in range(peers)}


def _counts(schedule):
    return {p: schedule.count(p) for p in set(schedule)}


def _assert_equal(got, want, what):
    for p in want:
        assert len(got[p]) == len(want[p])
        for i, (g, w) in enumerate(zip(got[p], want[p])):
            assert torch.equal(g, w), f"{what}: peer {p} frame {i} differs (max |d| {(g.int() - w.int()).abs().max().item()})"


def _assert_discriminating(got, glob, peers, what):
    for p in peers:
        assert any(not torch.equal(g, w) for g, w in zip(got[p], glob[p])), f"{what}: peer {p}'s frames equal the global ones"


def _dedicated(ded, tl, frames, steps):
    """Each peer's frames alone through a one-lane shared-mode pipeline, prepared with the global values (the constructor's
    t_index_list) before each peer; steps[p] = [(frame index, callable(ded)), ...] updates applied before that frame."""
    outs = {}
    for p, fs in frames.items():
        torch.cuda.synchronize()
        ded.model.prepare(prompt=ded.prompt, t_index_list=list(tl), num_inference_steps=50, guidance_scale=0.0)
        todo = dict(steps.get(p, []))
        outs[p] = []
        for i, f in enumerate(fs):
            for upd in todo.get(i, []):
                upd(ded)
            outs[p].append(ded(f).cpu())
    return outs


def _set_prompt(prompt):
    return lambda target: target.update_prompt(prompt)


def _set_tl(tl):
    return lambda target: target.update_t_index_list(tl)


def _own(p, T):
    """peer p's updates at its first frame"""
    ups = ([_set_prompt(PROMPTS[p])] if p in PROMPTS else []) + ([_set_tl(TLISTS[T][p])] if p in TLISTS[T] else [])
    return [(0, ups)] if ups else []


@pytest.mark.parametrize("model_id,tl,hw,lanes,peers", [
    ("tiny-sd15", T4, 128, 1, 3),
    ("tiny-sd15", T4, 128, 2, 3),
    ("tiny-sd15", T4, 128, 3, 3),
    ("tiny-turbo", [20, 40], 128, 2, 3),
    ("tiny-turbo", [32], 128, 4, 3),
    ("tiny-sd15", T4, (128, 192), 2, 3),
    ("runwayml/stable-diffusion-v1-5", T4, 512, 2, 3),
], ids=["sd15-T4-1lane", "sd15-T4-2lanes", "sd15-T4-3lanes", "turbo-T2", "turbo-T1-4lanes", "sd15-T4-128x192",
        "sd15-T4-512-full"])
def test_peers_with_their_own_conditioning_match_dedicated_pipelines(cuda, monkeypatch, model_id, tl, hw, lanes, peers):
    height, width = (hw, hw) if isinstance(hw, int) else hw
    pool, ded = _pipelines(model_id, tl, hw, [dict(per_peer_streams=True, lanes=lanes), dict(lanes=1, policy=lanes)],
                           monkeypatch)
    T = len(tl)
    schedule = SCHEDULE[peers]
    frames = _frames(peers, _counts(schedule), height, width)
    streams, tickets, pos = {}, {p: [] for p in frames}, {p: 0 for p in frames}
    for p in schedule:                                 # each viewer sets its conditioning when it joins, before its first frame
        if p not in streams:
            streams[p] = pool.open_stream()
            for _, ups in _own(p, T):
                for upd in ups:
                    upd(streams[p])
        tickets[p].append(streams[p].enqueue(frames[p][pos[p]]))
        pos[p] += 1
    assert streams[1].prompt == PROMPTS[1] and streams[1].t_index_list == TLISTS[T][1]
    assert streams[0].prompt == pool.prompt and streams[0].t_index_list == tl
    got = {p: [t.result().cpu() for t in ts] for p, ts in tickets.items()}
    for s in streams.values():
        s.close()
    what = f"{model_id} T={T} lanes={lanes}"
    _assert_equal(got, _dedicated(ded, tl, frames, {p: _own(p, T) for p in frames}), what)
    _assert_discriminating(got, _dedicated(ded, tl, frames, {}), [1, 2], what)


def test_mid_stream_update_switches_at_the_submission(cuda, monkeypatch):
    """Peer 1 updates while frames of every peer are pending on both lanes: its frames switch exactly at the call."""
    pool, ded = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=True, lanes=2), dict(lanes=1, policy=2)], monkeypatch)
    schedule, cut = SCHEDULE[3], 6
    frames = _frames(3, _counts(schedule), 128, 128, base=100)
    streams = {p: pool.open_stream() for p in frames}
    tickets, pos = {p: [] for p in frames}, {p: 0 for p in frames}
    # Every lane waits for the caller's stream, which now spins for about 0.5 s (1e9 cycles at under 2 GHz): submitting six tiny
    # frames takes a few milliseconds, so at the cut every peer's frames are still pending.
    torch.cuda._sleep(1_000_000_000)
    for k, p in enumerate(schedule):
        if k == cut:
            assert not any(ts[-1].done() for ts in tickets.values()), "frames of every peer are pending"
            streams[1].update_prompt(PROMPTS[1])
            streams[1].update_t_index_list(TLISTS[4][1])
        tickets[p].append(streams[p].enqueue(frames[p][pos[p]]))
        pos[p] += 1
    got = {p: [t.result().cpu() for t in ts] for p, ts in tickets.items()}
    for s in streams.values():
        s.close()
    before = schedule[:cut].count(1)
    _assert_equal(got, _dedicated(ded, T4, frames, {1: [(before, [_set_prompt(PROMPTS[1]), _set_tl(TLISTS[4][1])])]}),
                  "mid-stream update")
    glob = _dedicated(ded, T4, frames, {})
    assert [torch.equal(g, w) for g, w in zip(got[1], glob[1])][:before] == [True] * before
    _assert_discriminating({1: got[1][before:]}, {1: glob[1][before:]}, [1], "mid-stream update")


def test_global_updates_are_per_key(cuda, monkeypatch):
    """A has its own prompt, B its own t_index_list, C neither; then a global prompt update (A follows it, B keeps its list) and
    a global t_index_list update (B follows it)."""
    pool, ded = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=True, lanes=2), dict(lanes=1, policy=2)], monkeypatch)
    frames = _frames(3, {0: 6, 1: 6, 2: 6}, 128, 128, base=200)
    a, b, c = (pool.open_stream() for _ in range(3))
    a.update_prompt(PROMPTS[1])
    b.update_t_index_list(TLISTS[4][1])
    g_prompt, g_tl = "a global prompt", [12, 24, 36, 48]
    tickets = {p: [] for p in frames}
    for phase in range(3):
        if phase == 1:
            pool.update_prompt(g_prompt)
            assert (a.prompt, b.prompt, c.prompt) == (g_prompt,) * 3 and b.t_index_list == TLISTS[4][1]
        if phase == 2:
            pool.update_t_index_list(g_tl)
            assert (a.t_index_list, b.t_index_list, c.t_index_list) == (g_tl,) * 3
        for i in range(2 * phase, 2 * phase + 2):
            for p, s in enumerate((a, b, c)):
                tickets[p].append(s.enqueue(frames[p][i]))
    got = {p: [t.result().cpu() for t in ts] for p, ts in tickets.items()}
    for s in (a, b, c):
        s.close()
    later = [(2, [_set_prompt(g_prompt)]), (4, [_set_tl(g_tl)])]
    want = _dedicated(ded, T4, frames, {0: [(0, [_set_prompt(PROMPTS[1])])] + later, 1: [(0, [_set_tl(TLISTS[4][1])])] + later,
                                        2: later})
    _assert_equal(got, want, "per-key global updates")
    glob = _dedicated(ded, T4, frames, {p: later for p in frames})
    _assert_discriminating({p: got[p][:2] for p in (0, 1)}, {p: glob[p][:2] for p in (0, 1)}, [0, 1], "per-key")


def _engines(tl, controlnet=False, hed=False, tiny_vae=True):
    """(a pool root, a dedicated engine) over the same seeded tiny SD-1.5 weights and the synthetic prompt encoder"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(False)
    usd = ow.make_unet_weights(cfg)
    vsd = ow.make_taesd_weights() if tiny_vae else A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL)
    cn = ocn.make_weights(cfg) if controlnet else None
    hed_sd = {k: v.half().float() for k, v in A.synthetic_hed().items()} if hed else None
    out = []
    for _ in range(2):
        sd = StreamDiffusion(A.TINY_SD15, usd, vsd, tl, SyntheticPromptEncoder(cfg.cross_attention_dim), width=128, height=128,
                             controlnet_sd=cn, hed_sd=hed_sd, use_tiny_vae=tiny_vae)
        sd.set_concurrency(2)
        sd.prepare("p", guidance_scale=0.0)
        out.append(sd)
    return out


def _engine_dedicated(ded, frames, own):
    outs = {}
    for p, fs in frames.items():
        ded.t_list = list(T4)
        ded.prepare("p", guidance_scale=0.0)
        if own and p in PROMPTS:
            ded.update_prompt(PROMPTS[p])
        if own and p in TLISTS[4]:
            ded.t_list = TLISTS[4][p]
            ded.sub_timesteps = [ded.timesteps[t] for t in ded.t_list]
            ded.sync_timesteps()
        outs[p] = [ded.step_u8(f).cpu() for f in fs]
    return outs


@pytest.mark.parametrize("variant", ["controlnet-hed", "autoencoder-kl"])
def test_own_conditioning_with_controlnet_and_full_vae(cuda, variant):
    """Configurations the agent's pipeline does not build, through the engine API the pipeline uses: lanes in rotation on
    their own CUDA streams, each peer's update computed on the lane that takes its next frame."""
    kw = dict(controlnet=True, hed=True) if variant == "controlnet-hed" else dict(tiny_vae=False)
    root, ded = _engines(T4, **kw)
    schedule = SCHEDULE[3]
    frames = _frames(3, _counts(schedule), 128, 128, base=300)
    engines = [root, root.add_lane()]
    streams = [torch.cuda.Stream() for _ in engines]
    ready = torch.cuda.Event()
    ready.record()
    states, outs, pos = {}, {p: [] for p in frames}, {p: 0 for p in frames}
    for k, p in enumerate(schedule):
        i = k % 2
        with torch.cuda.stream(streams[i]):
            streams[i].wait_event(ready)
            if p not in states:
                states[p] = root.new_state()
                if p in PROMPTS:
                    states[p].set_prompt(PROMPTS[p], engine=engines[i])
                if p in TLISTS[4]:
                    states[p].set_t_index_list(TLISTS[4][p], engine=engines[i])
            outs[p].append(engines[i].step_u8(frames[p][pos[p]], state=states[p]))
        pos[p] += 1
    torch.cuda.synchronize()
    got = {p: [o.cpu() for o in v] for p, v in outs.items()}
    for s in states.values():
        s.close()
    _assert_equal(got, _engine_dedicated(ded, frames, True), variant)
    _assert_discriminating(got, _engine_dedicated(ded, frames, False), [1, 2], variant)


@pytest.mark.parametrize("tl,lanes", [(T4, 2), ([32], 4)], ids=["sd15-T4", "turbo-T1"])
def test_no_conditioning_copies_without_overrides(cuda, monkeypatch, tl, lanes):
    model_id = "tiny-sd15" if len(tl) > 1 else "tiny-turbo"
    pool, = _pipelines(model_id, tl, 128, [dict(per_peer_streams=True, lanes=lanes)], monkeypatch)
    frames = _frames(3, _counts(SCHEDULE[3]), 128, 128, base=400)
    streams, pos = {}, {p: 0 for p in frames}
    for p in SCHEDULE[3]:
        if p not in streams:
            streams[p] = pool.open_stream()
        streams[p].enqueue(frames[p][pos[p]])
        pos[p] += 1
    pool.enqueue(frames[0][0]).result()
    assert [e.conditioning_binds() for e in pool._engines] == [0] * lanes
    streams[1].update_prompt(PROMPTS[1])             # the counter counts: an override is copied where it is not held, and the
    for _ in range(lanes):                           # global block back where the next frame follows the global prompt
        streams[1].enqueue(frames[1][0])
    streams[0].enqueue(frames[0][0]).result()
    assert sum(e.conditioning_binds() for e in pool._engines) > 0
    for s in streams.values():
        s.close()


@pytest.mark.parametrize("encoder", ["synthetic", "blocking-upload"])
def test_update_does_not_wait_for_queued_frames(cuda, monkeypatch, encoder):
    """Viewer B has 8 full-size 512x512 T=4 frames queued (well over 100 ms of device work) when viewer A updates its prompt:
    the update returns while B's last frame on each lane is still pending, and A's frames are right.  "blocking-upload": the
    encoder ends in a blocking host-to-device copy, as CLIP's upload of the token ids does, which synchronises the stream it
    runs on."""
    pool, ded = _pipelines("runwayml/stable-diffusion-v1-5", T4, 512, [dict(per_peer_streams=True, lanes=2),
                                                                       dict(lanes=1, policy=2)], monkeypatch)
    if encoder == "blocking-upload":
        synthetic = pool.model.stream.prompt_encoder
        for eng in pool._engines:
            eng.prompt_encoder = lambda p: synthetic(p).to("cuda") * 1.0
    frames = _frames(2, {0: 4, 1: 8}, 512, 512, base=500)
    with pool.open_stream() as warm:                 # warm-up: each lane's first launches, the first override
        warm.update_prompt("warm-up")
        for f in frames[1][:2]:
            warm.enqueue(f)
    torch.cuda.synchronize()
    a, b = pool.open_stream(), pool.open_stream()
    got_a = [a.enqueue(frames[0][0])]
    tb = [b.enqueue(f) for f in frames[1]]
    t0 = time.perf_counter()
    a.update_prompt(PROMPTS[1])
    host_ms = (time.perf_counter() - t0) * 1e3
    pending = not tb[-1].done() and not tb[-2].done()   # B's last frame on either lane
    got_a += [a.enqueue(f) for f in frames[0][1:]]
    got = {0: [t.result().cpu() for t in got_a]}
    print(f"per-peer update_prompt ({encoder} encoder): {host_ms:.2f} ms on the host; B's last frames pending after it: {pending}")
    assert pending, f"the update waited for queued frames ({host_ms:.1f} ms)"
    a.close()
    b.close()
    _assert_equal(got, _dedicated(ded, T4, {0: frames[0]}, {0: [(1, [_set_prompt(PROMPTS[1])])]}), "update under load")


def test_state_conditioning_refusals(cuda):
    import ctypes as C
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    _, cfg, usd, vsd = _weights("tiny-sd15")
    enc = SyntheticPromptEncoder(cfg.cross_attention_dim)
    mk = lambda tl=T4, **kw: StreamDiffusion(A.TINY_SD15, usd, vsd, tl, enc, width=128, height=128, **kw)
    root = mk()
    root.prepare("p", guidance_scale=0.0)
    state = root.new_state()
    lane = root.add_lane()
    state.set_prompt("x", engine=lane)               # any lane of the store, same batch and size
    state.set_t_index_list([10, 20, 30, 40], engine=lane)
    other_store = mk()
    other_store.prepare("p", guidance_scale=0.0)
    other_size = StreamDiffusion(A.TINY_SD15, {}, {}, T4, enc, width=192, height=128, parent=root)
    other_size.prepare("p", guidance_scale=0.0)
    other_batch = StreamDiffusion(A.TINY_SD15, {}, {}, [18, 35], enc, width=128, height=128, parent=root)
    other_batch.prepare("p", guidance_scale=0.0)
    for eng in (other_store, other_size, other_batch):
        with pytest.raises(capi.B2Error, match="another weight store, batch or size"):
            state.set_prompt("x", engine=eng)
    with pytest.raises(capi.B2Error, match="another weight store, batch or size"):
        state.set_t_index_list(T4, engine=other_store)
    with pytest.raises(ValueError, match="t_index_list length 3 != stream batch 4"):
        state.set_t_index_list([10, 20, 30])
    lib = capi.lib()
    raw = mk()                                        # never prepared
    emb = torch.zeros((77, cfg.cross_attention_dim), dtype=torch.float16, device="cuda")
    assert lib.b2sd_state_set_prompt_embeds(raw._handle, state.handle, emb.data_ptr(), None) != 0
    assert b"b2sd_prepare" in lib.b2sd_last_error()
    assert lib.b2sd_state_set_timesteps(root._handle, state.handle, None, None) != 0 and b"null" in lib.b2sd_last_error()
    assert lib.b2sd_state_clear_conditioning(state.handle, 2) != 0
    state.close()
    with pytest.raises(RuntimeError, match="closed"):
        state.set_prompt("x")
    torch.cuda.synchronize()


def test_override_memory_is_returned(cuda):
    """An override costs its block, at the granularity of its pool; after 100 updates and a close the pool keeps at most its
    release threshold (64 MiB here); dropping the engines gives everything back, all without the garbage collector."""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import weights as ow
    _, cfg, usd, vsd = _weights("tiny-sd15")
    frame = ow.make_frame(512, 512, seed=600).cuda()

    def free():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[0]

    gc.collect()
    gc.disable()
    try:
        base = free()
        sd = StreamDiffusion(A.TINY_SD15, usd, vsd, T4, SyntheticPromptEncoder(cfg.cross_attention_dim), width=512, height=512)
        sd.prepare("p", guidance_scale=0.0)
        lane = sd.add_lane()
        state = sd.new_state()
        free0 = free()
        state.set_prompt("one")
        one = free0 - free()
        for i in range(100):
            eng = (sd, lane)[i % 2]
            if i % 3:
                state.set_prompt(f"prompt {i}", engine=eng)
            else:
                state.set_t_index_list([10 + i % 7, 20, 30, 40], engine=eng)
            eng.step_u8(frame, state=state)
        state.close()
        kept = free0 - free()
        del sd, lane, state, eng
        left = base - free()
    finally:
        gc.enable()
    print(f"one prompt override: {one} bytes of device memory; after 100 updates and close the pool keeps {kept} bytes; "
          f"{left} bytes left after dropping the engines")
    assert 0 < one <= (32 << 20), "an override costs its block, at the pool's granularity"
    assert kept <= (64 << 20)
    # a leaked override would keep a whole pool chunk (32 MiB, the cost of `one` above) mapped
    assert left <= (16 << 20), "overrides leaked"
