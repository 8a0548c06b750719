"""Per-peer temporal streams on the GPU: several viewers interleaved through one pipeline each get exactly what a pipeline of
their own would give them, bit for bit; the shared mode demonstrably mixes them; the pipeline's own stream is unchanged; the
lifecycle (close / reopen, global updates, prepare) and the refusals of the C ABI; the memory a state costs, and device
memory returned as soon as engines, lanes, states and pipelines are dropped."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]
# peer of each submission: late joins (peer 1 at submission 2, peer 2 at 5) and uneven frame counts (5 / 4 / 3)
SCHEDULE = {2: [0, 0, 1, 0, 1, 1, 0, 1, 0], 3: [0, 0, 1, 0, 1, 2, 1, 0, 2, 0, 1, 2]}


def _weights(model_id):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config("turbo" in model_id) if model_id.startswith("tiny") else ounet.config_for(model_id)
    return A.arch_for(model_id), cfg, ow.make_unet_weights(cfg), ow.make_taesd_weights()


def _pipelines(model_id, tl, hw, specs, monkeypatch):
    """One StreamDiffusionPipeline per entry of `specs` (constructor keywords; "policy" sets the launch policy's frames in
    flight, so that a one-lane reference runs the same launches as a pool of lanes), all over one set of seeded weights."""
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


def _interleaved(pipe, frames, schedule, per_peer=True):
    """Submit every frame at once in schedule order (each peer's stream opened at its first frame), then read the results."""
    streams, tickets, pos = {}, {p: [] for p in frames}, {p: 0 for p in frames}
    for p in schedule:
        if per_peer and p not in streams:
            streams[p] = pipe.open_stream()
        target = streams[p] if per_peer else pipe
        tickets[p].append(target.enqueue(frames[p][pos[p]]))
        pos[p] += 1
    outs = {p: [t.result().cpu() for t in ts] for p, ts in tickets.items()}
    for s in streams.values():
        s.close()
    return outs


def _fresh(pipe):
    """Back to a fresh stream (prepare zeroes the latent buffer, re-seeds the noise, re-encodes the prompt)."""
    torch.cuda.synchronize()
    pipe.model.prepare(prompt=pipe.prompt, num_inference_steps=50, guidance_scale=0.0)


def _dedicated(pipe, frames):
    """Each peer's frames alone through a one-lane pipeline with the shared (reference) stream, restarted per peer."""
    outs = {}
    for p, fs in frames.items():
        _fresh(pipe)
        outs[p] = [pipe(f).cpu() for f in fs]
    return outs


def _assert_equal(got, want, what):
    for p in want:
        assert len(got[p]) == len(want[p])
        for i, (g, w) in enumerate(zip(got[p], want[p])):
            assert torch.equal(g, w), f"{what}: peer {p} frame {i} differs (max |d| {(g.int() - w.int()).abs().max().item()})"


@pytest.mark.parametrize("model_id,tl,hw,lanes,peers", [
    ("tiny-sd15", T4, 128, 1, 3),
    ("tiny-sd15", T4, 128, 2, 3),
    ("tiny-sd15", T4, 128, 3, 3),
    ("tiny-turbo", [20, 40], 128, 2, 2),
    ("tiny-turbo", [32], 128, 4, 3),
    ("tiny-sd15", T4, (128, 192), 2, 2),
    ("runwayml/stable-diffusion-v1-5", T4, 512, 2, 3),
], ids=["sd15-T4-1lane", "sd15-T4-2lanes", "sd15-T4-3lanes", "turbo-T2", "turbo-T1-4lanes", "sd15-T4-128x192",
        "sd15-T4-512-full"])
def test_peers_are_isolated_bit_for_bit(cuda, monkeypatch, model_id, tl, hw, lanes, peers):
    height, width = (hw, hw) if isinstance(hw, int) else hw
    pool, ded = _pipelines(model_id, tl, hw, [dict(per_peer_streams=True, lanes=lanes), dict(lanes=1, policy=lanes)],
                           monkeypatch)
    assert pool.lanes == lanes and ded.lanes == 1
    assert all(e.launches_per_step == ded.model.stream.launches_per_step for e in pool._engines)
    schedule = SCHEDULE[peers]
    frames = _frames(peers, _counts(schedule), height, width)
    got = _interleaved(pool, frames, schedule)
    _assert_equal(got, _dedicated(ded, frames), f"{model_id} T={len(tl)} lanes={lanes}")


def _engines(tl, concurrency, controlnet=False, hed=False, tiny_vae=True):
    """(a pool root, a dedicated engine) over the same seeded tiny SD-1.5 weights, both with `concurrency` frames in flight"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(False)
    usd = ow.make_unet_weights(cfg)
    vsd = ow.make_taesd_weights() if tiny_vae else A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL)
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    cn = ocn.make_weights(cfg) if controlnet else None
    hed_sd = {k: v.half().float() for k, v in A.synthetic_hed().items()} if hed else None
    out = []
    for _ in range(2):
        sd = StreamDiffusion(A.TINY_SD15, usd, vsd, tl, lambda p: emb, width=128, height=128, controlnet_sd=cn, hed_sd=hed_sd,
                             use_tiny_vae=tiny_vae)
        sd.set_concurrency(concurrency)
        sd.prepare("p", guidance_scale=0.0)
        out.append(sd)
    return out


def _engine_interleaved(root, lanes, frames, schedule):
    """The pipeline's per-peer scheme at the engine level: lanes in rotation, each on its own CUDA stream, one state per peer."""
    engines = [root] + [root.add_lane() for _ in range(lanes - 1)]
    streams = [torch.cuda.Stream() for _ in engines]
    ready = torch.cuda.Event()
    ready.record()
    states, outs, pos = {}, {p: [] for p in frames}, {p: 0 for p in frames}
    for k, p in enumerate(schedule):
        if p not in states:
            states[p] = root.new_state()
        i = k % lanes
        with torch.cuda.stream(streams[i]):
            streams[i].wait_event(ready)
            outs[p].append(engines[i].step_u8(frames[p][pos[p]], state=states[p]))
        pos[p] += 1
    torch.cuda.synchronize()
    for s in states.values():
        s.close()
    return {p: [o.cpu() for o in v] for p, v in outs.items()}


@pytest.mark.parametrize("variant", ["controlnet-hed", "autoencoder-kl"])
def test_peers_are_isolated_with_controlnet_and_full_vae(cuda, variant):
    """Configurations the agent's pipeline does not build, through the engine API the pipeline uses."""
    kw = dict(controlnet=True, hed=True) if variant == "controlnet-hed" else dict(tiny_vae=False)
    root, ded = _engines(T4, 2, **kw)
    schedule = SCHEDULE[3]
    frames = _frames(3, _counts(schedule), 128, 128, base=50)
    got = _engine_interleaved(root, 2, frames, schedule)
    want = {}
    for p, fs in frames.items():
        ded.prepare("p", guidance_scale=0.0)
        want[p] = [ded.step_u8(f).cpu() for f in fs]
    _assert_equal(got, want, variant)


def test_shared_mode_mixes_the_peers(cuda, monkeypatch):
    """The check above discriminates: the same interleaving through the shared (reference) mode gives every peer frames that
    differ from its dedicated pipeline's as soon as another peer's frame has entered the stream batch before them; the
    frames before that point are the same."""
    shared, ded = _pipelines("tiny-sd15", T4, 128, [dict(lanes=2), dict(lanes=1, policy=2)], monkeypatch)
    schedule = SCHEDULE[3]
    frames = _frames(3, _counts(schedule), 128, 128)
    got = _interleaved(shared, frames, schedule, per_peer=False)
    want = _dedicated(ded, frames)
    mixed = {p: [] for p in want}     # per peer and frame: has a foreign frame been submitted before it?
    for k, p in enumerate(schedule):
        mixed[p].append(any(q != p for q in schedule[:k]))
    for p in want:
        differ = [not torch.equal(g, w) for g, w in zip(got[p], want[p])]
        assert differ == mixed[p], f"peer {p}: frames that differ {differ}, frames after a foreign frame {mixed[p]}"


def test_pipeline_own_stream_unchanged(cuda, monkeypatch):
    """With per-peer streams on, pipeline.enqueue / pipeline(frame) still give exactly what the shared mode gives."""
    from oracle import weights as ow
    on, off = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=True, lanes=2), dict(per_peer_streams=False, lanes=2)],
                         monkeypatch)
    assert on.per_peer_streams and not off.per_peer_streams and on.lanes == off.lanes == 2
    frames = [ow.make_frame(128, 128, seed=300 + i).cuda() for i in range(8)]
    a = [t.result().cpu() for t in [on.enqueue(f) for f in frames]]
    b = [t.result().cpu() for t in [off.enqueue(f) for f in frames]]
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"frame {i}"
    assert torch.equal(on(frames[0]).cpu(), off(frames[0]).cpu())
    assert [e.launches_per_step for e in on._engines] == [e.launches_per_step for e in off._engines]


def test_closed_stream_reopened_is_fresh(cuda, monkeypatch):
    pool, ded = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=True, lanes=2), dict(lanes=1, policy=2)], monkeypatch)
    frames = _frames(2, {0: 4, 1: 5}, 128, 128, base=400)
    other = pool.open_stream()
    first = pool.open_stream()
    for f in frames[0]:
        first.enqueue(f)
        other.enqueue(frames[1][0])
    first.close()
    with pool.open_stream() as again:                # may reuse the freed memory: it must start from zeros all the same
        got = {1: [again.enqueue(f).result().cpu() for f in frames[1]]}
    other.close()
    _assert_equal(got, _dedicated(ded, {1: frames[1]}), "reopened stream")


def test_global_updates_reach_every_peer_at_the_matching_point(cuda, monkeypatch):
    """A prompt and t_index_list update issued between two submissions applies to each peer from its next frame on, as if its
    own pipeline had been updated at the same point of its own sequence."""
    pool, ded0, ded1 = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=True, lanes=2), dict(lanes=1, policy=2),
                                                          dict(lanes=1, policy=2)], monkeypatch)
    schedule, cut = SCHEDULE[2], 5
    frames = _frames(2, _counts(schedule), 128, 128, base=500)
    streams = {p: pool.open_stream() for p in frames}
    tickets, pos = {p: [] for p in frames}, {p: 0 for p in frames}
    for k, p in enumerate(schedule):
        if k == cut:
            pool.update_prompt("another prompt")
            pool.update_t_index_list([10, 20, 30, 40])
        tickets[p].append(streams[p].enqueue(frames[p][pos[p]]))
        pos[p] += 1
    got = {p: [t.result().cpu() for t in ts] for p, ts in tickets.items()}
    want = {}
    for p, ded in ((0, ded0), (1, ded1)):
        before = schedule[:cut].count(p)
        want[p] = [ded(f).cpu() for f in frames[p][:before]]
        ded.update_prompt("another prompt")
        ded.update_t_index_list([10, 20, 30, 40])
        want[p] += [ded(f).cpu() for f in frames[p][before:]]
    _assert_equal(got, want, "global update")


def test_prepare_resets_every_state(cuda, monkeypatch):
    """prepare() restarts every live state: the peers' and the pipeline's own, which is a state on two lanes with per-peer
    streams on and off."""
    for per_peer in (True, False):
        pool, ded = _pipelines("tiny-sd15", T4, 128, [dict(per_peer_streams=per_peer, lanes=2), dict(lanes=1, policy=2)],
                               monkeypatch)
        assert pool._own_state is not None
        frames = _frames(2, {0: 6, 1: 6}, 128, 128, base=600)
        frames[2] = frames[0]                         # the pipeline's own stream
        targets = {0: pool.open_stream(), 1: pool.open_stream()} if per_peer else {}
        targets[2] = pool
        for i in range(3):
            for p, target in targets.items():
                target.enqueue(frames[p][i])
        _fresh(pool)                                  # StreamDiffusion.prepare under the pipeline: every live state restarts
        got = {p: [target.enqueue(f) for f in frames[p][3:]] for p, target in targets.items()}
        got = {p: [t.result().cpu() for t in ts] for p, ts in got.items()}
        _assert_equal(got, _dedicated(ded, {p: frames[p][3:] for p in targets}), f"after prepare, per_peer={per_peer}")
        for p in targets.keys() - {2}:
            targets[p].close()


def test_state_refusals(cuda):
    """A state runs only on engines of its weight store, batch and size, and the engine must be prepared."""
    import ctypes as C
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import weights as ow
    _, cfg, usd, vsd = _weights("tiny-sd15")
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    mk = lambda tl=T4, **kw: StreamDiffusion(A.TINY_SD15, usd, vsd, tl, lambda p: emb, width=128, height=128, **kw)
    root = mk()
    root.prepare("p", guidance_scale=0.0)
    state = root.new_state()
    frame = ow.make_frame(128, 128, seed=700).cuda()
    root.step_u8(frame, state=state)
    lane = root.add_lane()
    lane.step_u8(frame, state=state)                 # any lane of the store, same batch and size
    other_store = mk()
    other_store.prepare("p", guidance_scale=0.0)
    other_size = StreamDiffusion(A.TINY_SD15, {}, {}, T4, lambda p: emb, width=192, height=128, parent=root)
    other_size.prepare("p", guidance_scale=0.0)
    other_batch = StreamDiffusion(A.TINY_SD15, {}, {}, [18, 35], lambda p: emb, width=128, height=128, parent=root)
    other_batch.prepare("p", guidance_scale=0.0)
    for eng in (other_store, other_size, other_batch):
        with pytest.raises(capi.B2Error, match="another weight store, batch or size"):
            eng.step_u8(frame, state=state)
    lib = capi.lib()
    raw = mk()                                        # never prepared
    h = C.c_void_p()
    assert lib.b2sd_state_create(raw._handle, C.byref(h), None) != 0 and b"b2sd_prepare" in lib.b2sd_last_error()
    out = torch.empty((1, 3, 128, 128), dtype=torch.uint8, device="cuda")
    assert lib.b2sd_step_state(raw._handle, state.handle, frame.data_ptr(), capi.IN_U8_NHWC, 128, 128, out.data_ptr(),
                               capi.OUT_U8_NCHW, None) != 0
    assert b"b2sd_prepare" in lib.b2sd_last_error()
    state.close()
    state.close()                                     # idempotent
    with pytest.raises(RuntimeError, match="closed"):
        root.step_u8(frame, state=state)
    torch.cuda.synchronize()


def test_engines_lanes_and_states_release_device_memory_without_the_garbage_collector(cuda, monkeypatch):
    """Engines, their lanes (stepping a state alternately or not), their stream states and a per-peer pipeline form no reference
    cycle: dropping the last reference returns their device memory at once.  Otherwise it stays allocated until the garbage
    collector happens to run, and a process that builds pipelines one after another can run out of HBM."""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import weights as ow
    _, cfg, usd, vsd = _weights("tiny-sd15")
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    frame = ow.make_frame(512, 512, seed=900).cuda()

    def free():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[0]

    gc.collect()
    gc.disable()
    try:
        free0 = free()
        root = StreamDiffusion(A.TINY_SD15, usd, vsd, T4, lambda p: emb, width=512, height=512)
        root.prepare("p", guidance_scale=0.0)
        lane = root.add_lane()
        state = root.new_state()
        lane.step_u8(frame, state=state)
        owner = StreamDiffusion(A.TINY_SD15, usd, vsd, T4, lambda p: emb, width=512, height=512)
        owner.prepare("p", guidance_scale=0.0)
        paired = owner.add_lane()
        shared = owner.new_state()
        owner.step_u8(frame, state=shared)
        paired.step_u8(frame, state=shared)
        pool, = _pipelines("tiny-sd15", T4, 512, [dict(per_peer_streams=True, lanes=2)], monkeypatch)
        with pool.open_stream() as peer:
            peer.enqueue(frame).result()
        pool.enqueue(frame).result()
        used = free0 - free()
        del root, lane, state, owner, paired, shared, pool, peer
        left = free0 - free()
    finally:
        gc.enable()
    print(f"engines, lanes, states and a pipeline held {used / 2**20:.0f} MiB; {left / 2**20:.0f} MiB left after dropping them")
    assert used > 256 << 20, "the check needs engines of a measurable size"
    assert left <= 32 << 20


def test_state_memory_cost(cuda):
    """64 states of a 512x512 T=4 stream cost (T-1) * 64 * 64 * 4 fp16 values each, plus the stream-ordered allocator's
    granularity (its pool reserves device memory 32 MiB at a time), not a lane's activations."""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import weights as ow
    _, cfg, usd, vsd = _weights("tiny-sd15")
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    sd = StreamDiffusion(A.TINY_SD15, usd, vsd, T4, lambda p: emb, width=512, height=512)
    sd.prepare("p", guidance_scale=0.0)
    per_state = 3 * 64 * 64 * 8
    gc.collect()                                      # whatever an earlier test left to the collector
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    states = [sd.new_state() for _ in range(64)]
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    slack = 32 << 20
    print(f"64 states: {used} bytes of device memory (payload {64 * per_state})")
    assert used <= 64 * per_state + slack
    frame = ow.make_frame(512, 512, seed=800).cuda()
    outs = [sd.step_u8(frame, state=s) for s in states[:4]]
    torch.cuda.synchronize()
    assert all(torch.equal(o, outs[0]) for o in outs), "fresh states step identically"
    for s in states:
        s.close()
