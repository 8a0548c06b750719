"""Live LoRA switching on the GPU: the re-fused weights against a fresh engine and the CPU fuse, round trips, the ordering of a
switch against queued frames, viewers with their own conditioning, the fp32 oracle, and memory / frame programs across many
switches."""
import os
import struct

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]
TT = "transformer_blocks.0."
# modules the test LoRAs touch on the tiny SD-1.5 UNet: cross-attention K / V (the prompt blocks), time_emb_proj (the time
# blocks, read raw), q of the folded q/k/v and the GEGLU rows, proj_in / ff.net.2 (read raw), conv2 + shortcut, conv_in
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


def _cpu_fused(usd, lora_dict):
    from ai_rtc_agent_b200.host.weights import fuse_lora, load_lora_file
    out = dict(usd)
    for p, s in lora_dict.items():
        fuse_lora(out, load_lora_file(p), s)
    return out


def _engine(arch, usd, vsd, emb, tl, live, cn=None, hw=128):
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, width=hw, height=hw, live_lora=live, controlnet_sd=cn)
    sd.prepare("p", guidance_scale=0.0)
    return sd


def _blob(sd, path):
    """{name: (kind, bytes)} of an exported packed-weight blob (header: magic, version, b2sd_config, count)"""
    from ai_rtc_agent_b200.host import capi
    import ctypes
    sd.export_packed(str(path))
    data = open(path, "rb").read()
    off = 8 + 4 + ctypes.sizeof(capi.EngineConfig)
    (count,) = struct.unpack_from("<I", data, off)
    off += 4
    out = {}
    for _ in range(count):
        kind = data[off]
        (n,) = struct.unpack_from("<I", data, off + 1)
        name = data[off + 5: off + 5 + n].decode()
        off += 5 + n
        (ndim,) = struct.unpack_from("<I", data, off)
        off += 4 + 8 * ndim
        (nb,) = struct.unpack_from("<Q", data, off)
        off += 8
        out[name] = (kind, data[off: off + nb])
        off += nb
    assert off == len(data)
    return data, out


def _ulps(a, b):
    """|a - b| in fp16 ulps, elementwise (ordered-integer distance)"""
    def ordered(x):
        i = np.frombuffer(x, dtype=np.int16).astype(np.int32)
        return np.where(i < 0, -(i & 0x7FFF), i)
    return np.abs(ordered(a) - ordered(b))


@pytest.mark.parametrize("controlnet", [False, True])
def test_switched_weights_equal_a_fresh_engine_and_the_cpu_fuse(cuda, tmp_path, controlnet):
    from oracle import controlnet as ocn
    arch, cfg, usd, vsd, emb = _weights(False)
    cn = ocn.make_weights(cfg) if controlnet else None
    A_, B_ = _loras(tmp_path, usd)
    switched = _engine(arch, usd, vsd, emb, T4, True, cn)
    switched.apply_lora(B_)
    switched.apply_lora(A_)
    fresh = _engine(arch, usd, vsd, emb, T4, True, cn)
    fresh.apply_lora(A_)
    raw_s, ents_s = _blob(switched, tmp_path / "s.b2pack")
    raw_f, _ = _blob(fresh, tmp_path / "f.b2pack")
    assert raw_s == raw_f, "the switched engine's weights must equal a fresh live engine's byte for byte"
    base = _engine(arch, usd, vsd, emb, T4, True, cn)
    _, ents_b = _blob(base, tmp_path / "b.b2pack")
    cpu = _engine(arch, _cpu_fused(usd, A_), vsd, emb, T4, False, cn)
    _, ents_c = _blob(cpu, tmp_path / "c.b2pack")
    assert ents_c.keys() == ents_s.keys()
    changed, n16, d16, worst32, worst_fold = 0, 0, 0, 0.0, 0
    for name, (kind, got) in ents_s.items():
        want = ents_c[name][1]
        assert len(got) == len(want), name
        changed += got != ents_b[name][1]
        if kind in (0, 1):
            u = _ulps(got, want)
            n16 += u.size
            d16 += int((u > 0).sum())
            if "+ln" in name:   # W diag(gamma) rounded again: a 1-ulp difference of W may become 2 there
                worst_fold = max(worst_fold, int(u.max(initial=0)))
                assert u.max(initial=0) <= 2, f"{name}: {u.max()} ulp from the CPU fuse"
            else:
                assert u.max(initial=0) <= 1, f"{name}: {u.max()} ulp from the CPU fuse"
        else:
            g, w = np.frombuffer(got, np.float32), np.frombuffer(want, np.float32)
            worst32 = max(worst32, float(np.abs(g - w).max(initial=0) / max(float(np.abs(w).max(initial=0)), 1e-30)))
    print(f"live vs CPU fuse: {d16} of {n16} fp16 values differ ({d16 / n16:.2e}), at most {worst_fold} ulp in the LayerNorm-"
          f"folded rows and 1 elsewhere; worst fp32 vector difference {worst32:.2e} of the vector's largest magnitude; "
          f"{changed} blob entries changed by the LoRAs")
    assert changed >= 12 and worst32 < 1e-3


def _pipe(model_id, tl, live, monkeypatch, lanes=None, per_peer=False):
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    arch, _, usd, vsd, _ = _weights("turbo" in model_id)
    W.register_preloaded(model_id, arch, usd, vsd)
    try:
        return StreamDiffusionPipeline(model_id, t_index_list=tl, width=128, height=128, lanes=lanes, live_lora=live,
                                       per_peer_streams=per_peer)
    finally:
        W._PRELOADED.pop(model_id, None)


def _frame(i):
    from oracle import weights as ow
    return ow.make_frame(128, 128, seed=300 + i).cuda()


def _run(pipe, idx, target=None):
    tickets = [(target or pipe).enqueue(_frame(i)) for i in idx]
    return [t.result().cpu() for t in tickets]


def _equal(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"{what}: frame {i} differs (max |d| {(g.int() - w.int()).abs().max().item()})"


@pytest.mark.parametrize("model_id,tl,lanes", [("tiny-turbo", [32], 8), ("tiny-sd15", T4, 2)], ids=["T1-8lanes", "T4-2lanes"])
def test_round_trips_are_bit_exact(cuda, tmp_path, monkeypatch, model_id, tl, lanes):
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.setenv("B200SD_SYNTHETIC_WEIGHTS", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    _, _, usd, _, _ = _weights("turbo" in model_id)
    A_, B_ = _loras(tmp_path, usd)
    n = 9
    plain = _run(_pipe(model_id, tl, False, monkeypatch, lanes), range(n))
    base = _run(_pipe(model_id, tl, True, monkeypatch, lanes), range(n))
    _equal(base, plain, "live mode without a switch vs the default mode")
    # {} after construction without LoRAs, {} -> B -> {}, and {} again
    p = _pipe(model_id, tl, True, monkeypatch, lanes)
    p.update_lora({})
    got = _run(p, range(3))
    p.update_lora(B_)
    p.update_lora(None)
    got += _run(p, range(3, 6))
    p.update_lora({})
    got += _run(p, range(6, n))
    _equal(got, base, "base -> B -> base")
    # A -> B -> A, and A again
    ref = _pipe(model_id, tl, True, monkeypatch, lanes)
    ref.update_lora(A_)
    want = _run(ref, range(n))
    assert all(not torch.equal(a, b) for a, b in zip(want, base)), "LoRA A must change every frame"
    p = _pipe(model_id, tl, True, monkeypatch, lanes)
    launches = p.model.stream.launches_per_step
    p.update_lora(A_)
    got = _run(p, range(3))
    p.update_lora(B_)
    p.update_lora(A_)
    got += _run(p, range(3, 6))
    p.update_lora(A_)
    got += _run(p, range(6, n))
    _equal(got, want, "A -> B -> A")
    # twenty more switches: no device memory and no arena growth, the same frame programs
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(20):
        p.update_lora(B_ if k % 2 == 0 else A_)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    assert p.model.stream.launches_per_step == launches
    assert all(e.launches_per_step == launches for e in p._engines)


def test_switch_is_ordered_between_queued_frames(cuda, tmp_path, monkeypatch):
    """T = 4, two stage-pipelined lanes: frames enqueued before update_lora (still queued) use the old weights, frames
    enqueued after it the new ones, with the stream state carried across the switch"""
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    _, _, usd, _, _ = _weights(False)
    A_, B_ = _loras(tmp_path, usd)
    never = _pipe("tiny-sd15", T4, True, monkeypatch)
    never.update_lora(A_)
    want_before = _run(never, range(8))
    sync = _pipe("tiny-sd15", T4, True, monkeypatch)
    sync.update_lora(A_)
    _run(sync, range(4))
    torch.cuda.synchronize()
    sync.update_lora(B_)
    torch.cuda.synchronize()
    want_after = _run(sync, range(4, 8))
    p = _pipe("tiny-sd15", T4, True, monkeypatch)
    p.update_lora(A_)
    first = [p.enqueue(_frame(i)) for i in range(4)]
    p.update_lora(B_)
    second = [p.enqueue(_frame(i)) for i in range(4, 8)]
    _equal([t.result().cpu() for t in first], want_before[:4], "frames enqueued before the switch")
    _equal([t.result().cpu() for t in second], want_after, "frames enqueued after the switch")
    assert all(not torch.equal(a, b) for a, b in zip(want_after, want_before[4:]))


def test_viewers_keep_their_conditioning_across_a_switch(cuda, tmp_path, monkeypatch):
    """Per-peer streams at T = 1: two viewers with their own prompts and one with its own t_index_list; after update_lora each
    viewer's frames equal a fresh pipeline's with the new weights and that viewer's conditioning"""
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.delenv("B200SD_LANES", raising=False)
    _, _, usd, _, _ = _weights(True)
    A_, B_ = _loras(tmp_path, usd)
    own = [lambda s: s.update_prompt("a red fox in the snow"), lambda s: s.update_prompt("a city street at night"),
           lambda s: s.update_t_index_list([45])]
    pool = _pipe("tiny-turbo", [32], True, monkeypatch, lanes=2, per_peer=True)
    pool.update_lora(A_)
    peers = [pool.open_stream() for _ in own]
    for s, f in zip(peers, own):
        f(s)
    before = [_run(pool, range(3), s) for s in peers]
    pool.update_lora(B_)
    after = [_run(pool, range(3), s) for s in peers]
    for v, f in enumerate(own):
        ref = _pipe("tiny-turbo", [32], True, monkeypatch, lanes=2, per_peer=True)
        ref.update_lora(B_)
        s = ref.open_stream()
        f(s)
        _equal(after[v], _run(ref, range(3), s), f"viewer {v} after the switch")
        assert all(not torch.equal(a, b) for a, b in zip(after[v], before[v])), f"viewer {v}: the switch changed nothing"
    assert not torch.equal(after[0][0], after[1][0]) and not torch.equal(after[0][0], after[2][0])


@pytest.mark.parametrize("turbo,tl", [(False, T4), (True, [32])], ids=["sd15-T4", "turbo-T1"])
@pytest.mark.parametrize("controlnet", [False, True])
def test_switched_engine_matches_the_oracle(cuda, tmp_path, turbo, tl, controlnet):
    """After A -> B, frames match the fp32 oracle run on the CPU-fused weights of B (DESIGN.md section 2's u8 tolerance)"""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import stream as ostream
    from oracle import weights as ow
    arch, cfg, usd, vsd, emb = _weights(turbo)
    cn = ocn.make_weights(cfg) if controlnet else None
    if turbo:   # the tiny-turbo UNet: LoRAs on the modules it shares with the tiny SD-1.5 one
        mods = [m for m in MODS_A + MODS_B if m + ".weight" in usd]
        A_ = {_write_lora(tmp_path / "ta.safetensors", usd, mods[::2], 4, torch.float16, 5): 1.0}
        B_ = {_write_lora(tmp_path / "tb.safetensors", usd, mods[1::2], 8, torch.float32, 6): 0.9}
    else:
        A_, B_ = _loras(tmp_path, usd)
    sd = _engine(arch, usd, vsd, emb, tl, True, cn)
    sd.apply_lora(A_)
    sd.apply_lora(B_)
    fused = ow.to_float(_cpu_fused(usd, B_))
    if controlnet:
        orc = ocn.ControlNetStreamOracle(fused, cfg, ow.to_float(vsd), ow.to_float(cn), tl, 128, 128)
    else:
        orc = ostream.StreamOracle(fused, cfg, ow.to_float(vsd), tl, 128, 128)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    for i in range(len(tl) + 2):
        frame = ow.make_frame(128, 128, seed=40 + i)
        got = sd.step_u8(frame.to(cuda)).cpu()
        ref = opipe.frame_to_u8(orc, frame)
        d = (got.int() - ref.int()).abs()
        print(f"frame {i}: u8 max |d| {d.max().item()}, share within 2: {(d <= 2).float().mean().item():.5f}")
        assert (d <= 2).float().mean().item() >= 0.999 and d.max().item() <= 8, f"frame {i}: max |d| {d.max().item()}"


def test_refusals(cuda, tmp_path):
    from ai_rtc_agent_b200.host import capi
    arch, cfg, usd, vsd, emb = _weights(False)
    plain = _engine(arch, usd, vsd, emb, [32], False)
    with pytest.raises(RuntimeError, match="live_lora"):
        plain.apply_lora({})
    rc = plain._lib.b2sd_apply_lora(plain._handle, 0, None, plain._stream())
    assert rc != 0 and b"not live" in plain._lib.b2sd_last_error()
    live = _engine(arch, usd, vsd, emb, [32], True)
    blob = str(tmp_path / "x.b2pack")
    plain.export_packed(blob)
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    with pytest.raises(ValueError):
        StreamDiffusion(arch, {}, {}, [32], lambda p: emb, width=128, height=128, packed_blob=blob, live_lora=True)
    f = capi.LoraFactor(b"vae.encoder.layers.0.weight", 1, 1, 4, 0, 1.0)
    assert live._lib.b2sd_apply_lora(live._handle, 1, f, live._stream()) != 0
    assert b"not a UNet weight matrix" in live._lib.b2sd_last_error()
    k = b"conv_in.weight"
    assert live._lib.b2sd_load_tensor(live._handle, k, usd["conv_in.weight"].data_ptr(), 0,
                                      (capi.C.c_int64 * 4)(*usd["conv_in.weight"].shape), 4) != 0
