"""The ControlNet conditioning scale through the public interface on the H100: viewers of a per-peer pipeline with settings of
their own (one on a LoRA style), each bit-identical to a pipeline whose global settings are that viewer's; updates enqueued
between queued frames; and the packed-blob round trip with settings set after the import."""
import pytest
import torch

from tests.test_peer_styles_gpu import _equal, _frame, _loras, _weights

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]


@pytest.fixture
def env(monkeypatch):
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.setenv("B200SD_SYNTHETIC_WEIGHTS", "1")
    for v in ("B200SD_LANES", "B200SD_MAX_STYLES", "B200SD_POLICY_FRAMES", "B200SD_CONTROLNET"):
        monkeypatch.delenv(v, raising=False)
    return monkeypatch


def _pipe(model_id, tl, lanes=None, processor=None):
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    arch, _, usd, vsd, _ = _weights("turbo" in model_id)
    W.register_preloaded(model_id, arch, usd, vsd)
    try:
        return StreamDiffusionPipeline(model_id, t_index_list=tl, width=128, height=128, lanes=lanes, live_lora=True,
                                       per_peer_streams=True, controlnet="synthetic-controlnet", controlnet_processor=processor)
    finally:
        W._PRELOADED.pop(model_id, None)


def _single(model_id, tl, lanes, control, idx, lora=None, t_index_list=None, processor=None):
    """One viewer alone on a pipeline whose global ControlNet settings (and style) are `control` (and `lora`)"""
    p = _pipe(model_id, tl, lanes, processor)
    if lora:
        p.update_lora(lora)
    p.update_controlnet_scale(*control)
    with p.open_stream() as v:
        if t_index_list is not None:
            v.update_t_index_list(t_index_list)
        return [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in idx]]


@pytest.mark.parametrize("model_id,tl,lanes,own_t", [("tiny-sd15", T4, 2, [10, 20, 30, 40]), ("tiny-turbo", [32], 8, [20])],
                         ids=["T4-2lanes", "T1-8lanes"])
def test_viewers_with_their_own_settings_equal_single_viewer_pipelines(cuda, tmp_path, env, model_id, tl, lanes, own_t):
    """Viewer 0 follows the global settings, viewer 1 has its own scale, viewer 2 its own window and its own t_index_list,
    viewer 3 its own scale on a LoRA style (set before its style move, kept through it).  Interleaved frames on the lanes."""
    _, _, usd, _, _ = _weights("turbo" in model_id)
    lora, _ = _loras(tmp_path, usd)
    n = 4
    p = _pipe(model_id, tl, lanes)
    launches = p.model.stream.launches_per_step
    views = [p.open_stream() for _ in range(4)]
    views[1].update_controlnet_scale(0.6)
    views[2].update_t_index_list(own_t)
    views[2].update_controlnet_scale(1.0, 0.5, 1.0)
    views[3].update_controlnet_scale(-0.5)
    views[3].update_lora(lora)
    assert [v.controlnet_scale for v in views] == [(1.0, 0.0, 1.0), (0.6, 0.0, 1.0), (1.0, 0.5, 1.0), (-0.5, 0.0, 1.0)]
    tickets = {k: [] for k in range(4)}
    for i in range(n):
        for k, v in enumerate(views):
            tickets[k].append(v.enqueue(_frame(10 * k + i)))
    got = {k: [t.result().cpu() for t in ts] for k, ts in tickets.items()}
    wants = [dict(control=(1.0, 0.0, 1.0)), dict(control=(0.6, 0.0, 1.0)),
             dict(control=(1.0, 0.5, 1.0), t_index_list=own_t), dict(control=(-0.5, 0.0, 1.0), lora=lora)]
    for k, w in enumerate(wants):
        _equal(got[k], _single(model_id, tl, lanes, idx=[10 * k + i for i in range(n)], **w), f"viewer {k}")
    assert not torch.equal(got[1][0], _single(model_id, tl, lanes, (1.0, 0.0, 1.0), [10])[0]), "scale 0.6 changes the frames"
    assert p.model.stream.launches_per_step == launches
    # a global update replaces every viewer's own settings; the viewers' own t_index_list stays
    p.update_controlnet_scale(0.8, 0.0, 0.9)
    assert [v.controlnet_scale for v in views] == [(0.8, 0.0, 0.9)] * 4 and views[2].t_index_list == own_t
    for v in views:
        v.close()


def test_updates_split_queued_frames_at_the_call(cuda, env):
    """T = 4: frames enqueued before a global, then a per-viewer update use the old settings, those after it the new ones,
    with no wait in between.  The reference runs the same sequence with the device idle around each update."""
    def run(sync):
        p = _pipe("tiny-sd15", T4, processor="hed")
        launches = p.model.stream.launches_per_step
        out = []
        with p.open_stream() as v:
            for i, update in enumerate([None, lambda: p.update_controlnet_scale(0.6, 0.0, 0.6),
                                        lambda: v.update_controlnet_scale(-0.4, 0.3, 1.0)]):
                if update is not None:
                    if sync:
                        torch.cuda.synchronize()
                    update()
                    if sync:
                        torch.cuda.synchronize()
                ts = [v.enqueue(_frame(4 * i + j)) for j in range(4)]
                out += [t.result().cpu() for t in ts] if sync else ts
            out = [t if isinstance(t, torch.Tensor) else t.result().cpu() for t in out]
        assert p.model.stream.launches_per_step == launches
        return out
    want = run(sync=True)
    got = run(sync=False)
    _equal(got, want, "frames around queued updates")
    assert not torch.equal(want[4], _single("tiny-sd15", T4, None, (1.0, 0.0, 1.0), [4], processor="hed")[0])


@pytest.mark.parametrize("processor", [None, "hed"])
def test_packed_blob_round_trip_with_settings_set_after_import(cuda, tmp_path, processor):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import weights as ow
    arch, cfg, usd, vsd, emb = _weights(False)
    cn = ocn.make_weights(cfg)
    hed = {k: v.half().float() for k, v in A.synthetic_hed().items()} if processor else None
    kw = dict(width=128, height=128)
    fresh = StreamDiffusion(arch, usd, vsd, T4, lambda p: emb, controlnet_sd=cn, hed_sd=hed, **kw)
    fresh.prepare("p", guidance_scale=0.0)
    blob = str(tmp_path / "cn.b2pack")
    fresh.export_packed(blob)
    imported = StreamDiffusion(arch, {}, {}, T4, lambda p: emb, packed_blob=blob, controlnet_sd={},
                               hed_sd={} if processor else None, **kw)
    imported.prepare("p", guidance_scale=0.0)
    for sd in (fresh, imported):
        sd.set_control_scale(0.6, 0.2, 0.8)
    for i in range(4):
        f = ow.make_frame(128, 128, seed=70 + i).cuda()
        assert torch.equal(fresh.step_u8(f).cpu(), imported.step_u8(f).cpu()), f"frame {i}"
