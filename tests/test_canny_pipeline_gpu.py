"""Canny thresholds through the public interface on the H100: StreamDiffusionPipeline(controlnet_processor="canny") viewers
with thresholds of their own (one on a LoRA style, set before its style move and kept through it and through a
ControlNet-scale update), each bit-identical to a pipeline whose global thresholds are that viewer's; a global update replaces
them; updates between enqueued frames; a pipeline without a Canny net refuses the update."""
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


def _pipe(model_id, tl, lanes=None, processor="canny"):
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    arch, _, usd, vsd, _ = _weights("turbo" in model_id)
    W.register_preloaded(model_id, arch, usd, vsd)
    try:
        return StreamDiffusionPipeline(model_id, t_index_list=tl, width=128, height=128, lanes=lanes, live_lora=True,
                                       per_peer_streams=True, controlnet="synthetic-controlnet", controlnet_processor=processor)
    finally:
        W._PRELOADED.pop(model_id, None)


def _single(model_id, tl, lanes, thresholds, idx, lora=None):
    """One viewer alone on a pipeline whose global thresholds (and style) are `thresholds` (and `lora`)"""
    p = _pipe(model_id, tl, lanes)
    if lora:
        p.update_lora(lora)
    p.update_canny_thresholds(*thresholds)
    with p.open_stream() as v:
        return [t.result().cpu() for t in [v.enqueue(_frame(i)) for i in idx]]


@pytest.mark.parametrize("model_id,tl,lanes", [("tiny-sd15", T4, 2), ("tiny-turbo", [32], 4)], ids=["T4-2lanes", "T1-4lanes"])
def test_viewers_with_their_own_thresholds_equal_single_viewer_pipelines(cuda, tmp_path, env, model_id, tl, lanes):
    _, _, usd, _, _ = _weights("turbo" in model_id)
    lora, _ = _loras(tmp_path, usd)
    n = 4
    p = _pipe(model_id, tl, lanes)
    views = [p.open_stream() for _ in range(3)]
    views[1].update_canny_thresholds(40, 90)
    views[2].update_canny_thresholds(150, 60)
    views[2].update_lora(lora)      # a style move keeps the viewer's thresholds
    views[2].update_controlnet_scale(1.0)   # and so does a ControlNet update (here to the global settings' values)
    assert views[0].canny_thresholds == (100.0, 200.0) and views[2].canny_thresholds == (150.0, 60.0)
    got = [[] for _ in views]
    for i in range(n):
        for k, v in enumerate(views):
            got[k].append(v.enqueue(_frame(i)))
    got = [[t.result().cpu() for t in g] for g in got]
    want = [_single(model_id, tl, lanes, th, range(n), lora=lo)
            for th, lo in (((100, 200), None), ((40, 90), None), ((150, 60), lora))]
    for k in range(3):
        _equal(got[k], want[k], f"viewer {k}")
    assert not torch.equal(got[1][0], got[0][0]), "the thresholds must change the frame"
    p.update_canny_thresholds(70, 140)   # a global update replaces the viewers' own thresholds
    assert all(v.canny_thresholds == (70.0, 140.0) for v in views)
    for v in views:
        v.close()


def test_updates_between_enqueued_frames(cuda, env):
    """Frames enqueued before a global or per-viewer update use the old thresholds, frames after it the new ones"""
    p = _pipe("tiny-turbo", [32], 2)
    v = p.open_stream()
    tickets = [v.enqueue(_frame(0))]
    p.update_canny_thresholds(30, 60)
    tickets.append(v.enqueue(_frame(1)))
    v.update_canny_thresholds(180, 90)
    tickets.append(v.enqueue(_frame(2)))
    got = [t.result().cpu() for t in tickets]
    v.close()
    for i, th in enumerate([(100, 200), (30, 60), (180, 90)]):
        _equal(got[i:i + 1], _single("tiny-turbo", [32], 2, th, [i]), f"frame {i}")


def test_a_pipeline_without_canny_refuses_the_update(cuda, env):
    p = _pipe("tiny-turbo", [32], 1, processor="hed")
    with pytest.raises(RuntimeError, match="canny"):
        p.update_canny_thresholds(50, 100)
    with p.open_stream() as v, pytest.raises(RuntimeError, match="canny"):
        v.update_canny_thresholds(50, 100)
