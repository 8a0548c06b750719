"""Canny ControlNet processor on the CPU: the restatement oracle/canny.py against cv2.Canny (golden fixtures, and cv2 itself
where it is installed), the float-frame round trip, thresholds, argument handling and packed-blob keys."""
import os

import numpy as np
import pytest
import torch
from scipy import ndimage

from oracle import canny as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_equals_cv2_on_the_golden_fixtures():
    z = np.load(os.path.join(ROOT, "tests", "golden", "canny_cv2.npz"))
    n = 0
    for i in range(6):
        for j, (lo, hi) in enumerate(z["thresholds"]):
            assert np.array_equal(oc.canny(z[f"img{i}"], lo, hi), z[f"edge{i}_{j}"]), (i, lo, hi)
            n += int(z[f"edge{i}_{j}"].any())
    assert n >= 20   # most cases have edges


def _images(seed):
    rng = np.random.default_rng(seed)
    for k in range(12):
        h, w = (int(v) for v in rng.integers(3, 120, 2))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if k % 3 == 1:
            img = ndimage.gaussian_filter(img.astype(np.float64), (rng.uniform(0.8, 2.5),) * 2 + (0,)).clip(0, 255).astype(np.uint8)
        elif k % 3 == 2:
            yy, xx = np.mgrid[:h, :w]
            img = np.stack([(xx * 7 + yy * 3) % 256, ((xx // 5 + yy // 5) % 2) * 200, (yy * yy + xx) % 256], -1).astype(np.uint8)
        yield img


@pytest.mark.parametrize("th", [(100, 200), (200, 100), (75, 75), (10.9, 99.99), (0, 0), (500, 2100), (-2.5, 40)])
def test_oracle_equals_cv2(th):
    cv2 = pytest.importorskip("cv2")
    for img in _images(sum(map(int, th)) & 0xffff):
        assert np.array_equal(oc.canny(img, *th), cv2.Canny(img, *th)), (img.shape, th)


def test_oracle_equals_cv2_on_a_serpentine_1024():
    """One strong spot feeding a weak serpentine across a 1024^2 frame, and diagonal staircases (tests/test_canny_gpu.py's
    adversarial hysteresis cases): every candidate of the serpentine is kept"""
    from tests.test_canny_gpu import _diagonal, _serpentine
    for make in (_serpentine, _diagonal):
        img = make()[0].numpy()
        cls = oc.classes(img)
        e = oc.hysteresis(cls)
        assert (cls == 2).sum() < 0.05 * (cls > 0).sum() and (e == 255).sum() > 0.5 * (cls > 0).sum()
        try:
            import cv2
        except ImportError:
            continue
        assert np.array_equal(e, cv2.Canny(img, 100, 200))


def test_float_frames_from_u8_round_trip():
    """u8 v -> v / 255 in fp32 or fp16 -> rint(clamp(x, 0, 1) * 255) gives back v (fp16 error <= 255 * 2^-11 < 0.5)"""
    v = torch.arange(256, dtype=torch.uint8).view(1, 16, 16).repeat(3, 1, 1)
    for dt in (torch.float32, torch.float16):
        x = (v.float() / 255.0).to(dt)
        assert np.array_equal(oc.to_u8(x.numpy()), v.permute(1, 2, 0).numpy()), dt
    assert np.array_equal(oc.to_u8(np.array([-0.5, 0.0019, 1.7, np.nan], dtype=np.float32).reshape(1, 1, 4).repeat(3, 0))[0, :, 0],
                          [0, 0, 255, 0])


def test_thresholds():
    assert oc.thresholds(200, 100) == (100, 200)
    assert oc.thresholds(50.9, 50.2) == (50, 50)
    assert oc.thresholds(-0.5, 3000.7) == (-1, 3000)
    from ai_rtc_agent_b200.host.stream import check_canny_thresholds
    assert check_canny_thresholds(1, 2) == (1.0, 2.0)
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError, match="finite"):
            check_canny_thresholds(bad, 100)


def _load_model_calls(monkeypatch, **kw):
    """Construct a wrapper with canny_processor set (as StreamDiffusionPipeline does) and _load_model replaced by a recorder"""
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    calls = []
    monkeypatch.setattr(StreamDiffusionWrapper, "_load_model", lambda self, **a: calls.append(a) or None)
    w = StreamDiffusionWrapper.__new__(StreamDiffusionWrapper)
    w.canny_processor = True
    w.__init__("tiny-turbo", [32], **kw)
    return calls


def test_plain_wrapper_keeps_the_reference_refusal_of_canny(monkeypatch):
    """Without canny_processor the constructor refuses "canny" by name, as the reference's does"""
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    monkeypatch.setattr(StreamDiffusionWrapper, "_load_model", lambda self, **a: None)
    for ids, procs in (("c", "canny"), (["a", "b"], ["hed", "canny"]), (["a"], ["canny"])):
        with pytest.raises(NotImplementedError, match="'canny'.*canny_processor"):
            StreamDiffusionWrapper("tiny-turbo", [32], controlnet_id_or_path=ids, controlnet_processor_id=procs)


def test_pipeline_enables_canny_on_its_wrapper(monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P

    class Stop(Exception):
        pass
    seen = []

    def init(self, **kw):
        seen.append((self.canny_processor, kw["controlnet_processor_id"]))
        raise Stop
    monkeypatch.setattr(P.StreamDiffusionWrapper, "__init__", init)
    monkeypatch.delenv("B200SD_CONTROLNET", raising=False)
    with pytest.raises(Stop):
        P.StreamDiffusionPipeline("model", controlnet="c", controlnet_processor="canny")
    assert seen == [(True, "canny")]


def test_wrapper_takes_canny_alone_and_in_lists(monkeypatch):
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path="c", controlnet_processor_id="canny")
    assert calls[0]["controlnet_processor_id"] == "canny"
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path=["c"], controlnet_processor_id=["canny"])
    assert (calls[0]["controlnet_id_or_path"], calls[0]["controlnet_processor_id"]) == ("c", "canny")
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path=["a", "b", "c"], controlnet_processor_id=["canny", "hed", None])
    assert calls[0]["controlnet_processor_id"] == ["canny", "hed", None]
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path=["a", "b"], controlnet_processor_id="canny")
    assert calls[0]["controlnet_processor_id"] == ["canny", "canny"]


@pytest.mark.parametrize("proc", ["depth", "openpose", "mlsd", "Canny"])
def test_wrapper_rejects_other_control_preprocessors(proc):
    """With canny_processor set every id other than "hed", "canny" and None is still refused by name"""
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    for ids, procs in (("c", proc), (["a", "b"], ["canny", proc])):
        w = StreamDiffusionWrapper.__new__(StreamDiffusionWrapper)
        w.canny_processor = True
        with pytest.raises(NotImplementedError, match=repr(proc)):
            w.__init__("tiny-turbo", [32], controlnet_id_or_path=ids, controlnet_processor_id=procs)


def test_stream_refuses_bad_processor_lists():
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    with pytest.raises(NotImplementedError, match="'depth'"):
        StreamDiffusion(A.TINY_TURBO, {}, {}, [32], None, controlnet_sd={}, control_processors=["depth"])
    with pytest.raises(ValueError, match="one processor per ControlNet"):
        StreamDiffusion(A.TINY_TURBO, {}, {}, [32], None, controlnet_sd={}, control_processors=["canny", None])
    with pytest.raises(ValueError, match="hed_sd"):
        StreamDiffusion(A.TINY_TURBO, {}, {}, [32], None, controlnet_sd={}, control_processors=["hed"])


def test_blob_keys_tell_canny_from_hed_and_the_frame():
    from ai_rtc_agent_b200.host import weights as W
    args = ("eng", "lykon/dreamshaper-8", "sd15", True, None, None, None, False)
    keys = {W.packed_blob_path(*args, controlnet="c", control_processor=p) for p in ("canny", "hed", None)}
    keys |= {W.packed_blob_path(*args, controlnet=["a", "b"], control_processor=p)
             for p in (["canny", None], ["hed", None], [None, None], ["canny", "hed"])}
    assert len(keys) == 7


def test_pack_cli_takes_canny():
    from ai_rtc_agent_b200 import pack
    a = pack.build_parser().parse_args(["--controlnet-id", "lllyasviel/control_v11p_sd15_canny", "--controlnet-processor-id",
                                        "canny"])
    assert a.controlnet_processor_id == "canny"


def test_ctypes_mirrors_of_the_canny_launch_records(tmp_path):
    """sizeof / offsetof of the two Canny launch-record structs against their ctypes mirrors"""
    import ctypes
    import shutil
    import subprocess
    if not shutil.which("gcc"):
        pytest.skip("no gcc")
    from ai_rtc_agent_b200.host import capi
    lines, want = [], []
    for name, cls in {"b2sd_canny_head_args": capi.CannyHeadArgs, "b2sd_canny_ccl_args": capi.CannyCclArgs}.items():
        lines.append(f'printf("%zu\\n", sizeof({name}));')
        want.append(ctypes.sizeof(cls))
        for field, _ in cls._fields_:
            lines.append(f'printf("%zu\\n", offsetof({name}, {field}));')
            want.append(getattr(cls, field).offset)
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sd.h"\nint main(void){\n' + "\n".join(lines) +
                   "\nreturn 0;}\n")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(tmp_path / "l")], check=True)
    got = [int(v) for v in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True, check=True).stdout.split()]
    assert got == want
