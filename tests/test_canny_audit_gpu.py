"""Launch audit of a full-size synthetic SD-1.5 512x512 T=4 frame with a Canny ControlNet: every launch is issued as recorded
(the count equals launches_per_step), and the Canny launches are compared exactly: canny_head's class map with
oracle/canny.py's on the frame, the hysteresis output with the oracle's edge image, and the scratch forest with the rule that
every candidate ends up pointing at a root of its own component."""
import numpy as np
import pytest
import torch

from oracle import canny as oc
from tests.test_canny_gpu import T4, _engine, _models, _nets, _structured

pytestmark = pytest.mark.gpu


class _Dev:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "strides": None, "typestr": typestr, "data": (ptr, False), "version": 3}


def _read(ptr, n, typestr="|u1"):
    return torch.as_tensor(_Dev(int(ptr), int(n), typestr), device="cuda").clone().cpu().numpy()


def test_audit_fullsize_sd15_canny_512(cuda):
    from ai_rtc_agent_b200.host import capi
    from scipy import ndimage
    models = _models(False, full=True)
    sd = _engine(models, T4, 512, _nets(models[0], 1)[0], ["canny"])
    sd.set_canny_thresholds(80, 170)
    frame = _structured(512, 512, 7)
    img = frame[0].numpy()
    want_cls = oc.classes(img, 80, 170)
    want = oc.hysteresis(want_cls)
    seen = []

    def check(i, after, rec):
        if not after:
            seen.append(rec.kind)
            return
        if rec.kind == capi.LAUNCH_CANNY_HEAD:
            a = rec.canny_head
            assert (a.h, a.w, a.low, a.high, a.in_flags) == (512, 512, 80, 170, capi.SC_IN_U8)
            assert np.array_equal(_read(a.cls, 512 * 512).reshape(512, 512), want_cls), "canny_head class map"
        elif rec.kind == capi.LAUNCH_CANNY_CCL:
            a = rec.canny_ccl
            if a.stage == 2:   # every candidate points at a root, one root per component
                parent = _read(a.parent, 512 * 512 * 4, "|u1").view(np.int32)
                lab, _ = ndimage.label(want_cls > 0, structure=np.ones((3, 3), dtype=bool))
                cand = np.flatnonzero(want_cls.ravel() > 0)
                roots = parent[cand]
                assert np.array_equal(parent[roots], roots), "a candidate's parent is not a root"
                assert np.array_equal(lab.ravel()[roots], lab.ravel()[cand]), "a root outside its pixel's component"
                pairs = set(zip(lab.ravel()[cand].tolist(), roots.tolist()))
                assert len(pairs) == len(set(lab.ravel()[cand].tolist())), "a component with several roots"
            if a.stage == 3:
                out = _read(a.out, 512 * 512 * 3).reshape(512, 512, 3)
                assert np.array_equal(out, np.repeat(want[..., None], 3, 2)), "hysteresis output"

    sd.audit_step(frame.cuda(), check)
    assert len(seen) == sd.launches_per_step
    assert seen.count(capi.LAUNCH_CANNY_HEAD) == 1 and seen.count(capi.LAUNCH_CANNY_CCL) == 4
    assert capi.LAUNCH_OTHER not in seen
