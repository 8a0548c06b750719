"""Launch audit of a ControlNet engine whose conditioning scale is not 1 and whose guidance window masks some slots: every
launch of a full-size SD-1.5 512x512 T=4 ControlNet + HED frame checked against float64 (tests/test_launch_audit_gpu.py's
Auditor), the zero convs' reference applying each slot's scale as the launch reads it (b2sd_igemm_desc.acc_scale_b), and the
audited frame equal to a CUDA-graph step of an identical lane."""
import pytest
import torch

from tests import launch_ref as R
from tests.test_launch_audit_gpu import Auditor, _dev, _engine, _release_device_memory, _vec

pytestmark = pytest.mark.gpu


def _scaled(epilogue, scale):
    """launch_ref.epilogue with the per-item factor: s[b] * (what the epilogue makes of acc + bias) + res_scale * res"""
    def epi(d, acc, colbias=None, res=None, rowstat_in=None, colsum=None):
        assert not d["flags"] & (R.IG_RELU | R.IG_SILU | R.IG_GEGLU) and colsum is None
        x = epilogue(d, acc, colbias, None, rowstat_in, colsum)
        b = torch.arange(x.shape[0], device=x.device) // (d["ho"] * d["wo"])
        x = x * scale.double().to(x.device)[b][:, None]
        return x if res is None else x + d["res_scale"] * res.double()
    return epi


class ScaleAuditor(Auditor):
    def __init__(self):
        super().__init__()
        self.scaled = 0          # launches with a per-item scale checked
        self.scales = set()

    def _before_igemm(self, rec):
        s = super()._before_igemm(rec)
        d = R.as_dict(rec.igemm)
        if d["acc_scale_b"]:
            s["acc_scale_b"] = _vec(d["acc_scale_b"], d["nb"])
        return s

    def _after_igemm(self, rec, kind, label, s):
        scale = s.get("acc_scale_b")
        if scale is None:
            return super()._after_igemm(rec, kind, label, s)
        d = R.as_dict(rec.igemm)
        # wrong references of the scale itself, added to the audit's own (lost K, residual omitted, ...)
        rows = R.rows_of(d)
        atol, rtol = R.TOL["contraction"]
        acc = R.contraction_acc(d, s["src"], s["w"], None, torch.float32)
        out = _dev(d["out"], rows, d["n_valid"], d["ldc"])
        right = _scaled(R.epilogue, scale)(d, acc, s["colbias"], s["res"])
        s_row = scale.double().to(right.device)[torch.arange(rows, device=right.device) // (d["ho"] * d["wo"])][:, None]
        extra = {"per-slot scale ignored": R.epilogue(d, acc, s["colbias"], s["res"]),
                 "slot 0's scale for every slot": _scaled(R.epilogue, scale[:1].expand_as(scale))(d, acc, s["colbias"], s["res"]),
                 "scale on the residual too": right + (s_row - 1.0) * s["res"].double()}
        extra = {k: R.tol_units(v, right, atol, rtol) for k, v in extra.items()}
        assert R.tol_units(out, right, atol, rtol) <= 1.0, f"{label}: zero conv off its per-slot reference"
        assert max(extra.values()) >= 10.0, f"{label}: the scale checks do not discriminate: {extra}"
        record = self._record

        def with_extra(cls, lbl, units, wrongs, exact=False):
            return record(cls, lbl, units, {**wrongs, **extra}, exact)
        epilogue = R.epilogue
        R.epilogue, self._record = _scaled(epilogue, scale), with_extra
        try:
            super()._after_igemm(rec, kind, label, s)
        finally:
            R.epilogue = epilogue
            del self._record
        self.scaled += 1
        self.scales.add(tuple(scale.tolist()))


def test_launch_audit_with_a_scaled_and_windowed_controlnet(cuda):
    from ai_rtc_agent_b200.host.stream import control_scales
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    control = (0.7, 0.0, 0.6)   # slots 0 and 1 kept (19 / 50, 27 / 50 <= 0.6), slots 2 and 3 masked
    want_scales = control_scales(control, tl, 50)
    assert want_scales == [0.7, 0.7, 0.0, 0.0]
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    _release_device_memory()
    sd = lane = None
    try:
        sd, lane, _ = _engine(turbo=False, tl=tl, hw=512, full=True, cn=True, hed=True)
        sd.set_control_scale(*control)   # the engine and its lane
        frames = [ow.make_frame(512, 512, seed=300 + i).cuda() for i in range(2)]
        sd.step_u8(frames[0])
        lane.step_u8(frames[0])
        aud = ScaleAuditor()
        got = sd.audit_step(frames[1], aud).clone()
        want = lane.step_u8(frames[1])
        torch.cuda.synchronize()
        print("\n" + aud.table("sd15-T4-512-cn-hed scaled"))
        assert not aud.other, dict(aud.other)
        for cls in aud.launches:
            assert aud.checked[cls] == aud.launches[cls], cls
        assert aud.calls == sd.launches_per_step
        assert aud.scaled == 13, aud.scaled   # 12 controlnet_down_blocks + controlnet_mid_block
        assert aud.scales == {tuple(torch.tensor(want_scales, dtype=torch.float32).tolist())}, aud.scales
        assert torch.equal(got, want), "the audited frame differs from a graph step of an identical lane"
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        if sd is not None:
            sd.lanes.clear()
        sd = lane = None
        _release_device_memory()
