"""Launch audit of a two-ControlNet engine: every launch of a full-size SD-1.5 512x512 T=4 frame with a frame net and a HED
net checked against float64 (tests/test_launch_audit_gpu.py's Auditor), each net's zero convs against a reference that applies
that net's own per-slot scales as the launch reads them (tests/test_controlnet_scale_audit_gpu.py's ScaleAuditor), and the
audited frame equal to a CUDA-graph step of an identical lane."""
import pytest
import torch

from tests.test_controlnet_scale_audit_gpu import ScaleAuditor
from tests.test_launch_audit_gpu import _release_device_memory

pytestmark = pytest.mark.gpu


def _engine(tl, procs):
    """A full-size SD-1.5 engine at 512x512 with one seeded ControlNet per entry of procs, and a lane with its launch policy"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.SD15
    usd, vsd = ow.make_unet_weights(cfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    nets = [ocn.make_weights(cfg, seed=5678 + 31 * i) for i in range(len(procs))]
    hed = {k: v.half().float() for k, v in A.synthetic_hed().items()} if "hed" in procs else None
    sd = StreamDiffusion(A.SD15, usd, vsd, tl, lambda p: emb, width=512, height=512, device="cuda", controlnet_sd=nets,
                         control_processors=procs, hed_sd=hed)
    sd.prepare("p", guidance_scale=0.0)
    lane = sd.add_lane()
    lane.set_concurrency(1)   # the audited engine's launch policy, so that both compute bit-identical frames
    lane._prepare_like(sd)
    return sd, lane


def test_launch_audit_of_a_frame_and_a_hed_controlnet(cuda):
    from ai_rtc_agent_b200.host.stream import control_scales
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    scale, start, end = [0.7, 1.2], [0.0, 0.3], [0.6, 1.0]
    rows = [control_scales((scale[i], start[i], end[i]), tl, 50) for i in range(2)]
    assert rows == [[0.7, 0.7, 0.0, 0.0], [1.2, 1.2, 1.2, 1.2]]   # net 0 masks half the slots, net 1 none
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    _release_device_memory()
    sd = lane = None
    try:
        sd, lane = _engine(tl, [None, "hed"])
        sd.set_control_scale(scale, start, end)   # the engine and its lane
        frames = [ow.make_frame(512, 512, seed=400 + i).cuda() for i in range(2)]
        sd.step_u8(frames[0])
        lane.step_u8(frames[0])
        aud = ScaleAuditor()
        got = sd.audit_step(frames[1], aud).clone()
        want = lane.step_u8(frames[1])
        torch.cuda.synchronize()
        print("\n" + aud.table("sd15-T4-512 frame + HED ControlNets"))
        assert not aud.other, dict(aud.other)
        for cls in aud.launches:
            assert aud.checked[cls] == aud.launches[cls], cls
        assert aud.calls == sd.launches_per_step
        assert aud.scaled == 26, aud.scaled   # 12 controlnet_down_blocks + controlnet_mid_block, per net
        assert aud.scales == {tuple(torch.tensor(r, dtype=torch.float32).tolist()) for r in rows}, aud.scales
        assert torch.equal(got, want), "the audited frame differs from a graph step of an identical lane"
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        if sd is not None:
            sd.lanes.clear()
        sd = lane = None
        _release_device_memory()
