"""Canny ControlNet processor on the H100: the `canny` tap (u8 edge image) and `canny_class` tap (class map) equal the integer
restatement oracle/canny.py exactly, at every size, input kind and resize, and on adversarial hysteresis cases; repeated steps
are bit-identical; the whole frame matches the fp32 restatement tests/canny_ref.py; Canny runs once per frame however many nets
read it; threshold updates, per-state thresholds on lanes and styles, and packed blobs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import canny as oc
from tests.canny_ref import CannyStreamOracle

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]


def _models(turbo=True, full=False):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    if full:
        cfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
    else:
        cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    return cfg, arch, ow.make_unet_weights(cfg), ow.make_taesd_weights(), ow.make_prompt_embeds(cfg.cross_attention_dim)


def _nets(cfg, n):
    from oracle import controlnet as ocn
    return [ocn.make_weights(cfg, seed=5678 + 31 * i) for i in range(n)]


def _engine(models, tl, hw, cns, procs, hed=None, graph=True, blob=None, live_lora=False, concurrency=1):
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    cfg, arch, usd, vsd, emb = models
    height, width = (hw, hw) if isinstance(hw, int) else hw
    kw = dict(width=width, height=height, use_cuda_graph=graph, live_lora=live_lora, control_processors=procs)
    if blob is not None:
        sd = StreamDiffusion(arch, {}, {}, tl, lambda p: emb, packed_blob=blob, hed_sd={} if hed is not None else None,
                             controlnet_sd=[{}] * len(procs) if isinstance(cns, list) else {}, **kw)
    else:
        sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, controlnet_sd=cns, hed_sd=hed, **kw)
    if concurrency > 1:   # lanes run the throughput launch policy: compare them with engines that run it too
        sd.set_concurrency(concurrency)
    sd.prepare("p", guidance_scale=0.0)
    return sd


def _hed16():
    from ai_rtc_agent_b200.host import arch as A
    return {k: v.half().float() for k, v in A.synthetic_hed().items()}


def _structured(h, w, seed):
    """(1, h, w, 3) u8: discs and bars of several contrasts over a noisy colour field (edges of every strength)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float64)
    img = 90 + 40 * np.sin(xx / 17.0 + seed) * np.cos(yy / 23.0)
    for _ in range(8):
        cy, cx, r, c = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(4, max(6, min(h, w) / 3)), rng.uniform(-90, 90)
        img = img + c * ((yy - cy) ** 2 + (xx - cx) ** 2 < r * r)
    img = img[..., None] + np.array([0, 25, -20]) + rng.normal(0, 6, (h, w, 3))
    return torch.from_numpy(img.clip(0, 255).astype(np.uint8))[None]


def _resized(frame_u8, h, w):
    """the engine's nearest resize of a (1, H', W', 3) u8 frame to h x w (torch's index rule)"""
    x = frame_u8.permute(0, 3, 1, 2).float()
    return F.interpolate(x, size=(h, w), mode="nearest").round().to(torch.uint8)[0].permute(1, 2, 0).numpy()


def _taps(sd):
    edge = sd.get_tensor("canny")[0].to(torch.uint8).numpy()
    cls = sd.get_tensor("canny_class")[0, ..., 0].to(torch.uint8).numpy()
    return edge, cls


def _check_taps(sd, img_u8, lo, hi, what):
    edge, cls = _taps(sd)
    want_cls = oc.classes(img_u8, lo, hi)
    want = np.repeat(oc.hysteresis(want_cls)[..., None], 3, axis=2)
    assert np.array_equal(cls, want_cls), f"{what}: class map differs at {np.argwhere(cls != want_cls)[:5].tolist()}"
    assert np.array_equal(edge, want), f"{what}: edge map differs at {int((edge != want).sum())} values"
    return edge


def _step(sd, frame_u8, kind, state=None):
    """one step of sd on the (1, H', W', 3) u8 frame, given as u8, or as fp32 / fp16 v / 255 NCHW"""
    f = frame_u8.cuda()
    if kind == "u8":
        return sd.step_u8(f, state=state)
    x = f.permute(0, 3, 1, 2).float() / 255.0
    return sd(x.half() if kind == "f16" else x, state=state)


# ---- the tap against the oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,inp", [(64, (64, 64)), ((128, 192), (128, 192)), ((192, 128), (192, 128)), (512, (512, 512)),
                                    (1024, (1024, 1024)), (512, (480, 640)), ((256, 448), (720, 1280)), (128, (97, 131))])
def test_canny_tap_equals_the_oracle(cuda, hw, inp):
    """Every size from 64^2 to 1024^2, non-square engines and camera-sized frames resized by the engine, each input kind, and
    thresholds reversed, equal, fractional, 0 and above 2040: the class map and the edge image exactly."""
    h, w = (hw, hw) if isinstance(hw, int) else hw
    sd = _engine(_models(), [32], hw, _nets(_models()[0], 1)[0], ["canny"])
    for i, (kind, th) in enumerate([("u8", (100, 200)), ("f32", (200, 100)), ("f16", (60, 60)), ("u8", (50.7, 120.2)),
                                    ("u8", (0, 0)), ("u8", (30, 2100))]):
        frame = _structured(*inp, seed=i)
        sd.set_canny_thresholds(*th)
        _step(sd, frame, kind)
        _check_taps(sd, _resized(frame, h, w), *th, f"{hw} from {inp}, {kind}, thresholds {th}")


def test_float_frames_from_u8_give_the_same_map(cuda):
    """A frame that came from u8 as v / 255 in fp32 or fp16 gives back v: the three input kinds give the same edge image"""
    sd = _engine(_models(), [32], 128, _nets(_models()[0], 1)[0], ["canny"])
    frame = torch.arange(256, dtype=torch.uint8).repeat(128 * 128 * 3 // 256 + 1)[:128 * 128 * 3].view(1, 128, 128, 3)
    frame = frame[:, torch.randperm(128, generator=torch.Generator().manual_seed(0))]
    maps = []
    for kind in ("u8", "f32", "f16"):
        _step(sd, frame, kind)
        maps.append(_taps(sd))
    for m in maps[1:]:
        assert np.array_equal(m[0], maps[0][0]) and np.array_equal(m[1], maps[0][1])
    _check_taps(sd, frame[0].numpy(), 100, 200, "f16 frame")


def _serpentine(n=1024, band=24, contrast=30):
    """A low-contrast band snaking across an n x n frame (its border crosses every tile border), strong at one spot only"""
    mask = np.zeros((n, n), dtype=bool)
    for k, y in enumerate(range(8, n - band, 2 * band)):
        mask[y:y + band, 8:n - 8] = True
        x = n - 8 - band if k % 2 == 0 else 8
        mask[y:y + 2 * band + 1, x:x + band] = True
    img = np.full((n, n), 100.0) + contrast * mask
    img[:40, :40] += 100 * mask[:40, :40]   # the only strong edges
    return torch.from_numpy(np.repeat(img[..., None], 3, 2).clip(0, 255).astype(np.uint8))[None]


def _diagonal(n=1024, contrast=30):
    """Staircase boundaries at 45 degrees: candidates joined only through diagonal neighbours, strong at one end"""
    yy, xx = np.mgrid[:n, :n]
    img = 100.0 + (contrast + 60 * np.exp(-(yy / 12.0) ** 2)) * (((xx - yy) // 97) % 2)
    return torch.from_numpy(np.repeat(img[..., None], 3, 2).clip(0, 255).astype(np.uint8))[None]


@pytest.mark.parametrize("make", [_serpentine, _diagonal])
def test_adversarial_hysteresis_1024(cuda, make):
    """One strong spot feeding a long weak chain across every tile border of a 1024^2 frame, and diagonal-only chains: the
    edge image equals the oracle's, most of the weak chain is kept, and repeated steps are bit-identical."""
    sd = _engine(_models(), [32], 1024, _nets(_models()[0], 1)[0], ["canny"])
    frame = make()
    _step(sd, frame, "u8")
    edge = _check_taps(sd, frame[0].numpy(), 100, 200, make.__name__)
    cls = oc.classes(frame[0].numpy(), 100, 200)
    assert (cls == 2).sum() < 0.05 * (cls > 0).sum(), "the case must be mostly weak candidates"
    assert (edge[..., 0] == 255).sum() > 0.5 * (cls > 0).sum(), "hysteresis must carry the strong spot along the chain"
    for _ in range(3):
        _step(sd, frame, "u8")
        assert np.array_equal(_taps(sd)[0], edge)


def test_repeated_steps_are_bit_identical(cuda):
    sd = _engine(_models(), [32], 512, _nets(_models()[0], 1)[0], ["canny"])
    frame = _structured(512, 512, 3)
    outs = [(_step(sd, frame, "u8").cpu(), _taps(sd)) for _ in range(4)]
    for o, (e, c) in outs[1:]:
        assert torch.equal(o, outs[0][0]) and np.array_equal(e, outs[0][1][0]) and np.array_equal(c, outs[0][1][1])


# ---- the frame against the restatement ---------------------------------------------------------------------------------------
def _u8_check(got, ref, what):
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"


def _against_oracle(models, tl, hw, procs, frames, thresholds, hed=None):
    from oracle import pipeline as opipe
    from oracle import weights as ow
    cfg, arch, usd, vsd, emb = models
    nets = _nets(cfg, len(procs))
    h, w = (hw, hw) if isinstance(hw, int) else hw
    sd = _engine(models, tl, hw, nets, procs, hed=hed)
    orc = CannyStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), [ow.to_float(n) for n in nets], procs, tl, w, h, hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    orc.to("cuda")
    try:
        for i, f in enumerate(frames):
            sd.set_canny_thresholds(*thresholds[i])
            orc.thresholds = thresholds[i]
            out = sd.step_u8(f.cuda())
            with torch.no_grad():
                ref = opipe.frame_to_u8(orc, f.cuda())
            assert np.array_equal(_taps(sd)[0], (orc.last_canny[0].permute(1, 2, 0) * 255).round().byte().cpu().numpy())
            _u8_check(out, ref, f"frame {i}")
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("turbo,tl,hw,procs", [(False, T4, 128, ["canny"]), (True, [32], (64, 192), ["canny", None]),
                                               (False, [18, 35], (192, 128), [None, "canny"])])
def test_tiny_frames_match_the_restatement(cuda, turbo, tl, hw, procs):
    h, w = (hw, hw) if isinstance(hw, int) else hw
    frames = [_structured(h, w, 10 + i) for i in range(3)]
    _against_oracle(_models(turbo), tl, hw, procs, frames, [(100, 200), (40, 90), (150, 60)])


def test_fullsize_sd15_canny_matches_the_restatement_512(cuda):
    frames = [_structured(512, 512, 20 + i) for i in range(2)]
    _against_oracle(_models(False, full=True), T4, 512, ["canny"], frames, [(100, 200), (70, 140)])


# ---- launches, lanes, graphs -------------------------------------------------------------------------------------------------
def test_canny_hed_and_frame_nets_run_canny_once(cuda):
    from ai_rtc_agent_b200.host import capi
    models = _models()
    procs = ["canny", "hed", None, "canny"]
    sd = _engine(models, [32], 128, _nets(models[0], 4), procs, hed=_hed16())
    one = _engine(models, [32], 128, _nets(models[0], 1)[0], ["canny"])
    plain = _engine(models, [32], 128, _nets(models[0], 1)[0], None)
    assert one.launches_per_step == plain.launches_per_step + 1 + 4   # canny_head + four hysteresis launches
    seen = []
    frame = _structured(128, 128, 5).cuda()
    sd.audit_step(frame, lambda i, after, rec: seen.append((rec.kind, rec.label, rec.canny_ccl.stage)) if not after else None)
    assert sum(k == capi.LAUNCH_CANNY_HEAD for k, _, _ in seen) == 1
    assert [s for k, _, s in seen if k == capi.LAUNCH_CANNY_CCL] == [0, 1, 2, 3]
    assert sum(k == capi.LAUNCH_HED_FUSE for k, _, _ in seen) == 1
    assert len(seen) == sd.launches_per_step
    _check_taps(sd, frame[0].cpu().numpy(), 100, 200, "four nets")


def test_lanes_and_graphs(cuda):
    """A lane and an eager engine give the graph engine's frames and maps, bit for bit"""
    models = _models()
    net = _nets(models[0], 1)[0]
    sd = _engine(models, [32], 256, net, ["canny"], concurrency=2)
    eager = _engine(models, [32], 256, net, ["canny"], graph=False, concurrency=2)
    sd.set_canny_thresholds(80, 160)
    eager.set_canny_thresholds(80, 160)
    lane = sd.add_lane()
    assert lane.canny_thresholds == (80.0, 160.0)
    for i in range(3):
        f = _structured(256, 256, 30 + i)
        a = _step(sd, f, "u8").cpu()
        ta = _taps(sd)
        b = _step(lane, f, "u8").cpu()
        c = _step(eager, f, "u8").cpu()
        assert torch.equal(a, b) and torch.equal(a, c)
        assert np.array_equal(ta[0], _taps(lane)[0]) and np.array_equal(ta[0], _taps(eager)[0])


def test_threshold_updates_between_queued_frames(cuda):
    """Frames submitted before an update use the old thresholds, frames after it the new ones, with no synchronisation"""
    models = _models()
    net = _nets(models[0], 1)[0]
    sd = _engine(models, [32], 256, net, ["canny"])
    settings = [(100, 200), (30, 60), (30, 60), (220, 110)]
    frames = [_structured(256, 256, 40 + i).cuda() for i in range(4)]
    outs = []
    for th, f in zip(settings, frames):
        sd.set_canny_thresholds(*th)
        outs.append(sd.step_u8(f))   # nothing waits for the frame
    torch.cuda.synchronize()
    for th, f, o in zip(settings, frames, outs):
        ref = _engine(models, [32], 256, net, ["canny"])
        ref.set_canny_thresholds(*th)
        assert torch.equal(o.cpu(), ref.step_u8(f).cpu()), th


def test_two_states_with_own_thresholds_on_lanes_and_a_style(cuda):
    """Two T = 4 streams with their own thresholds stepped alternately on two lanes and a style of the engine each equal a
    single engine with those thresholds as its global ones; a global update replaces both"""
    models = _models(False)
    net = _nets(models[0], 1)[0]
    sd = _engine(models, T4, 128, net, ["canny"], live_lora=True, concurrency=2)
    engines = [sd, sd.add_lane(), sd.add_style()]
    s1, s2 = sd.new_state(), sd.new_state()
    s1.set_canny_thresholds(40, 90)
    s2.set_canny_thresholds(150, 70)
    refs = []
    for th in [(40, 90), (150, 70)]:
        r = _engine(models, T4, 128, net, ["canny"], concurrency=2)
        r.set_canny_thresholds(*th)
        refs.append(r)
    for i in range(6):
        f = _structured(128, 128, 50 + i).cuda()
        a = engines[i % 3].step_u8(f, state=s1).cpu()
        b = engines[(i + 1) % 3].step_u8(f, state=s2).cpu()
        assert torch.equal(a, refs[0].step_u8(f).cpu()), f"state 1, frame {i}"
        assert torch.equal(b, refs[1].step_u8(f).cpu()), f"state 2, frame {i}"
    sd.set_canny_thresholds(100, 200)
    assert s1.own_canny is None and s2.own_canny is None


def test_packed_blob_round_trip(cuda, tmp_path):
    models = _models()
    nets = _nets(models[0], 2)
    sd = _engine(models, [32], 128, nets, ["canny", None])
    blob = str(tmp_path / "canny.b2pack")
    sd.export_packed(blob)
    again = _engine(models, [32], 128, nets, ["canny", None], blob=blob)
    for i in range(2):
        f = _structured(128, 128, 60 + i).cuda()
        assert torch.equal(sd.step_u8(f).cpu(), again.step_u8(f).cpu())
