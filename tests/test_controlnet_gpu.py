"""ControlNet on the H100: the new kernel paths against float64 references, the engine against the fp32 oracle
(oracle/controlnet.py) on identical seeded weights, and the bit-exactness properties of lanes, packed blobs and a freshly
initialised ControlNet.

Tolerances as in tests/test_engine_gpu.py: activations max|d| <= 2e-2 * max|ref| and cosine >= 0.999; u8 frames |d| <= 2 LSB on
>= 99.9 % of the pixels, max |d| <= 8."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_discriminates, guarded, hetero

pytestmark = pytest.mark.gpu


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _conv64(x_nhwc, w_oihw, stride=1):
    x = x_nhwc.double().permute(0, 3, 1, 2)
    y = F.conv2d(x, w_oihw.double(), None, stride=stride, padding=w_oihw.shape[-1] // 2)
    return y.permute(0, 2, 3, 1)


def _w(shape, seed, device):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) / math.sqrt(math.prod(shape[1:]))).half().to(device)


# ---- kernels ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,cin,cin_pad,cout,pitch,stride,bn,splits", [
    (128, 128, 16, 64, 16, 64, 1, 16, 1),     # embedding blocks.0: 16 channels stored 64 wide, N tile 16
    (128, 128, 16, 64, 32, 64, 2, 32, 1),     # blocks.1: stride 2, 16 -> 32
    (64, 64, 32, 64, 96, 128, 2, 32, 2),      # blocks.3: 32 -> 96 (N tiles of 32), split-K epilogue
    (32, 32, 96, 128, 256, 256, 2, 0, 1),     # blocks.5: 96 -> 256, the N tile the engine's policy picks
])
def test_igemm_silu_epilogue(cuda, h, w, cin, cin_pad, cout, pitch, stride, bn, splits):
    """SiLU applied to acc + bias, on the narrow conditioning-embedding shapes (zero weights on the padding channels).
    Catches: ReLU instead of SiLU; SiLU applied before the bias.  Columns beyond the output's own must stay untouched."""
    ops = _ops()
    x = hetero((1, h, w, cin_pad), (3,), 1, cuda, offset=1.0)
    x[..., cin:] = 0
    wt = _w((cout, cin, 3, 3), 2, cuda)
    wpad = torch.zeros((cout, cin_pad, 3, 3), dtype=torch.float16, device=cuda)
    wpad[:, :cin] = wt
    bias = (torch.randn((1, cout), generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 2).float().to(cuda)
    ho, wo = h // stride, w // stride
    g = guarded((ho * wo, cout), pitch=pitch + 8, device=cuda)
    out = g.view.view(1, ho, wo, cout)
    wp = ops.pack_conv_weight(wpad)
    kw = dict(stride=stride, colbias=bias.contiguous(), silu=True)
    if bn == 0:
        plan = ops.igemm_engine_plan([(x, 9)], wp, out, autotile=1, allow_swap=False, **kw)
        bn, splits = plan.bn, plan.splits
    ops.igemm([(x, 9)], wp, out, bn=bn, splits=splits, **kw)
    acc = _conv64(x, wpad, stride)
    pre = acc + bias.double()[0]
    ref = F.silu(pre)
    assert_discriminates(out, ref, F.relu(pre), 2e-3, 4e-3, "SiLU epilogue", bug="ReLU instead of SiLU")
    assert_discriminates(out, ref, F.silu(acc) + bias.double()[0], 2e-3, 4e-3, "SiLU epilogue", bug="SiLU before the bias")
    g.assert_untouched("igemm SiLU")


def test_tconv_refuses_the_silu_epilogue(cuda):
    """The halo-tile kernel has no SiLU epilogue (no 64 -> 64 layer of the conditioning embedding needs one, and compiling it in
    would cost the TAESD body time): asked for one, it refuses instead of silently skipping the activation."""
    from ai_rtc_agent_b200.host import capi
    ops = _ops()
    x = hetero((1, 256, 256, 64), (3,), 4, cuda)
    out = torch.empty((1, 256, 256, 64), dtype=torch.float16, device=cuda)
    with pytest.raises(capi.B2Error):
        ops.igemm([(x, 9)], ops.pack_conv_weight(_w((64, 64, 3, 3), 5, cuda)), out, silu=True, tconv=True)


def _frame_ref(frame_u8, h, w):
    """The control image as the engine sees it: nearest resize, /255, fp16-rounded (float64 NHWC)."""
    x = frame_u8.permute(0, 3, 1, 2).double()
    x = F.interpolate(x, size=(h, w), mode="nearest") / 255.0
    return x.half().double()


def test_smallconv_u8_silu_cout16(cuda):
    """The embedding's conv_in: u8 frame (nearest-resized) / 255 -> 3x3 conv 3 -> 16 -> SiLU, written 16 of 64 columns wide.
    Catches ReLU instead of SiLU; the padding columns must stay untouched."""
    ops = _ops()
    from oracle import weights as ow
    frame = ow.make_frame(96, 160, seed=7).to(cuda)
    wt = _w((16, 3, 3, 3), 8, cuda) * 4
    bias = (torch.randn(16, generator=torch.Generator().manual_seed(9)) * 0.5).float().to(cuda)
    g = guarded((128 * 128, 16), pitch=64, device=cuda)
    out = g.view.view(1, 128, 128, 16)
    ops.smallconv_ex(frame, wt, bias, out, flags=1 | 32)
    x = _frame_ref(frame.cpu(), 128, 128).to(cuda)
    pre = F.conv2d(x, wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    assert_discriminates(out, F.silu(pre), F.relu(pre), 2e-3, 4e-3, "smallconv SiLU", bug="ReLU instead of SiLU")
    g.assert_untouched("smallconv cout 16")


@pytest.mark.parametrize("broadcast", [True, False])
def test_smallconv_batch_residual(cuda, broadcast):
    """ControlNet conv_in(x) + cond over the T slots: residual batch stride 0 broadcasts the one embedding to every slot.
    Catches: the slot-0 residual added to slot 0 only (broadcast), slot 0's residual used for every slot (per-item)."""
    ops = _ops()
    T, h, w, cout = 4, 32, 32, 128
    x = hetero((T, h, w, 4), (0, 3), 10, cuda)
    wt = _w((cout, 4, 3, 3), 11, cuda)
    bias = torch.randn(cout, generator=torch.Generator().manual_seed(12)).float().to(cuda)
    res = hetero((1 if broadcast else T, h, w, cout), (0, 3), 13, cuda)
    out = torch.full((T, h, w, cout), float("nan"), dtype=torch.float16, device=cuda)
    ops.smallconv_ex(x, wt, bias, out, res=res, res_bstride=0 if broadcast else None)
    conv = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    ref = conv + res.double()
    if broadcast:
        wrong = conv.clone()
        wrong[0] += res.double()[0]
        bug = "residual added to slot 0 only"
    else:
        wrong = conv + res.double()[0:1]
        bug = "slot 0's residual for every slot"
    assert_discriminates(out, ref, wrong, 2e-3, 4e-3, "smallconv residual", bug=bug)


def test_smallconv_offset_input(cuda):
    """HED's first conv: the u8 frame on the 0..255 scale minus a per-channel offset, zero padding in the shifted domain, ReLU.
    Catches: the offset subtracted after padding (border pixels see -offset instead of 0)."""
    ops = _ops()
    from oracle import weights as ow
    frame = ow.make_frame(64, 96, seed=11).to(cuda)
    off = torch.tensor([117.0, 104.5, 96.25], device=cuda)
    wt = _w((64, 3, 3, 3), 12, cuda)
    bias = (torch.randn(64, generator=torch.Generator().manual_seed(13)) * 0.5).float().to(cuda)
    out = torch.full((1, 64, 96, 64), float("nan"), dtype=torch.float16, device=cuda)
    ops.smallconv_ex(frame, wt, bias, out, flags=1 | 4 | 64, in_off=off)
    h = (frame.permute(0, 3, 1, 2).double() - off.double().view(1, 3, 1, 1)).half().double()
    ref = F.relu(F.conv2d(h, wt.double(), bias.double(), padding=1)).permute(0, 2, 3, 1)
    padded_then_shifted = F.pad(frame.permute(0, 3, 1, 2).double(), (1, 1, 1, 1)) - off.double().view(1, 3, 1, 1)
    wrong = F.relu(F.conv2d(padded_then_shifted, wt.double(), bias.double())).permute(0, 2, 3, 1)
    assert_discriminates(out, ref, wrong, 5e-2, 4e-3, "smallconv offset input", bug="offset subtracted after padding")


def test_maxpool2x2(cuda):
    """NHWC 2x2/2 max-pool.  Catches: average pooling; the window shifted by one pixel."""
    ops = _ops()
    x = hetero((2, 32, 48, 128), (0, 3), 14, cuda)
    y = guarded((2 * 16 * 24, 128), pitch=128, device=cuda)
    ops.maxpool2x2(x, y.view.view(2, 16, 24, 128))
    xd = x.double().permute(0, 3, 1, 2)
    ref = F.max_pool2d(xd, 2, 2).permute(0, 2, 3, 1)
    avg = F.avg_pool2d(xd, 2, 2).permute(0, 2, 3, 1)
    shifted = F.max_pool2d(F.pad(xd, (0, 1, 0, 1), value=-1e9)[..., 1:, 1:], 2, 2).permute(0, 2, 3, 1)
    got = y.view.view(2, 16, 24, 128)
    assert_discriminates(got, ref, avg, 1e-3, 1e-3, "maxpool", bug="average pooling")
    assert_discriminates(got, ref, shifted, 1e-3, 1e-3, "maxpool", bug="window shifted by one")
    y.assert_untouched("maxpool")


def test_hed_projection(cuda):
    """Per-pixel C -> 1 dot product, fp32 out.  Catches: the bias left out."""
    ops = _ops()
    x = hetero((1, 32, 32, 256), (3,), 15, cuda)
    w = torch.randn(256, generator=torch.Generator().manual_seed(16)).float().to(cuda) * 0.06
    b = torch.tensor([0.75], device=cuda)
    out = torch.empty(32 * 32, dtype=torch.float32, device=cuda)
    ops.hed_project(x, w, b, out)
    dot = (x.double().reshape(-1, 256) @ w.double())
    assert_discriminates(out, dot + 0.75, dot, 1e-3, 1e-4, "hed projection", bug="bias left out")


def test_hed_fuse(cuda):
    """Side outputs -> u8 edge image: bilinear half-pixel upsampling, mean, sigmoid, * 255, truncation, 3 channels.
    Catches: align_corners=True; rounding instead of truncation."""
    ops = _ops()
    H, W = 128, 192
    g = torch.Generator().manual_seed(17)
    maps = [(torch.randn((H >> k, W >> k), generator=g) * 1.5).float().to(cuda) for k in range(5)]
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=cuda)
    edge = torch.empty((H, W), dtype=torch.float16, device=cuda)
    ops.hed_fuse(maps, out, edge)

    def fuse(align, rnd):
        ups = [F.interpolate(m.double()[None, None], size=(H, W), mode="bilinear", align_corners=align) for m in maps]
        e = torch.sigmoid(torch.stack(ups).mean(0))[0, 0] * 255.0
        return (e.round() if rnd else e.floor()).clamp(0, 255)
    ref, ac, rnd = fuse(False, False), fuse(True, False), fuse(False, True)
    got = out[..., 0].double()
    d = (got - ref).abs()
    assert d.max() <= 1 and (d == 0).float().mean() >= 0.999, (d.max().item(), (d == 0).float().mean().item())
    assert torch.equal(out[..., 0], out[..., 1]) and torch.equal(out[..., 0], out[..., 2])
    assert torch.equal(edge.double(), got)
    assert ((ac - ref).abs() > 2).float().mean() > 0.01, "align_corners=True would not be caught"
    assert ((rnd - ref) != 0).float().mean() > 0.3 and ((got - rnd) != 0).float().mean() > 0.3, "rounding would not be caught"


# ---- engine -------------------------------------------------------------------------------------------------------------------
def _cmp(got_nhwc, ref_nchw):
    got = got_nhwc.float().permute(0, 3, 1, 2)
    ref = ref_nchw.float().cpu()
    err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
    cos = F.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
    return err, cos


def _u8_check(got, ref, what):
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"
    return frac, d.max().item()


def _hed16():
    """Seeded HED weights rounded to fp16 (what the engine stores), as fp32 for both sides."""
    from ai_rtc_agent_b200.host import arch as A
    return {k: v.half().float() for k, v in A.synthetic_hed().items()}


def _engine(turbo, t_index_list, hw, cn16, full=False, graph=True, blob=None, concurrency=1, hed=None):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import unet as ounet
    from oracle import weights as ow
    if full:
        cfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
    else:
        cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    usd, vsd = ow.make_unet_weights(cfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    if blob is not None:
        sd = StreamDiffusion(arch, {}, {}, t_index_list, lambda p: emb, width=hw, height=hw, use_cuda_graph=graph,
                             packed_blob=blob, controlnet_sd={} if cn16 is not None else None,
                             hed_sd={} if hed is not None else None)
    else:
        sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, use_cuda_graph=graph,
                             controlnet_sd=cn16, hed_sd=hed)
    if concurrency > 1:
        sd.set_concurrency(concurrency)
    sd.prepare("p", guidance_scale=0.0)
    return sd, cfg, usd, vsd, emb


def _oracle(cfg, usd, vsd, cn16, emb, t_index_list, hw, init_noise, hed=None):
    from oracle import controlnet as ocn
    from oracle import weights as ow
    orc = ocn.ControlNetStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), ow.to_float(cn16), t_index_list, hw, hw,
                                     hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=init_noise.float())
    return orc


@pytest.mark.parametrize("processor", [None, "hed"])
@pytest.mark.parametrize("turbo,t_index_list", [(True, [32]), (False, [32]), (True, [18, 26, 35, 45]),
                                                (False, [18, 26, 35, 45])])
def test_tiny_controlnet_engine_matches_oracle(cuda, turbo, t_index_list, processor):
    """Both architectures, T = 1 and 4, 8 frames: every ControlNet tap and every UNet tap on the first and last frame, the u8
    frames and the x_t_latent_buffer state on every frame."""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(turbo)
    cn16 = ocn.make_weights(cfg)
    hed = _hed16() if processor == "hed" else None
    sd, cfg, usd, vsd, emb = _engine(turbo, t_index_list, 128, cn16, hed=hed)
    orc = _oracle(cfg, usd, vsd, cn16, emb, t_index_list, 128, sd.init_noise, hed=hed)
    T = len(t_index_list)
    for i in range(8):
        frame = ow.make_frame(128, 128, seed=20 + i)
        out = sd.step_u8(frame.to(cuda))
        ref = opipe.frame_to_u8(orc, frame)
        _u8_check(out, ref, f"frame {i}")
        if T > 1:
            e, c = _cmp(sd.get_tensor("unet_in")[1:], orc.x_t_latent_buffer)
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: x_t_latent_buffer relerr {e:.3e} cos {c:.6f}"
        if hed is not None:   # the u8 edge image
            _u8_check(sd.get_tensor("control").permute(0, 3, 1, 2).round().to(torch.uint8), orc.last["control"], f"control {i}")
        if i not in (0, 7):
            continue
        cn, un = orc.last["cn_taps"], orc.last["unet_taps"]
        pairs = [("cn_cond", cn["cond"]), ("cn.conv_in", cn["conv_in"]), ("cn.mid", un["cn_mid"]), ("mid", un["mid"]),
                 ("conv_in", un["conv_in"]), ("eps", orc.last["eps"]), ("x0", orc.last["x0"])]
        pairs += [(f"cn.res.{k}", un[f"res.{k}"]) for k in range(12)]
        pairs += [(n, un[n]) for n in un if n.startswith(("down.", "up."))]
        rows = []
        for name, r in pairs:
            e, c = _cmp(sd.get_tensor(name), r)
            rows.append((name, e, c))
        table = "\n".join(f"{n:12s} relerr={e:.2e} cos={c:.6f}" for n, e, c in rows)
        print(f"frame {i}\n{table}")
        for n, e, c in rows:
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: tap {n} out of tolerance\n{table}"


def test_zero_initialised_controlnet_is_bit_identical(cuda):
    """A fresh ControlNet (zero convs = 0) adds exactly nothing: frames equal those of the same engine without one, bit for bit."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    plain, *_ = _engine(False, tl, 128, None)
    cnz, *_ = _engine(False, tl, 128, ocn.make_weights(ounet.tiny_config(False), zero_init=True))
    for i in range(4):
        f = ow.make_frame(128, 128, seed=40 + i).to(cuda)
        assert torch.equal(plain.step_u8(f).cpu(), cnz.step_u8(f).cpu()), f"frame {i}"


def test_controlnet_lanes_are_bit_identical(cuda):
    """Two stage-pipelined lanes of one T=4 stream equal a single engine bit for bit; four independent T=1 lanes under the
    throughput policy equal their parent processing the same frames one after another."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    cn16 = ocn.make_weights(ounet.tiny_config(True))
    hed = _hed16()
    # a lane runs the launch policy of two frames in flight: the single engine uses the same one (same summation order)
    single, *_ = _engine(True, tl, 128, cn16, concurrency=2, hed=hed)
    owner, *_ = _engine(True, tl, 128, cn16, concurrency=2, hed=hed)
    lane = owner.add_lane(share_state=True)
    for i in range(6):
        f = ow.make_frame(128, 128, seed=60 + i).to(cuda)
        a = single.step_u8(f).cpu()
        b = (owner if i % 2 == 0 else lane).step_u8(f).cpu()
        assert torch.equal(a, b), f"stage-pipelined frame {i}"
    par, *_ = _engine(True, [32], 128, cn16, concurrency=4, hed=hed)
    lanes = [par.add_lane() for _ in range(3)]
    frames = [ow.make_frame(128, 128, seed=80 + i).to(cuda) for i in range(4)]
    outs = [eng.step_u8(f) for eng, f in zip([par] + lanes, frames)]
    torch.cuda.synchronize()
    for i, f in enumerate(frames):
        assert torch.equal(outs[i].cpu(), par.step_u8(f).cpu()), f"lane {i}"


@pytest.mark.parametrize("processor", [None, "hed"])
def test_controlnet_packed_blob_round_trip(cuda, tmp_path, processor):
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cn16 = ocn.make_weights(ounet.tiny_config(False))
    hed = _hed16() if processor == "hed" else None
    a, *_ = _engine(False, [18, 35], 128, cn16, hed=hed)
    path = str(tmp_path / "cn.b2pack")
    a.export_packed(path)
    b, *_ = _engine(False, [18, 35], 128, cn16, blob=path, hed=hed)
    for i in range(3):
        f = ow.make_frame(128, 128, seed=90 + i).to(cuda)
        assert torch.equal(a.step_u8(f).cpu(), b.step_u8(f).cpu()), f"frame {i}"
    from ai_rtc_agent_b200.host import capi
    with pytest.raises(capi.B2Error):   # a blob with a ControlNet does not load into an engine without one
        _engine(False, [18, 35], 128, None, blob=path)


def test_fullsize_sd15_controlnet_hed_512(cuda):
    """SD-1.5 + ControlNet + HED at 512x512, T=4, 3 frames, against the fp32 oracle run by torch on the GPU."""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import unet as ounet
    from oracle import weights as ow
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    tl = [18, 26, 35, 45]
    cn16 = ocn.make_weights(ounet.SD15)
    hed = _hed16()
    sd, cfg, usd, vsd, emb = _engine(False, tl, 512, cn16, full=True, hed=hed)
    orc = _oracle(cfg, usd, vsd, cn16, emb, tl, 512, sd.init_noise, hed=hed).to(cuda)
    for i in range(3):
        frame = ow.make_frame(512, 512, seed=i)
        out = sd.step_u8(frame.to(cuda))
        with torch.no_grad():
            ref = opipe.frame_to_u8(orc, frame.to(cuda))
        un, cn = orc.last["unet_taps"], orc.last["cn_taps"]
        rows = [(n, *_cmp(sd.get_tensor(n), r)) for n, r in [("cn_cond", cn["cond"]), ("cn.conv_in", cn["conv_in"]),
                                                             ("cn.res.0", un["res.0"]), ("cn.res.11", un["res.11"]),
                                                             ("cn.mid", un["cn_mid"]), ("eps", orc.last["eps"])]]
        frac, mx = _u8_check(out, ref, f"frame {i}")
        cf, cm = _u8_check(sd.get_tensor("control").permute(0, 3, 1, 2).round().to(torch.uint8), orc.last["control"], f"control {i}")
        print(f"frame {i}: HED edge image frac(|d|<=2) {cf:.5f} max {cm}")
        print(f"frame {i}: u8 frac(|d|<=2) {frac:.5f} max {mx}\n" +
              "\n".join(f"  {n:10s} relerr={e:.2e} cos={c:.6f}" for n, e, c in rows))
        for n, e, c in rows:
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: {n} relerr {e:.2e} cos {c:.6f}"
