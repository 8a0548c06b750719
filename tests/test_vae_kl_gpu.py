"""The model's own AutoencoderKL (use_tiny_vae=False) on the H100: its two new kernel variants and GroupNorm at its shapes against
float64 references, the engine against the fp32 oracle (oracle/autoencoder_kl.py) on identical seeded weights, and the
bit-exactness of lanes and packed blobs.

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


# ---- single-head attention, head dim 512 --------------------------------------------------------------------------------------
def _attn512(q, k, v, scale):
    s = (q.double() @ k.double().T) * scale
    return torch.softmax(s, dim=-1) @ v.double()


@pytest.mark.parametrize("tokens", [64, 2400, 2411, 4096, 4608, 9216])
def test_attention_d512(cuda, tokens):
    """softmax(Q K^T / sqrt(512)) V for one 512-wide head, the AutoencoderKL mid-block attention (4096 tokens at 512x512, 9216 at
    768x768; 2400 is not a multiple of the 128-row query tile, 2411 not one of the 32-key block either).  The rows after the
    last key hold large keys and values, which must be masked.  Catches: the scale of a 128-column slice (1/sqrt(128)); every
    column slice computed with slice 0's V^T; keys past skv not masked (2411 only: elsewhere no key block is partial).  Two runs
    are bit-identical."""
    ops = _ops()
    C, extra = 512, 40
    rows = tokens + extra
    q = hetero((tokens, C), (1,), 1, cuda, offset=0.3, scale=(0.3, 1.5))
    k = hetero((rows, C), (1,), 2, cuda, offset=0.3, scale=(0.3, 1.5))
    v = hetero((rows, C), (1,), 3, cuda, offset=0.3, scale=(0.3, 1.5))
    k[tokens:] = 8.0                              # past skv: keys that would dominate the softmax ...
    v[tokens:] = 30.0                             # ... and values that would show
    vt_ld = (rows + 7) // 8 * 8
    vt = torch.zeros((C, vt_ld), dtype=torch.float16, device=cuda)
    vt[:, :rows] = v.T
    g = guarded((tokens, C), pitch=C + 8, device=cuda)
    kw = dict(nb=1, heads=1, sq=tokens, skv=tokens, d_real=C, dp=C, k_bstride=0, vt_bstride=0)
    ops.attention(q, k, vt, g.view, **kw)
    torch.cuda.synchronize()
    first = g.view.clone()
    ops.attention(q, k, vt, g.view, **kw)
    assert torch.equal(first.view(torch.int16), g.view.view(torch.int16)), "two runs differ"
    g.assert_untouched("attention d512")
    ref = _attn512(q, k[:tokens], v[:tokens], 1 / math.sqrt(C))
    tol = (2e-3, 1e-2)
    what = f"attention d512 tokens={tokens}"
    assert_discriminates(g.view, ref, _attn512(q, k[:tokens], v[:tokens], 1 / math.sqrt(128)), *tol, what, "scale 1/sqrt(128)")
    v0 = v[:tokens, :128].repeat(1, 4)
    assert_discriminates(g.view, ref, _attn512(q, k[:tokens], v0, 1 / math.sqrt(C)), *tol, what, "slice 0's V^T for every slice")
    if tokens % 32:
        end = (tokens + 31) // 32 * 32
        assert_discriminates(g.view, ref, _attn512(q, k[:end], v[:end], 1 / math.sqrt(C)), *tol, what, "keys past skv not masked")


# ---- stride-2 conv with the zero padding after the last row / column (Downsample2D(padding=0)) ----------------------------------
def _w(shape, seed, device):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) / math.sqrt(math.prod(shape[1:]))).half().to(device)


@pytest.mark.parametrize("h,w,c", [(512, 512, 128), (256, 256, 256), (128, 128, 512), (384, 512, 128), (448, 768, 128),
                                   (224, 384, 256)])
def test_igemm_pad0_stride2(cuda, h, w, c):
    """F.conv2d(F.pad(x, (0, 1, 0, 1)), W, b, stride=2) with the plan the engine's tile policy picks, at the VAE encoder's three
    downsampler levels of 512x512 and at non-square levels.  Catches: the UNet downsampler's symmetric padding of 1."""
    ops = _ops()
    x = hetero((1, h, w, c), (3,), 3, cuda, offset=1.0)
    wt = _w((c, c, 3, 3), 4, cuda)
    bias = (0.3 * torch.randn((1, c), generator=torch.Generator().manual_seed(5), dtype=torch.float64)).float().to(cuda)
    ho, wo = h // 2, w // 2
    g = guarded((ho * wo, c), device=cuda)
    out = g.view.view(1, ho, wo, c)
    wp = ops.pack_conv_weight(wt)
    plan = ops.igemm_engine_plan([(x, 9)], wp, out, autotile=1, allow_swap=False, stride=2, colbias=bias, pad0=True)
    assert plan.mode == 0 and plan.swap == 0 and plan.bn in (64, 128, 256)
    ops.igemm([(x, 9)], wp, out, stride=2, colbias=bias, pad0=True, bn=plan.bn, splits=plan.splits)
    xd = x.double().permute(0, 3, 1, 2)
    ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wt.double(), bias.double()[0], stride=2).permute(0, 2, 3, 1)
    wrong = F.conv2d(xd, wt.double(), bias.double()[0], stride=2, padding=1).permute(0, 2, 3, 1)
    print(f"pad0 {h}x{w}x{c}: bn={plan.bn} splits={plan.splits}")
    assert_discriminates(out, ref, wrong, 2e-3, 4e-3, f"pad0 conv {h}x{w}x{c}", "symmetric padding of 1")
    g.assert_untouched("pad0 conv")


def test_igemm_pad0_refuses_pairs_and_swap(cuda):
    from ai_rtc_agent_b200.host import capi
    ops = _ops()
    x = torch.zeros((1, 64, 64, 128), dtype=torch.float16, device=cuda)
    wp = ops.pack_conv_weight(torch.zeros((128, 128, 3, 3), dtype=torch.float16, device=cuda))
    out = torch.empty((1, 32, 32, 128), dtype=torch.float16, device=cuda)
    for kw in (dict(pair=True, bn=128), dict(swap=True, bn=128), dict(bn=32)):
        with pytest.raises(capi.B2Error):
            ops.igemm([(x, 9)], wp, out, stride=2, pad0=True, **kw)
    plan = ops.igemm_engine_plan([(x, 9)], wp, out, autotile=2, allow_swap=True, stride=2, pad0=True)
    assert plan.mode == 0 and plan.swap == 0, "the throughput policy must keep tap-origin-0 contractions on single CTAs"


# ---- GroupNorm at the VAE's shapes ---------------------------------------------------------------------------------------------
def _gn_ref(x, gamma, beta, eps, silu, shift=0):
    nb, h, w, c = x.shape
    xg = x.double().reshape(nb, h * w, 32, c // 32)
    mean, var = xg.mean(dim=(1, 3)), xg.var(dim=(1, 3), unbiased=False)
    mean, var = mean.roll(shift, 1), var.roll(shift, 1)
    grp = torch.arange(c, device=x.device) // (c // 32)
    y = (x.double() - mean[:, grp][:, None, None]) * (var[:, grp] + eps).rsqrt()[:, None, None] * gamma.double() + beta.double()
    return F.silu(y) if silu else y


@pytest.mark.parametrize("h,w,c", [(512, 512, 128), (256, 256, 256), (128, 128, 512)])
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_vae_shapes(cuda, h, w, c, silu):
    """GroupNorm(32, eps 1e-6) with 4 / 8 / 16 channels per group at the AutoencoderKL's largest level of each width (groups too
    large for the cluster path).  Logs the path and its device time.  Group 5 is shrunk 1000x so that eps matters (its mean stays
    within 100 standard deviations, the kernels' operating range).
    Catches: eps 1e-5 (the UNet's); the neighbouring group's statistics."""
    ops = _ops()
    x = hetero((1, h, w, c), (3,), 7, cuda, offset=2.0)
    cpg = c // 32
    x[..., 5 * cpg:6 * cpg] = (x[..., 5 * cpg:6 * cpg].float() * 1e-3).half()
    gamma = (1 + 0.2 * torch.randn(c, generator=torch.Generator().manual_seed(8))).float().to(cuda)
    beta = (0.2 * torch.randn(c, generator=torch.Generator().manual_seed(9))).float().to(cuda)
    y = torch.full((1, h, w, c), float("nan"), dtype=torch.float16, device=cuda)
    _, path = ops.groupnorm(x, None, gamma, beta, y, eps=1e-6, silu=silu, return_path=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ops.groupnorm(x, None, gamma, beta, y, eps=1e-6, silu=silu)
    e1.record()
    torch.cuda.synchronize()
    print(f"groupnorm {h}x{w}x{c} ({cpg} channels/group): path={path} {e0.elapsed_time(e1) / 20 * 1e3:.1f} us "
          f"on {torch.cuda.get_device_name()}")
    ref = _gn_ref(x, gamma, beta, 1e-6, silu)
    what = f"groupnorm[{path}] {h}x{w}x{c}"
    assert_discriminates(y, ref, _gn_ref(x, gamma, beta, 1e-5, silu), 3e-3, 2e-3, what, "eps 1e-5")
    assert_discriminates(y, ref, _gn_ref(x, gamma, beta, 1e-6, silu, shift=1), 3e-3, 2e-3, what, "statistics of group g-1")


# ---- engine ---------------------------------------------------------------------------------------------------------------------
def _cmp(got_nhwc, ref_nchw):
    got = got_nhwc.double().permute(0, 3, 1, 2)
    ref = ref_nchw.double().cpu()
    err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
    cos = F.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
    return err, cos


def _u8_check(got, ref, what):
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"
    return frac, d.max().item()


def _engine(turbo, t_index_list, hw, full=False, graph=True, blob=None, concurrency=1, cn16=None, tiny_vae=False):
    """hw: an int for a square engine or (height, width)"""
    height, width = (hw, hw) if isinstance(hw, int) else hw
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import unet as ounet
    from oracle import weights as ow
    if full:
        cfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
        varch = A.AUTOENCODER_KL
    else:
        cfg, arch, varch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15), A.TINY_AUTOENCODER_KL
    usd = ow.make_unet_weights(cfg)
    vsd = ow.make_taesd_weights() if tiny_vae else A.synthetic_autoencoder_kl(varch)
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    kw = dict(width=width, height=height, use_cuda_graph=graph, use_tiny_vae=tiny_vae,
              controlnet_sd=None if cn16 is None else ({} if blob else cn16))
    if blob is not None:
        sd = StreamDiffusion(arch, {}, {}, t_index_list, lambda p: emb, packed_blob=blob, **kw)
    else:
        sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, **kw)
    if concurrency > 1:
        sd.set_concurrency(concurrency)
    sd.prepare("p", guidance_scale=0.0)
    return sd, cfg, usd, vsd, emb


def _oracle(cfg, usd, vsd, emb, t_index_list, hw, init_noise, full=False, cn16=None):
    from oracle import autoencoder_kl as oakl
    from oracle import stream_kl as oskl
    from oracle import weights as ow
    height, width = (hw, hw) if isinstance(hw, int) else hw
    kl = oakl.FULL if full else oakl.TINY
    if cn16 is not None:
        orc = oskl.KLControlNetStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), ow.to_float(cn16), t_index_list, width,
                                            height, vae_kl=kl)
    else:
        orc = oskl.KLStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), t_index_list, width, height, vae_kl=kl)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=init_noise.float())
    return orc


VAE_TAPS = [f"vae.enc.down.{i}" for i in range(4)] + ["vae.enc.mid", "vae.dec.mid"] + [f"vae.dec.up.{i}" for i in range(4)]


def _check_taps(sd, orc, what):
    rows = [(n, *_cmp(sd.get_tensor(n), orc.last[n])) for n in VAE_TAPS]
    rows += [(n, *_cmp(sd.get_tensor(n), orc.last[n])) for n in ("x_t", "x0")]
    rows.append(("image", *_cmp(sd.get_tensor("image"), (orc.last["image"] + 1) / 2)))   # the engine keeps it on the [0, 1] scale
    table = "\n".join(f"{n:16s} relerr={e:.2e} cos={c:.6f}" for n, e, c in rows)
    print(f"{what}\n{table}")
    for n, e, c in rows:
        assert e <= 2e-2 and c >= 0.999, f"{what}: tap {n} out of tolerance\n{table}"


@pytest.mark.parametrize("turbo,t_index_list,hw", [
    (True, [32], 128), (False, [32], 128), (True, [18, 26, 35, 45], 128), (False, [18, 26, 35, 45], 128),
    (True, [32], (192, 128)), (False, [18, 26, 35, 45], (192, 128)),
])
def test_tiny_kl_engine_matches_oracle(cuda, turbo, t_index_list, hw):
    """Both architectures, T = 1 and 4, square and non-square, 8 frames: every VAE tap, x_t, x0 and the image on the first and
    last frame, the u8 frames and the x_t_latent_buffer on every frame.  The synthetic quant_conv / post_quant_conv biases are
    nonzero, so a bias folded across a zero-padded conv fails on the border pixels."""
    from oracle import pipeline as opipe
    from oracle import weights as ow
    sd, cfg, usd, vsd, emb = _engine(turbo, t_index_list, hw)
    orc = _oracle(cfg, usd, vsd, emb, t_index_list, hw, sd.init_noise)
    for i in range(8):
        frame = ow.make_frame(orc.height, orc.width, seed=120 + i)
        out = sd.step_u8(frame.to(cuda))
        ref = opipe.frame_to_u8(orc, frame)
        if i in (0, 7):
            _check_taps(sd, orc, f"frame {i}")
        _u8_check(out, ref, f"frame {i}")
        if len(t_index_list) > 1:
            e, c = _cmp(sd.get_tensor("unet_in")[1:], orc.x_t_latent_buffer)
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: x_t_latent_buffer relerr {e:.3e} cos {c:.6f}"


def test_tiny_kl_engine_with_controlnet(cuda):
    """A ControlNet (processor None: the frame itself) next to the AutoencoderKL: both read the caller's frame."""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import unet as ounet
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    cn16 = ocn.make_weights(ounet.tiny_config(False))
    sd, cfg, usd, vsd, emb = _engine(False, tl, 128, cn16=cn16)
    orc = _oracle(cfg, usd, vsd, emb, tl, 128, sd.init_noise, cn16=cn16)
    for i in range(4):
        frame = ow.make_frame(128, 128, seed=140 + i)
        _u8_check(sd.step_u8(frame.to(cuda)), opipe.frame_to_u8(orc, frame), f"frame {i}")
    _check_taps(sd, orc, "controlnet frame 3")


def test_kl_float_entries_match_u8(cuda):
    """The f32 and f16 NCHW entries apply the same 2x - 1 (offset input mode) as the u8 entry: same frame, same output."""
    from oracle import weights as ow
    sd, *_ = _engine(True, [32], 128)
    frame = ow.make_frame(128, 128, seed=150).to(cuda)
    u8 = sd.step_u8(frame).cpu()
    x = frame.permute(0, 3, 1, 2).float() / 255.0
    for t in (x, x.half()):
        img = sd(t)
        got = ((img.float() / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8).cpu()
        assert (got.int() - u8.int()).abs().max().item() <= 1, f"{t.dtype} entry"


def test_kl_lanes_stepping_one_state_are_bit_identical(cuda):
    """One T=4 stream state stepped alternately on two lanes (stage-pipelined) equals a single engine bit for bit; eight
    independent T=1 lanes under the throughput policy equal their parent processing the same frames one after another."""
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    single, *_ = _engine(True, tl, 128, concurrency=2)
    owner, *_ = _engine(True, tl, 128, concurrency=2)
    lane = owner.add_lane()
    state = owner.new_state()
    for i in range(6):
        f = ow.make_frame(128, 128, seed=160 + i).to(cuda)
        got = (owner if i % 2 == 0 else lane).step_u8(f, state=state).cpu()
        assert torch.equal(single.step_u8(f).cpu(), got), f"stage-pipelined frame {i}"
    par, *_ = _engine(True, [32], 128, concurrency=8)
    lanes = [par.add_lane() for _ in range(7)]
    frames = [ow.make_frame(128, 128, seed=170 + i).to(cuda) for i in range(8)]
    outs = [eng.step_u8(f) for eng, f in zip([par] + lanes, frames)]
    torch.cuda.synchronize()
    for i, f in enumerate(frames):
        assert torch.equal(outs[i].cpu(), par.step_u8(f).cpu()), f"lane {i}"


def test_kl_packed_blob_round_trip(cuda, tmp_path):
    """A KL blob reproduces its engine bit for bit, and is refused by a TAESD engine (and a TAESD blob by a KL engine)."""
    from ai_rtc_agent_b200.host import capi
    from oracle import weights as ow
    a, *_ = _engine(False, [18, 35], 128)
    path = str(tmp_path / "kl.b2pack")
    a.export_packed(path)
    b, *_ = _engine(False, [18, 35], 128, blob=path)
    for i in range(3):
        f = ow.make_frame(128, 128, seed=180 + i).to(cuda)
        assert torch.equal(a.step_u8(f).cpu(), b.step_u8(f).cpu()), f"frame {i}"
    with pytest.raises(capi.B2Error):
        _engine(False, [18, 35], 128, blob=path, tiny_vae=True)
    t, *_ = _engine(False, [18, 35], 128, tiny_vae=True)
    tpath = str(tmp_path / "taesd.b2pack")
    t.export_packed(tpath)
    with pytest.raises(capi.B2Error):
        _engine(False, [18, 35], 128, blob=tpath)


# ---- full size: engine, fp32 torch oracle on the GPU, fp16 torch ------------------------------------------------------------------
@pytest.mark.parametrize("turbo,t_index_list,hw", [
    (False, [18, 26, 35, 45], 512), (True, [32], 768), (True, [32], (448, 768)),
])
def test_fullsize_kl_three_implementations(cuda, turbo, t_index_list, hw):
    """SD-1.5 + LCM T=4 at 512x512, SD-Turbo T=1 at 768x768 (9216-token attention) and at 448x768, 2 frames: the engine and a
    plain fp16 torch run of the same restatement against the fp32 oracle on the GPU."""
    from oracle import autoencoder_kl as oakl
    from oracle import pipeline as opipe
    from oracle import stream_kl as oskl
    from oracle import torch_gpu
    from oracle import weights as ow
    height, width = (hw, hw) if isinstance(hw, int) else hw
    sd, cfg, usd, vsd, emb = _engine(turbo, t_index_list, hw, full=True)
    mk = lambda dt: oskl.build(cfg, usd, vsd, t_index_list, height, emb, sd.init_noise, dtype=dt, width=width, vae_kl=oakl.FULL)
    o32, o16 = mk(torch.float32), mk(torch.float16)
    for i in range(2):
        frame = ow.make_frame(height, width, seed=190 + i)
        out = sd.step_u8(frame.to(cuda))
        with torch.no_grad():
            r32 = opipe.frame_to_u8(o32, frame.to(cuda))
            with torch_gpu.fused_attention():
                r16 = opipe.frame_to_u8(o16, frame.to(cuda))
        f_e, m_e = _u8_check(out, r32, f"engine frame {i}")
        f_t, m_t = _u8_check(r16, r32, f"fp16 torch frame {i}")
        print(f"frame {i}: engine frac {f_e:.5f} max {m_e}; fp16 torch frac {f_t:.5f} max {m_t}")
        _check_taps(sd, o32, f"full size frame {i}")
