"""The optional branches of the frame program -- AutoencoderKL, ControlNet, HED -- at the regimes tests/test_config_space_branches.py
finds in the accepted configuration space (sides 64 .. 1024, stream batch 1 .. 16), on the H100.

Operator cases: each kernel against a float64 reference of the same operation, with guard bands around the outputs and named
wrong alternatives that the reference must reject by >= 10x the tolerance (the margin is printed).  Engine configurations
(SWEEP_BRANCHES): each launch-audited (tests/test_launch_audit_gpu.py) with the regimes it records checked against the CPU
model's prediction, then run for T + 2 frames through the stream loop against the fp32 oracle on the GPU: the u8 image within
2 LSB and, for T > 1, the stream-batch latent buffer, as tests/test_config_space_gpu.py does for the UNet."""
from __future__ import annotations

import math
import time

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_discriminates, guarded, hetero

pytestmark = pytest.mark.gpu

# ---- the lists the CPU model checks (tests/test_config_space_branches.py) ---------------------------------------------------
D512_TOKENS = [64, 192, 320, 12288, 14400, 15360, 16384]   # 64 x 64, 64 x 192, 64 x 320, 1024 x 768, 960 x 960, 1024 x 960, 1024^2
# stride-2 pad0 conv inputs (h, w, c): the encoder levels of 64 x 64, 64 x 192, 192 x 64, 960 x 704 and 1024 x 960 frames
PAD0_CASES = [(64, 64, 128), (32, 32, 256), (16, 16, 512), (16, 48, 512), (48, 16, 512), (240, 176, 512), (256, 240, 512),
              (1024, 1024, 128)]
# GroupNorm (h, w, c) at the AutoencoderKL's levels: 4 / 8 / 16 channels per group, each cluster size and the non-cluster kernels
GN_CASES = [(8, 8, 512), (32, 32, 128), (16, 16, 256), (32, 32, 512), (64, 64, 128), (32, 64, 256), (32, 64, 512), (64, 128, 128),
            (64, 64, 256), (56, 72, 512), (64, 256, 128), (64, 128, 256), (88, 88, 512), (112, 144, 256), (256, 240, 512),
            (512, 480, 256), (1024, 1024, 128)]
HED_CASES = [(64, 64), (64, 192), (1024, 1024), (1024, 960)]        # frames: max-pool chain and hed_fuse
EMBEDDING_CASES = [(64, 64), (64, 192), (192, 64), (960, 704), (1024, 960)]   # frames: the conditioning embedding's SiLU convs
COND_RES_BATCHES = [1, 3, 4]


def _entry(turbo, t, hw, kl=False, cn=False, hed=False):
    tl = [32] if t == 1 else [int(10 + 35 * i / (t - 1)) for i in range(t)]
    size = str(hw) if isinstance(hw, int) else f"{hw[0]}x{hw[1]}"
    name = f"{'turbo' if turbo else 'sd15'}-T{t}-{size}" + "".join(f"-{k}" for k, on in (("kl", kl), ("cn", cn), ("hed", hed)) if on)
    return pytest.param(dict(turbo=turbo, tl=tl, hw=hw, kl=kl, cn=cn, hed=hed), id=name)


# Chosen by tests/test_config_space_branches.py (each reaches a regime no other engine configuration reaches); full-size models
# (the AutoencoderKL's 128 / 256 / 512 channels, the ControlNet's 320 .. 1280).
SWEEP_BRANCHES = [
    _entry(True, 2, 64, kl=True, cn=True, hed=True),            # 64-token d512 (one partial query tile); 4-pixel HED maps
    _entry(False, 3, (64, 192), kl=True, cn=True, hed=True),    # odd stream batch under one conditioning image; 192 tokens
    _entry(True, 1, (192, 64), kl=True, cn=True, hed=True),     # Wo-wide tiles with a partial last row tile (pad0, SiLU)
    _entry(True, 1, (1024, 960), kl=True, cn=True, hed=True),   # 15360-token d512; 8-wide tiles; GroupNorm chunks of 7680 px
    _entry(True, 1, (960, 704), kl=True, cn=True, hed=True),    # 10560 tokens: long and a half query tile; 8-wide partial tiles
]


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _discriminates(got, ref, wrong, tol_abs, tol_rel, what, bug):
    assert_discriminates(got, ref, wrong, tol_abs, tol_rel, what, bug)
    wrong, ref = wrong.double().to(got.device), ref.double().to(got.device)
    margin = ((wrong - ref).abs() / (tol_abs + tol_rel * ref.abs())).nan_to_num(nan=float("inf")).max().item()
    print(f"  {what}: '{bug}' rejected by {margin:.3g}x the tolerance")


def _w(shape, seed, device):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) / math.sqrt(math.prod(shape[1:]))).half().to(device)


# ---- attn_d512_kernel at the engine's token counts ----------------------------------------------------------------------------
def _attn512(q, k, v, nk=None, chunk=2048):
    """softmax(Q K[:nk]^T / sqrt(512)) V[:nk] in float64, over chunks of query rows (a 16384^2 score matrix is 2 GiB)"""
    nk = k.shape[0] if nk is None else nk
    kd, vd = k[:nk].double(), v[:nk].double()
    out = torch.empty((q.shape[0], v.shape[1]), dtype=torch.float64, device=q.device)
    for r in range(0, q.shape[0], chunk):
        s = (q[r:r + chunk].double() @ kd.T) / math.sqrt(512)
        out[r:r + chunk] = torch.softmax(s, dim=-1) @ vd
    return out


@pytest.mark.parametrize("sq", D512_TOKENS)
def test_attention_d512_engine_lengths(cuda, sq):
    """The AutoencoderKL mid-block attention at the token counts of 64 x 64 (one 64-row query tile), 64 x 192 / 64 x 320 (a
    64-row query tail) and 768 .. 1024 px frames (up to 16384 tokens).  The last 32-key block within skv is made to matter
    (large keys along one channel, shifted values), the rows past skv hold keys and values that would dominate if unmasked.
    Catches: the last query tile's rows not written; the last key block dropped."""
    ops = _ops()
    C, extra = 512, 64
    rows = sq + extra
    q = hetero((sq, C), (1,), 21, cuda, offset=0.3, scale=(0.3, 1.5))
    k = hetero((rows, C), (1,), 22, cuda, offset=0.3, scale=(0.3, 1.5))
    v = hetero((rows, C), (1,), 23, cuda, offset=0.3, scale=(0.3, 1.5))
    q[:, 0] = (2.0 + 0.2 * torch.randn(sq, generator=torch.Generator().manual_seed(24))).half().to(cuda)
    k[sq - 32:sq, 0] = 48.0
    v[sq - 32:sq] = (v[sq - 32:sq].float() + 3.0).half()
    k[sq:] = 8.0
    v[sq:] = 30.0
    vt_ld = (rows + 7) // 8 * 8
    vt = torch.zeros((C, vt_ld), dtype=torch.float16, device=cuda)
    vt[:, :rows] = v.T
    g = guarded((sq, C), pitch=C + 8, device=cuda)
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    ops.attention(q, k, vt, g.view, nb=1, heads=1, sq=sq, skv=sq, d_real=C, dp=C, k_bstride=0, vt_bstride=0)
    t1.record()
    torch.cuda.synchronize()
    g.assert_untouched(f"attention d512 sq={sq}")
    ref = _attn512(q, k, v, sq)
    tail = sq - (sq - 1) // 128 * 128
    dropped = ref.clone()
    dropped[sq - tail:] = 0
    what = f"attention d512 sq={sq} ({t0.elapsed_time(t1) * 1e3:.0f} us incl. first launch, {torch.cuda.get_device_name()})"
    tol = (2e-3, 1e-2)
    _discriminates(g.view, ref, dropped, *tol, what, f"last query tile's {tail} rows not written")
    _discriminates(g.view, ref, _attn512(q, k, v, sq - 32), *tol, what, "last key block dropped")


# ---- igemm_pad0_kernel ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,c", PAD0_CASES)
def test_igemm_pad0_levels(cuda, h, w, c):
    """F.conv2d(F.pad(x, (0, 1, 0, 1)), W, b, stride=2) with the engine's plan, at the encoder levels of the smallest frames and of
    1024-px frames.  Catches: the padding on the leading edge (F.pad(x, (1, 0, 1, 0))); the UNet's symmetric padding."""
    ops = _ops()
    x = hetero((1, h, w, c), (3,), 31, cuda, offset=1.0)
    wt = _w((c, c, 3, 3), 32, cuda)
    bias = (0.3 * torch.randn((1, c), generator=torch.Generator().manual_seed(33), dtype=torch.float64)).float().to(cuda)
    ho, wo = h // 2, w // 2
    g = guarded((ho * wo, c), pitch=c + 8, device=cuda)
    out = g.view.view(1, ho, wo, c)
    wp = ops.pack_conv_weight(wt)
    plan = ops.igemm_engine_plan([(x, 9)], wp, out, autotile=1, allow_swap=True, stride=2, colbias=bias, pad0=True)
    ops.igemm([(x, 9)], wp, out, stride=2, colbias=bias, pad0=True, bn=plan.bn, splits=plan.splits)
    torch.cuda.synchronize()
    g.assert_untouched(f"pad0 {h}x{w}x{c}")
    xd = x.double().permute(0, 3, 1, 2)
    wd, bd = wt.double(), bias.double()[0]
    ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wd, bd, stride=2).permute(0, 2, 3, 1)
    what = f"pad0 conv {h}x{w}x{c} (bn {plan.bn}, splits {plan.splits}, tile {plan.tw}x{plan.th}x{plan.tn})"
    _discriminates(out, ref, F.conv2d(F.pad(xd, (1, 0, 1, 0)), wd, bd, stride=2).permute(0, 2, 3, 1), 2e-3, 4e-3, what,
                   "padding on the leading edge")
    _discriminates(out, ref, F.conv2d(xd, wd, bd, stride=2, padding=1).permute(0, 2, 3, 1), 2e-3, 4e-3, what,
                   "symmetric padding of 1")


# ---- GroupNorm with 4 / 8 / 16 channels per group ------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,c", GN_CASES)
def test_groupnorm_kl_regimes(cuda, h, w, c):
    """GroupNorm(32, eps 1e-6) + SiLU at the AutoencoderKL's levels, on every path the planner picks for 4 / 8 / 16 channels per
    group (cluster of 1 / 2 / 4 / 8 CTAs, the non-cluster kernels, chunks of up to 8192 pixels).  The path that ran is the one the
    CPU model predicts.  Group 5 is shrunk 1000x so that eps matters.  Catches: the neighbouring group's statistics; a channel
    put into the neighbouring group; eps 1e-5."""
    from tests import test_config_space_branches as B
    ops = _ops()
    x = hetero((1, h, w, c), (3,), 41, cuda, offset=2.0)
    cpg = c // 32
    x[..., 5 * cpg:6 * cpg] = (x[..., 5 * cpg:6 * cpg].float() * 1e-3).half()
    gamma = (1 + 0.2 * torch.randn(c, generator=torch.Generator().manual_seed(42))).float().to(cuda)
    beta = (0.2 * torch.randn(c, generator=torch.Generator().manual_seed(43))).float().to(cuda)
    g = guarded((h * w, c), pitch=c + 8, device=cuda)
    y = g.view.view(1, h, w, c)
    _, path = ops.groupnorm(x, None, gamma, beta, y, eps=1e-6, silu=True, return_path=True)
    torch.cuda.synchronize()
    g.assert_untouched(f"groupnorm {h}x{w}x{c}")
    regime = B.gn_regime(c, h * w)
    print(f"groupnorm {h}x{w}x{c}: {regime}, path {path}")
    if regime.startswith("gn:cl0"):
        assert path in ("fused", "stats+apply"), (regime, path)
        if regime.endswith("+long-chunk"):
            assert path == "stats+apply", (regime, path)
    else:
        assert path == "cluster", (regime, path)
    xd = x.double().reshape(1, h * w, 32, cpg)
    mean, var = xd.mean(dim=(1, 3)), xd.var(dim=(1, 3), unbiased=False)

    def apply(m, vv, eps=1e-6, grp=None):
        grp = torch.arange(c, device=cuda) // cpg if grp is None else grp
        return F.silu((x.double() - m[:, grp][:, None, None]) * (vv[:, grp] + eps).rsqrt()[:, None, None] * gamma.double()
                      + beta.double())
    ref = apply(mean, var)
    what = f"groupnorm[{path}] {h}x{w}x{c}"
    tol = (3e-3, 2e-3)
    _discriminates(y, ref, apply(mean.roll(1, 1), var.roll(1, 1)), *tol, what, "statistics of group g-1")
    _discriminates(y, ref, apply(mean, var, grp=((torch.arange(c, device=cuda) + 1) // cpg).clamp(max=31)), *tol, what,
                   "group boundary shifted by one channel")
    _discriminates(y, ref, apply(mean, var, eps=1e-5), *tol, what, "eps 1e-5")


# ---- HED: the max-pool chain and hed_fuse ------------------------------------------------------------------------------------
@pytest.mark.parametrize("height,width", HED_CASES)
def test_hed_pools_and_fuse(cuda, height, width):
    """HED's four max-pools at a frame's levels (64 .. 512 channels; a 64-px frame ends in 4 x 4 maps), then hed_fuse from five
    maps of H/1 .. H/16 (ratios 1 .. 16, different vertically and horizontally on non-square frames; above 540672 pixels the
    grid-stride loop iterates).  Max-pool: bit-exact; catches average pooling and the window shifted by one.  hed_fuse: within 1
    (fp32 vs float64 at truncation boundaries); catches align_corners=True and rounding instead of truncation."""
    from oracle import hed as ohed
    ops = _ops()
    what = f"hed {height}x{width}"
    for k in range(len(ohed.BLOCKS) - 1):
        h, w, c = height >> k, width >> k, ohed.BLOCKS[k][1]
        x = hetero((1, h, w, c), (3,), 50 + k, cuda)
        g = guarded(((h // 2) * (w // 2), c), device=cuda)   # dense output: guard rows before and after
        y = g.view.view(1, h // 2, w // 2, c)
        ops.maxpool2x2(x, y)
        torch.cuda.synchronize()
        g.assert_untouched(f"maxpool {h}x{w}x{c}")
        xd = x.double().permute(0, 3, 1, 2)
        ref = F.max_pool2d(xd, 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(y.double(), ref), f"{what}: max-pool of level {k} ({h}x{w}x{c}) is not exact"
        _discriminates(y, ref, F.avg_pool2d(xd, 2, 2).permute(0, 2, 3, 1), 1e-3, 1e-3, f"maxpool {h}x{w}x{c}", "average pooling")
        shifted = F.max_pool2d(F.pad(xd, (0, 1, 0, 1), value=-1e9)[..., 1:, 1:], 2, 2).permute(0, 2, 3, 1)
        _discriminates(y, ref, shifted, 1e-3, 1e-3, f"maxpool {h}x{w}x{c}", "window shifted by one")
    gen = torch.Generator().manual_seed(55)
    maps = [(torch.randn((height >> k, width >> k), generator=gen) * 1.5).float().to(cuda) for k in range(5)]
    out = torch.empty((height, width, 3), dtype=torch.uint8, device=cuda)
    edge = torch.empty((height, width), dtype=torch.float16, device=cuda)
    ops.hed_fuse(maps, out, edge)

    def fuse(align, rnd):
        ups = [F.interpolate(m.double()[None, None], size=(height, width), mode="bilinear", align_corners=align) for m in maps]
        e = torch.sigmoid(torch.stack(ups).mean(0))[0, 0] * 255.0
        return (e.round() if rnd else e.floor()).clamp(0, 255)
    ref = fuse(False, False)
    got = out[..., 0].double()
    d = (got - ref).abs()
    assert d.max() <= 1 and (d == 0).float().mean() >= 0.999, (what, d.max().item(), (d == 0).float().mean().item())
    assert torch.equal(out[..., 0], out[..., 1]) and torch.equal(out[..., 0], out[..., 2]) and torch.equal(edge.double(), got)
    for bug, wrong in (("align_corners=True", fuse(True, False)), ("rounding instead of truncation", fuse(False, True))):
        frac = ((wrong - ref).abs() > 1).float().mean().item() if bug.startswith("align") else (wrong != ref).float().mean().item()
        print(f"  {what} hed_fuse: '{bug}' differs on {100 * frac:.2f} % of the pixels")
        assert frac > 0.01, f"{what}: '{bug}' would not be caught"


# ---- the conditioning embedding's SiLU contractions ---------------------------------------------------------------------------
@pytest.mark.parametrize("height,width", EMBEDDING_CASES)
def test_embedding_silu_convs(cuda, height, width):
    """The six SiLU convs of ControlNetConditioningEmbedding (16 -> 16, 16 -> 32 / 2, 32 -> 32, 32 -> 96 / 2, 96 -> 96,
    96 -> 256 / 2) at a frame's full resolution, as the engine runs them: inputs stored 64 / 64 / 128 columns wide with zero
    padding, outputs into buffers of that width (the padding columns must stay untouched), the engine's plans.  Catches: ReLU
    instead of SiLU; SiLU before the bias."""
    from oracle import controlnet as ocn
    ops = _ops()
    e = ocn.EMBED_CHANNELS
    pad = lambda ch: -(-ch // 64) * 64
    h, w = height, width
    for i in range(len(e) - 1):
        for stride, cout in ((1, e[i]), (2, e[i + 1])):
            cin = e[i]
            x = hetero((1, h, w, pad(cin)), (3,), 60 + i, cuda, offset=1.0)
            x[..., cin:] = 0
            wt = torch.zeros((cout, pad(cin), 3, 3), dtype=torch.float16, device=cuda)
            wt[:, :cin] = _w((cout, cin, 3, 3), 61 + i, cuda)
            bias = (torch.randn((1, cout), generator=torch.Generator().manual_seed(62 + i), dtype=torch.float64) * 2).float().to(cuda)
            ho, wo = h // stride, w // stride
            g = guarded((ho * wo, cout), pitch=pad(cout), device=cuda)
            out = g.view.view(1, ho, wo, cout)
            wp = ops.pack_conv_weight(wt)
            kw = dict(stride=stride, colbias=bias, silu=True)
            plan = ops.igemm_engine_plan([(x, 9)], wp, out, autotile=1, allow_swap=False, **kw)
            ops.igemm([(x, 9)], wp, out, bn=plan.bn, splits=plan.splits, **kw)
            torch.cuda.synchronize()
            what = f"embedding {height}x{width}: {cin} -> {cout} / {stride} at {h}x{w} (bn {plan.bn}, splits {plan.splits})"
            g.assert_untouched(what)
            acc = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), None, stride=stride, padding=1).permute(0, 2, 3, 1)
            pre = acc + bias.double()[0]
            _discriminates(out, F.silu(pre), F.relu(pre), 2e-3, 4e-3, what, "ReLU instead of SiLU")
            _discriminates(out, F.silu(pre), F.silu(acc) + bias.double()[0], 2e-3, 4e-3, what, "SiLU before the bias")
        h, w = h // 2, w // 2


# ---- ControlNet conv_in(x) + cond: one conditioning image for every stream-batch slot ----------------------------------------
@pytest.mark.parametrize("t", COND_RES_BATCHES)
def test_cond_residual_broadcast(cuda, t):
    """smallconv with a residual of batch stride 0 into T slots (the ControlNet's conv_in(x) + cond at the 64 x 192 latent).
    Catches: the residual added to slot 0 only (T > 1); the residual omitted (T = 1)."""
    ops = _ops()
    h, w, cout = 8, 24, 320
    x = hetero((t, h, w, 4), (0, 3), 70, cuda)
    wt = _w((cout, 4, 3, 3), 71, cuda)
    bias = torch.randn(cout, generator=torch.Generator().manual_seed(72)).float().to(cuda)
    res = hetero((1, h, w, cout), (3,), 73, cuda)
    g = guarded((t * h * w, cout), pitch=cout + 8, device=cuda)
    out = g.view.view(t, h, w, cout)
    ops.smallconv_ex(x, wt, bias, out, res=res, res_bstride=0)
    torch.cuda.synchronize()
    g.assert_untouched(f"cond residual T={t}")
    conv = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    ref = conv + res.double()
    if t > 1:
        wrong = conv.clone()
        wrong[0] += res.double()[0]
        bug = "residual added to slot 0 only"
    else:
        wrong, bug = conv, "residual omitted"
    _discriminates(out, ref, wrong, 2e-3, 4e-3, f"cond residual T={t}", bug)


# ---- engine configurations --------------------------------------------------------------------------------------------------
def _stream_loop(cfg):
    """T + 2 frames through the stream loop of a fresh full-size engine against the fp32 oracle on the GPU"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import autoencoder_kl as oakl
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import stream_kl as oskl
    from oracle import unet as ounet
    from oracle import weights as ow
    from tests.test_engine_gpu import _cmp, _u8_check
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    turbo, tl, hw = cfg["turbo"], cfg["tl"], cfg["hw"]
    height, width = (hw, hw) if isinstance(hw, int) else hw
    ucfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
    usd16 = ow.make_unet_weights(ucfg)
    vsd16 = A.synthetic_autoencoder_kl(A.AUTOENCODER_KL) if cfg["kl"] else ow.make_taesd_weights()
    cn16 = ocn.make_weights(ucfg) if cfg["cn"] else None
    hed16 = {k: v.half().float() for k, v in A.synthetic_hed().items()} if cfg["hed"] else None
    emb = ow.make_prompt_embeds(ucfg.cross_attention_dim)
    sd = StreamDiffusion(arch, usd16, vsd16, tl, lambda p: emb, width=width, height=height, device="cuda",
                         use_tiny_vae=not cfg["kl"], controlnet_sd=cn16, hed_sd=hed16)
    sd.prepare("p", guidance_scale=0.0)
    args = (ow.to_float(usd16), ucfg, ow.to_float(vsd16))
    if cn16 is not None:
        kw = dict(hed_sd=hed16) | (dict(vae_kl=oakl.FULL) if cfg["kl"] else {})
        cls = oskl.KLControlNetStreamOracle if cfg["kl"] else ocn.ControlNetStreamOracle
        orc = cls(*args, ow.to_float(cn16), tl, width, height, **kw)
    elif cfg["kl"]:
        orc = oskl.KLStreamOracle(*args, tl, width, height, vae_kl=oakl.FULL)
    else:
        from oracle import stream as ostream
        orc = ostream.StreamOracle(*args, tl, width, height)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    orc = orc.to("cuda")
    T = len(tl)
    for i in range(T + 2):
        frame = ow.make_frame(height, width, seed=400 + i)
        out = sd.step_u8(frame.cuda())
        with torch.no_grad():
            ref = opipe.frame_to_u8(orc, frame.cuda())
        frac, mx = _u8_check(out, ref, f"frame {i}")
        print(f"  frame {i}: u8 frac(|d|<=2) {frac:.5f} max {mx}")
        if T > 1:
            e, c = _cmp("buffer", sd.get_tensor("unet_in")[1:].cpu(), orc.x_t_latent_buffer.cpu(), [])
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: x_t_latent_buffer relerr {e:.3e} cos {c:.6f}"


def _recorded(aud):
    """the branch regimes of the launches an audit saw"""
    from tests import test_config_space as CS
    from tests import test_config_space_branches as B
    got = {k: set() for k in B.BRANCH_CLASSES}
    for nb, ho, wo, tw, th, tn, swap, flags in aud.branch["igemm"]:
        got["contraction"].add(CS.variant_prefix(flags) + CS.contraction_regime(nb, ho, wo, tw, th, tn, swap))
    for kind, key in aud.branch["conv"]:
        if key == "hed.block1.convs.1.weight":
            got["contraction"].add(f"hed:{kind}")
    got["attention"] = {B.d512_regime(sq) for sq in aud.branch["d512"]}
    got["groupnorm"] = {B.gn_regime(ca, hw) for ca, cb, hw in aud.branch["groupnorm"] if cb == 0 and ca // 32 in (4, 8, 16)}
    got["hed"] = {B.maxpool_regime(*s) for s in aud.branch["maxpool2x2"]} | {B.fuse_regime(*s) for s in aud.branch["hed_fuse"]}
    got["batch"] = {B.cond_res_regime(nb) for label, nb in aud.branch["res_bs0"] if "controlnet.conv_in" in label}
    return got


@pytest.mark.parametrize("cfg", SWEEP_BRANCHES)
def test_config_space_branch_engine(cuda, request, cfg):
    from tests import test_config_space_branches as B
    from tests.test_config_space_gpu import _release
    from tests.test_launch_audit_gpu import _audit
    name = request.node.callspec.id
    t0 = time.time()
    aud = _audit(cuda, name, cfg, full=True)
    want, got = B.engine_branch_regimes(cfg), _recorded(aud)
    print(f"{name}: " + "; ".join(f"{k} {sorted(v)}" for k, v in got.items() if v))
    for k in B.BRANCH_CLASSES:
        assert want[k] <= got[k], f"{k} regimes predicted, never launched: {sorted(want[k] - got[k])}"
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    _stream_loop(cfg)
    print(f"{name}: audit + stream loop {time.time() - t0:.1f} s, free HBM before the stream loop {free0 / 2**30:.1f} GiB, "
          f"torch peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB on {torch.cuda.get_device_name()}")
    _release()
