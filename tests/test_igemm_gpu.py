"""GPU parity of the wgmma implicit-GEMM kernel (conv3x3 / 1x1 / Linear / GEGLU / split-K) through
the C ABI (b2sd_op_igemm) against plain PyTorch fp32 ops on the same fp16-rounded operands.

Tolerance: operands are exact fp16; accumulation is fp32 in both; the only difference is the final
fp16 rounding of the output (rel 2^-11) plus accumulation-order noise => abs 2e-3*scale + rel 2e-3.

References of the LayerNorm-folded and prompt-side / ragged-N contractions are float64 on the GPU; the large conv / GEMM
references stay fp32 with TF32 off (the cuda fixture)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close, assert_discriminates, guarded, hetero, offset_heavy_rows

pytestmark = pytest.mark.gpu


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


def _nhwc16(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(torch.float16)


def _ref_conv(x16_nhwc, w16_oihw, stride):
    x = x16_nhwc.float().permute(0, 3, 1, 2)
    y = F.conv2d(x, w16_oihw.float(), None, stride=stride, padding=w16_oihw.shape[-1] // 2)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("m,k,n,bn", [
    (128, 64, 64, 0),      # one tile, one k-block: descriptor sanity
    (128, 128, 64, 0),     # two k-blocks
    (256, 64, 128, 0),
    (4096, 320, 320, 0),   # UNet 64^2 attention projections (BN=160)
    (4096, 320, 320, 64),
    (1000, 640, 1280, 0),  # ragged M (TMA OOB rows), BN=128
    (77, 1024, 320, 0),    # cross-attention K projection of the prompt
    (64, 1280, 1280, 256),
])
def test_linear(cuda, m, k, n, bn):
    ops = _ops()
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    bias = _rand((1, n), cuda, 3).float().contiguous()
    out = torch.full((1, 1, m, n), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], w, out, colbias=bias, bn=bn)
    ref = x.float().reshape(m, k) @ w.float().t() + bias
    assert_close(out.reshape(m, n), ref, 2e-3, 2e-3, f"linear m={m} k={k} n={n} bn={bn}")


def test_linear_residual_scale(cuda):
    ops = _ops()
    m, k, n = 512, 320, 320
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    res = _rand((1, 1, m, n), cuda, 4).to(torch.float16)
    out = torch.empty((1, 1, m, n), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], w, out, res=res, acc_scale=0.5, res_scale=2.0)
    ref = 0.5 * (x.float().reshape(m, k) @ w.float().t()) + 2.0 * res.float().reshape(m, n)
    assert_close(out.reshape(m, n), ref, 4e-3, 2e-3, "linear + residual")


def test_geglu(cuda):
    """FeedForward GEGLU (diffusers attention.py GEGLU): proj -> chunk(h, gate) -> h * gelu(gate).
    Weight rows are packed per 128-wide tile as [64 value rows | 64 gate rows]."""
    ops = _ops()
    m, k, inner = 1024, 320, 1280
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((2 * inner, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    b = _rand((2 * inner,), cuda, 3).float()
    bn = 128
    half = bn // 2
    # pack: tile t holds value rows [t*half, (t+1)*half) then gate rows inner + same
    idx = []
    for t in range(inner // half):
        idx += list(range(t * half, (t + 1) * half))
        idx += list(range(inner + t * half, inner + (t + 1) * half))
    idx = torch.tensor(idx, device=cuda)
    wp = w[idx].contiguous()
    bp = b[idx].reshape(1, -1).contiguous()
    out = torch.empty((1, 1, m, inner), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], wp, out, colbias=bp, geglu=True, bn=bn, n_valid=inner)
    proj = x.float().reshape(m, k) @ w.float().t() + b
    ref = proj[:, :inner] * F.gelu(proj[:, inner:])
    assert_close(out.reshape(m, inner), ref, 3e-3, 3e-3, "geglu")


@pytest.mark.parametrize("nb,h,w,cin,cout,stride,splits,relu", [
    (1, 16, 16, 64, 64, 1, 1, False),     # smallest conv: taps + padding
    (1, 64, 64, 64, 64, 1, 1, True),      # TAESD block conv
    (1, 64, 64, 320, 320, 1, 1, False),   # UNet 64^2 resnet conv
    (1, 32, 32, 640, 640, 1, 2, False),   # split-K 2
    (1, 16, 16, 1280, 1280, 1, 4, False),
    (1, 8, 8, 1280, 1280, 1, 8, False),   # 64-row tile (half-empty M)
    (4, 8, 8, 1280, 1280, 1, 4, False),   # batch packed into one M tile (tn=2)
    (4, 32, 32, 320, 640, 1, 1, False),
    (1, 64, 64, 320, 320, 2, 1, False),   # Downsample2D: stride 2 via TMA elementStrides
    (1, 128, 128, 64, 64, 2, 1, False),   # TAESD encoder stride-2 conv
    (2, 24, 24, 128, 64, 1, 1, True),     # 768-class odd extents (partial tiles)
    (1, 64, 64, 320, 4, 1, 1, False),     # conv_out: Cout=4 padded to N=16
    (1, 12, 7, 1280, 1280, 1, 4, False),  # 768x448 12x7 level: a 12-row x 7-column tile (84 pixels)
    (4, 56, 96, 320, 320, 1, 1, False),   # 448x768 top level at batch 4
    (1, 96, 56, 320, 320, 2, 1, False),   # 768x448 downsample to 48x28
    (1, 56, 96, 320, 4, 1, 1, False),     # conv_out at 448x768
])
def test_conv3x3(cuda, nb, h, w, cin, cout, stride, splits, relu):
    ops = _ops()
    x = _nhwc16(_rand((nb, cin, h, w), cuda, 1))
    wt = _rand((cout, cin, 3, 3), cuda, 2, 1.0 / math.sqrt(9 * cin)).to(torch.float16)
    bias = _rand((nb, cout), cuda, 3).float().contiguous()  # per-sample: bias + time embedding
    ho, wo = h // stride, w // stride
    out = torch.full((nb, ho, wo, cout), float("nan"), dtype=torch.float16, device=cuda)
    wp = ops.pack_conv_weight(wt)
    if cout < 16:  # pad rows so the TMA box (16 rows) stays inside the allocation
        wp = torch.cat([wp, torch.zeros(16 - cout, wp.shape[1], dtype=wp.dtype, device=cuda)]).contiguous()
    ops.igemm([(x, 9)], wp, out, stride=stride, colbias=bias, relu=relu, splits=splits)
    ref = _ref_conv(x, wt, stride) + bias[:, None, None, :]
    if relu:
        ref = ref.relu()
    assert_close(out, ref, 3e-3, 3e-3, f"conv3x3 nb={nb} {h}x{w} {cin}->{cout} s{stride} splits={splits}")


def test_conv_concat_shortcut(cuda):
    """Up-block resnet tail: conv2(3x3 over normalised h) + conv_shortcut(1x1 over cat[xa, xb]) fused as
    one K loop with three TMA sources (diffusers resnet.py ResnetBlock2D: output = shortcut(x) + h)."""
    ops = _ops()
    nb, hh, ww, cmid, ca, cb, cout = 2, 32, 32, 640, 640, 320, 640
    hmid = _nhwc16(_rand((nb, cmid, hh, ww), cuda, 1))
    xa = _nhwc16(_rand((nb, ca, hh, ww), cuda, 2))
    xb = _nhwc16(_rand((nb, cb, hh, ww), cuda, 3))
    w2 = _rand((cout, cmid, 3, 3), cuda, 4, 1.0 / math.sqrt(9 * cmid)).to(torch.float16)
    ws = _rand((cout, ca + cb, 1, 1), cuda, 5, 1.0 / math.sqrt(ca + cb)).to(torch.float16)
    bias = _rand((1, cout), cuda, 6).float().contiguous()
    wp = torch.cat([ops.pack_conv_weight(w2), ws.reshape(cout, ca + cb)], dim=1).contiguous()
    out = torch.empty((nb, hh, ww, cout), dtype=torch.float16, device=cuda)
    ops.igemm([(hmid, 9), (xa, 1), (xb, 1)], wp, out, colbias=bias)
    xcat = torch.cat([xa, xb], dim=3)
    ref = _ref_conv(hmid, w2, 1) + _ref_conv(xcat, ws, 1) + bias[:, None, None, :]
    assert_close(out, ref, 4e-3, 3e-3, "conv2 + shortcut over concat")


def test_channel_slice_views(cuda):
    """Q/K slices of a fused [tokens, 2C] projection are read through strided views (ld > C)."""
    ops = _ops()
    m, c = 512, 320
    qk = _rand((1, 1, m, 2 * c), cuda, 1).to(torch.float16)
    w = _rand((c, c), cuda, 2, 1.0 / math.sqrt(c)).to(torch.float16)
    out = torch.empty((1, 1, m, c), dtype=torch.float16, device=cuda)
    kview = qk[..., c:]
    ops.igemm([(kview, 1)], w, out)
    ref = kview.float().reshape(m, c) @ w.float().t()
    assert_close(out.reshape(m, c), ref, 2e-3, 2e-3, "strided channel view")


def test_swapped_operands_vt(cuda):
    """V^T = Wv . X^T: weights on the M side, tokens on the N side -> [C][tokens] (K-major for P.V)."""
    ops = _ops()
    tokens, c = 1024, 320
    x = _rand((tokens, c), cuda, 1).to(torch.float16).contiguous()
    wv = _rand((1, 1, c, c), cuda, 2, 1.0 / math.sqrt(c)).to(torch.float16)
    out = torch.empty((1, 1, c, tokens), dtype=torch.float16, device=cuda)
    ops.igemm([(wv, 1)], x, out, bn=128)
    ref = wv.float().reshape(c, c) @ x.float().t()
    assert_close(out.reshape(c, tokens), ref, 2e-3, 2e-3, "V^T swapped-operand GEMM")


@pytest.mark.parametrize("nb,h,w,cin,cout,stride,bn,splits,res", [
    (1, 16, 16, 64, 128, 1, 256, 1, False),    # one pixel tile, one channel tile
    (1, 64, 64, 320, 320, 1, 256, 2, True),    # UNet 64^2 resnet conv2 (+x), 320 = 2.5 channel tiles
    (1, 32, 32, 640, 640, 1, 256, 4, False),
    (1, 16, 16, 1280, 1280, 1, 256, 8, True),
    (1, 8, 8, 1280, 1280, 1, 64, 8, False),
    (4, 8, 8, 1280, 1280, 1, 256, 8, False),   # four images in one pixel tile
    (1, 64, 64, 320, 320, 2, 256, 1, False),   # stride-2 downsample
    (2, 24, 24, 128, 192, 1, 128, 1, False),   # ragged extents
    (1, 6, 8, 1280, 1280, 1, 64, 8, False),    # 384x512 SD-Turbo 6x8 level: an 8x8 pixel tile with two masked rows
    (1, 12, 7, 1280, 1280, 1, 64, 8, True),    # 768x448 12x7 level: one masked column per pixel row
    (4, 2, 3, 256, 256, 1, 64, 4, False),      # tiny 128x192 2x3 level, four images in one pixel tile
    (1, 24, 14, 1280, 1280, 2, 128, 4, False), # 768x448 stride-2 downsample to 12x7
])
def test_conv3x3_swapped_orientation(cuda, nb, h, w, cin, cout, stride, bn, splits, res):
    """D^T = W . X^T: output channels on the MMA M side, a tile of bn pixels on the N side, transposed store."""
    ops = _ops()
    x = _nhwc16(_rand((nb, cin, h, w), cuda, 1))
    wt = _rand((cout, cin, 3, 3), cuda, 2, 1.0 / math.sqrt(9 * cin)).to(torch.float16)
    bias = _rand((nb, cout), cuda, 3).float().contiguous()
    ho, wo = h // stride, w // stride
    r = _nhwc16(_rand((nb, cout, ho, wo), cuda, 4)) if res else None
    out = torch.full((nb, ho, wo, cout), float("nan"), dtype=torch.float16, device=cuda)
    wp = ops.pack_conv_weight(wt)
    ops.igemm([(x, 9)], wp, out, stride=stride, colbias=bias, res=r, bn=bn, splits=splits, swap=True)
    ref = _ref_conv(x, wt, stride) + bias[:, None, None, :]
    if res:
        ref = ref + r.float()
    assert_close(out, ref, 4e-3, 3e-3, f"swapped conv nb={nb} {h}x{w} {cin}->{cout} s{stride} bn={bn} splits={splits}")


@pytest.mark.parametrize("m,k,n,bn,splits", [(4096, 320, 320, 256, 1), (1024, 640, 640, 256, 2), (256, 1280, 1280, 256, 4),
                                               (64, 1280, 1280, 64, 8), (77, 1024, 640, 128, 1), (4096, 1280, 320, 256, 4)])
def test_linear_swapped_orientation(cuda, m, k, n, bn, splits):
    ops = _ops()
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    bias = _rand((1, n), cuda, 3).float().contiguous()
    res = _rand((1, 1, m, n), cuda, 4).to(torch.float16)
    out = torch.full((1, 1, m, n), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], w, out, colbias=bias, res=res, bn=bn, splits=splits, swap=True)
    ref = x.float().reshape(m, k) @ w.float().t() + bias + res.float().reshape(m, n)
    assert_close(out.reshape(m, n), ref, 4e-3, 3e-3, f"swapped linear m={m} k={k} n={n}")


@pytest.mark.parametrize("nb,h,w,relu,res", [
    (1, 16, 8, False, False),      # exactly one 16x8 tile: descriptor / tap-shift sanity
    (1, 64, 64, True, True),       # TAESD block tail at the latent size: bias + skip + ReLU
    (1, 256, 256, True, False),    # 512 tiles on persistent CTAs: ring wrap-around, several tiles per CTA
    (2, 40, 28, True, True),       # ragged extents (partial tiles in h and w), two images
    (1, 512, 512, True, True),     # the full-size TAESD body convolution of the 512x512 configs
])
def test_tconv_persistent_halo(cuda, nb, h, w, relu, res):
    """Persistent halo-tile kernel (tconv.cu: resident weights, nine shifted descriptors over one halo tile) against
    F.conv2d; same tolerance as the tap-by-tap kernel, and bit-identical to it (same fp32 accumulation order per tap)."""
    ops = _ops()
    x = _nhwc16(_rand((nb, 64, h, w), cuda, 1))
    wt = _rand((64, 64, 3, 3), cuda, 2, 1.0 / math.sqrt(9 * 64)).to(torch.float16)
    bias = _rand((1, 64), cuda, 3).float().contiguous()
    r = _nhwc16(_rand((nb, 64, h, w), cuda, 4)) if res else None
    wp = ops.pack_conv_weight(wt)
    out = torch.full((nb, h, w, 64), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 9)], wp, out, colbias=bias, res=r, relu=relu, tconv=True)
    ref = _ref_conv(x, wt, 1) + bias[:, None, None, :]
    if res:
        ref = ref + r.float()
    if relu:
        ref = ref.relu()
    assert_close(out, ref, 3e-3, 3e-3, f"tconv nb={nb} {h}x{w} relu={relu} res={res}")
    base = torch.empty_like(out)
    ops.igemm([(x, 9)], wp, base, colbias=bias, res=r, relu=relu)
    assert_close(out, base, 1e-3, 1e-3, "tconv vs tap-by-tap kernel")


def test_tconv_rejects_other_shapes(cuda):
    ops = _ops()
    x = _nhwc16(_rand((1, 128, 16, 16), cuda, 1))
    wp = ops.pack_conv_weight(_rand((64, 128, 3, 3), cuda, 2).to(torch.float16))
    out = torch.empty((1, 16, 16, 64), dtype=torch.float16, device=cuda)
    with pytest.raises(Exception):
        ops.igemm([(x, 9)], wp, out, tconv=True)


# ---- LayerNorm folded into the consumer GEMM + fused q/k/v projection (BasicTransformerBlock without layernorm launches) ----
STAT_SCALE = float(1 << 20)


def _ln_fold_operands(w16, gamma, beta, bias):
    """What the engine prepares at load time (engine.cu fold_ln): W' = W diag(gamma) in fp16, colsum over the ROUNDED W',
    bias' = W beta + b."""
    wp = (w16.float() * gamma[None, :]).to(torch.float16).contiguous()
    colsum = wp.float().sum(dim=1).contiguous()
    bprime = (w16.float() @ beta + (bias if bias is not None else 0)).float().contiguous()
    return wp, colsum, bprime


@pytest.mark.parametrize("m,k,n,splits", [(4096, 320, 320, 1), (256, 1280, 1280, 4), (1000, 640, 640, 1)])
def test_linear_row_statistics(cuda, m, k, n, splits):
    """rowstat_out: (sum, sum of squares) of every stored fp16 row in 2^20 fixed point -- exactly what a LayerNorm reading the
    row back would reduce; integer atomics => bit-identical across runs (N tiles / split-K CTAs arrive in any order)."""
    ops = _ops()
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    bias = _rand((1, n), cuda, 3).float().contiguous()
    res = _rand((1, 1, m, n), cuda, 4).to(torch.float16)
    outs, stats = [], []
    for _ in range(3):
        out = torch.empty((1, 1, m, n), dtype=torch.float16, device=cuda)
        st = torch.zeros((m, 2), dtype=torch.int64, device=cuda)
        ops.igemm([(x, 1)], w, out, colbias=bias, res=res, splits=splits, rowstat_out=st)
        outs.append(out)
        stats.append(st)
    assert torch.equal(stats[0], stats[1]) and torch.equal(stats[0], stats[2]) and torch.equal(outs[0], outs[1])
    y = outs[0].reshape(m, n).double()
    want = torch.stack([y.sum(1), (y * y).sum(1)], dim=1)
    got = stats[0].double() / STAT_SCALE
    assert_close(got, want, 2e-3, 1e-5, "row statistics")


def _ln_rows(x2d, gamma, beta, neighbour=False):
    """float64 LayerNorm (eps 1e-5) of the rows of x2d; neighbour=True normalises row r with the statistics of row r-1 (the
    wrong reference for a row-indexing error of the folded epilogue under split-K, CTA pairs and N tiles)."""
    xd = x2d.double()
    mean, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    if neighbour:
        mean, var = mean.roll(1, 0), var.roll(1, 0)
    return (xd - mean) * (var + 1e-5).rsqrt() * gamma.double() + beta.double()


def _fixed_point_rowstats(x2d):
    xf = x2d.double()
    return torch.stack([xf.sum(1), (xf * xf).sum(1)], dim=1).mul(STAT_SCALE).round().to(torch.int64).contiguous()


@pytest.mark.parametrize("m,k,n,splits", [(4096, 320, 640, 1), (256, 1280, 2560, 2), (64, 1280, 1280, 4)])
def test_linear_layernorm_folded(cuda, m, k, n, splits):
    """y = LayerNorm(x) W^T + b computed as rstd (x W'^T - mean colsum) + bias' from the producer's row statistics.  Every row
    has its own offset and scale, so a row normalised with another row's statistics is off by O(1)."""
    ops = _ops()
    x = hetero((1, 1, m, k), (2,), 1, cuda)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    gamma = (1.0 + 0.1 * _rand((k,), cuda, 3)).float()
    beta = (0.1 * _rand((k,), cuda, 4)).float()
    bias = _rand((n,), cuda, 5).float()
    wp, colsum, bprime = _ln_fold_operands(w, gamma, beta, bias)
    st = _fixed_point_rowstats(x.reshape(m, k))
    out = torch.full((1, 1, m, n), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], wp, out, colbias=bprime.reshape(1, n).contiguous(), splits=splits, rowstat_in=st, colsum=colsum, ln_c=k)
    ref = _ln_rows(x.reshape(m, k), gamma, beta) @ w.double().t() + bias.double()
    wrong = _ln_rows(x.reshape(m, k), gamma, beta, neighbour=True) @ w.double().t() + bias.double()
    assert_discriminates(out.reshape(m, n), ref, wrong, 6e-3, 4e-3, f"LN-folded linear m={m} k={k} n={n}",
                         "statistics of the neighbouring row")


@pytest.mark.parametrize("m,k,n,splits", [(1024, 640, 640, 1), (256, 1280, 1280, 4)])
def test_linear_layernorm_folded_offset_heavy(cuda, m, k, n, splits):
    """Rows with |mean|/std of 30..100: the folded epilogue (ln_row_stats) takes the variance as E[x^2] - mean^2 in fp32 from
    the fixed-point row sums and subtracts mean * colsum from the accumulator; this pins that range as the one in which both
    hold the usual tolerance.  The error, in units of the tolerance, is printed."""
    ops = _ops()
    x = offset_heavy_rows(m, k, cuda).reshape(1, 1, m, k)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    gamma = (1.0 + 0.1 * _rand((k,), cuda, 3)).float()
    beta = (0.1 * _rand((k,), cuda, 4)).float()
    bias = _rand((n,), cuda, 5).float()
    wp, colsum, bprime = _ln_fold_operands(w, gamma, beta, bias)
    st = _fixed_point_rowstats(x.reshape(m, k))
    out = torch.full((1, 1, m, n), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], wp, out, colbias=bprime.reshape(1, n).contiguous(), splits=splits, rowstat_in=st, colsum=colsum, ln_c=k)
    ref = _ln_rows(x.reshape(m, k), gamma, beta) @ w.double().t() + bias.double()
    err = ((out.reshape(m, n).double() - ref).abs() / (6e-3 + 4e-3 * ref.abs())).max().item()
    print(f"LN-folded linear offset-heavy m={m} k={k} n={n} splits={splits}: max error = {err:.3f} x tolerance")
    wrong = _ln_rows(x.reshape(m, k), gamma, beta, neighbour=True) @ w.double().t() + bias.double()
    assert_discriminates(out.reshape(m, n), ref, wrong, 6e-3, 4e-3, f"offset-heavy LN-folded linear m={m} k={k} n={n}",
                         "statistics of the neighbouring row")


def fused_qkv_case(cuda, pair):
    """One GEMM over [Wq | Wk | Wv] with LayerNorm folded, q | k written with the engine's row pitch and V^T [C][tokens] through
    out2, both into guarded buffers whose pitch is wider than their data (the engine's bump-allocated arena has neighbours on
    both sides)."""
    ops = _ops()
    m, c = 4096, 320
    x = hetero((1, 1, m, c), (2,), 1, cuda)
    wq, wk, wv = (_rand((c, c), cuda, s, 1.0 / math.sqrt(c)).to(torch.float16) for s in (2, 3, 4))
    gamma = (1.0 + 0.1 * _rand((c,), cuda, 5)).float()
    beta = (0.1 * _rand((c,), cuda, 6)).float()
    w = torch.cat([wq, wk, wv]).contiguous()
    wp, colsum, bprime = _ln_fold_operands(w, gamma, beta, None)
    st = _fixed_point_rowstats(x.reshape(m, c))
    qk = guarded((m, 2 * c), pitch=2 * c + 64, device=cuda)
    vt = guarded((c, m), pitch=m + 64, device=cuda)
    ops.igemm([(x, 1)], wp, qk.view[None, None], colbias=bprime.reshape(1, -1).contiguous(), n_valid=3 * c, rowstat_in=st,
              colsum=colsum, ln_c=c, out2=vt.view, col2=2 * c, bn=160, pair=pair)
    qk.assert_untouched("q | k")
    vt.assert_untouched("V^T")
    ln, ln_wrong = _ln_rows(x.reshape(m, c), gamma, beta), _ln_rows(x.reshape(m, c), gamma, beta, neighbour=True)
    wqk = torch.cat([wq, wk]).double().t()
    bug = "statistics of the neighbouring row"
    assert_discriminates(qk.view, ln @ wqk, ln_wrong @ wqk, 6e-3, 4e-3, "q | k", bug)
    assert_discriminates(vt.view, (ln @ wv.double().t()).t(), (ln_wrong @ wv.double().t()).t(), 6e-3, 4e-3, "V^T", bug)


def test_fused_qkv_projection_with_transposed_v(cuda):
    """The V block stored as V^T [C][tokens] (the K-major operand of the attention P.V MMA), replacing a separate
    swapped-operand GEMM launch."""
    fused_qkv_case(cuda, pair=False)


def test_geglu_layernorm_folded(cuda):
    ops = _ops()
    m, k, inner = 1024, 320, 1280
    x = hetero((1, 1, m, k), (2,), 1, cuda)
    w = _rand((2 * inner, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    b = _rand((2 * inner,), cuda, 3).float()
    gamma = (1.0 + 0.1 * _rand((k,), cuda, 4)).float()
    beta = (0.1 * _rand((k,), cuda, 5)).float()
    half = 64
    idx = []
    for t in range(inner // half):
        idx += list(range(t * half, (t + 1) * half))
        idx += list(range(inner + t * half, inner + (t + 1) * half))
    idx = torch.tensor(idx, device=cuda)
    wp, colsum, bprime = _ln_fold_operands(w[idx].contiguous(), gamma, beta, b[idx])
    st = _fixed_point_rowstats(x.reshape(m, k))
    out = torch.empty((1, 1, m, inner), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], wp, out, colbias=bprime.reshape(1, -1).contiguous(), geglu=True, bn=128, n_valid=inner,
              rowstat_in=st, colsum=colsum, ln_c=k)

    def geglu_ref(neighbour):
        proj = _ln_rows(x.reshape(m, k), gamma, beta, neighbour) @ w.double().t() + b.double()
        return proj[:, :inner] * F.gelu(proj[:, inner:])
    assert_discriminates(out.reshape(m, inner), geglu_ref(False), geglu_ref(True), 8e-3, 5e-3, "LN-folded GEGLU",
                         "statistics of the neighbouring row")


# ---- prompt-side and ragged-N contractions, run with the tiles the engine's policy picks ----------------------------------------
def _engine_tiles(ops, srcs, w, out, autotile, allow_swap, **kw):
    info = ops.igemm_engine_plan(srcs, w, out, autotile=autotile, allow_swap=allow_swap, **kw)
    return dict(bn=info.bn, splits=info.splits, swap=bool(info.swap), pair=info.mode == 1)


def _gemm64(a, b):
    """float64 a @ b^T on the GPU (the prompt-side GEMMs are small)."""
    return a.double() @ b.double().t()


@pytest.mark.parametrize("autotile", [1, 2])
@pytest.mark.parametrize("d", [768, 1024])
@pytest.mark.parametrize("cp", [320, 512, 1024, 1536])
def test_prompt_vt_projection(cuda, cp, d, autotile):
    """The cross-attention V^T cache as the engine builds it (engine.cu, prompt program): to_v weights [Cp, D] on the M side,
    the 77-token context [77, D] on the N side, n_valid = 77 written with a row pitch of 128.  Columns 77..127 and the rows
    after Cp are guarded.  Catches: a ragged N tile storing past n_valid, V^T columns shifted by one token."""
    ops = _ops()
    L, pitch = 77, 128
    wv = _rand((1, 1, cp, d), cuda, 1, 1.0 / math.sqrt(d)).to(torch.float16)
    ctx = hetero((L, d), (0,), 2, cuda, offset=1.0, scale=(0.5, 2.0))
    out = guarded((cp, L), pitch=pitch, device=cuda)
    o4 = out.view[None, None]
    tiles = _engine_tiles(ops, [(wv, 1)], ctx, o4, autotile, False, n_valid=L)
    ops.igemm([(wv, 1)], ctx, o4, n_valid=L, **tiles)
    out.assert_untouched(f"prompt V^T cp={cp} d={d} {tiles}")
    ref = _gemm64(wv.reshape(cp, d), ctx)
    assert_discriminates(out.view, ref, ref.roll(1, 1), 2e-3, 2e-3, f"prompt V^T cp={cp} d={d} {tiles}",
                         "token columns shifted by one")


@pytest.mark.parametrize("autotile", [1, 2])
@pytest.mark.parametrize("cp", [512, 1024, 1536])
def test_prompt_k_projection_sd15(cuda, cp, autotile):
    """K of the SD-1.5 prompt cache: ctx [77, 768] x to_k [Cp, 768]^T, 77 rows (a partial M tile) with the tiles the engine
    picks; the rows after the 77th are guarded.  Catches: rows of the partial M tile written past the end, a dropped K block."""
    ops = _ops()
    L, d = 77, 768
    ctx = hetero((1, 1, L, d), (2,), 2, cuda, offset=1.0, scale=(0.5, 2.0))
    wk = _rand((cp, d), cuda, 1, 1.0 / math.sqrt(d)).to(torch.float16)
    out = guarded((L, cp), device=cuda)
    o4 = out.view[None, None]
    tiles = _engine_tiles(ops, [(ctx, 1)], wk, o4, autotile, False)
    ops.igemm([(ctx, 1)], wk, o4, **tiles)
    out.assert_untouched(f"prompt K cp={cp} {tiles}")
    ref = _gemm64(ctx.reshape(L, d), wk)
    wrong = _gemm64(ctx.reshape(L, d)[:, 64:], wk[:, 64:])
    assert_discriminates(out.view, ref, wrong, 2e-3, 2e-3, f"prompt K cp={cp} {tiles}", "first K block dropped")


@pytest.mark.parametrize("autotile", [1, 2])
@pytest.mark.parametrize("n", [77, 100, 120])
@pytest.mark.parametrize("m,k", [(4096, 320), (1024, 640), (256, 1280)])
def test_ragged_n_linear(cuda, m, k, n, autotile):
    """N not a multiple of 16, with bias and residual, through the plan the engine's tile policy picks (the swapped orientation
    where it allows it: n % 8 == 0), into a guarded output with spare columns up to the next multiple of 64.  Catches: stores
    past n_valid, bias / residual columns misaligned by one."""
    ops = _ops()
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    bias = _rand((1, n), cuda, 3).float().contiguous()
    pitch = -(-n // 64) * 64 + 64
    res = hetero((m, pitch), (1,), 4, cuda)[:, :n]     # the residual stream is read through the same kind of pitched view
    out = guarded((m, n), pitch=pitch, device=cuda)
    o4 = out.view[None, None]
    tiles = _engine_tiles(ops, [(x, 1)], w, o4, autotile, True, colbias=bias, res=res[None, None])
    ops.igemm([(x, 1)], w, o4, colbias=bias, res=res[None, None], **tiles)
    what = f"ragged linear m={m} k={k} n={n} {tiles}"
    out.assert_untouched(what)
    acc = _gemm64(x.reshape(m, k), w)
    ref = acc + bias.double() + res.double()
    assert_discriminates(out.view, ref, acc + bias.double() + res.double().roll(1, 1), 4e-3, 3e-3, what,
                         "residual columns shifted by one")
    assert_discriminates(out.view, ref, acc + bias.double().roll(1, 1) + res.double(), 4e-3, 3e-3, what,
                         "bias columns shifted by one")
