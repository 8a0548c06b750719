"""GPU parity of the CTA-pair form of the implicit-GEMM kernel (a 2-CTA cluster on neighbouring M tiles: every CTA loads half of the
weight tile and multicasts it to both) through the C ABI, against plain PyTorch fp32 ops on the same fp16-rounded operands and --
bit for bit -- against the single-CTA kernel with the same tile / split-K (same fp32 summation order per output element)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_igemm_gpu import STAT_SCALE, _nhwc16, _ops, _rand, _ref_conv, fused_qkv_case
from tests.util import assert_close

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m,k,n,bn,splits", [
    (256, 64, 64, 64, 1),        # one pair, one K-block: descriptor / barrier sanity
    (256, 512, 64, 64, 1),       # ring wraps (8 K-blocks)
    (4096, 320, 320, 160, 1),    # UNet 64^2 projections: 80 weight rows per CTA
    (4096, 320, 1280, 256, 1),   # widest tile: 128 weight rows per CTA
    (1000, 640, 1280, 128, 1),   # ragged M (TMA OOB rows)
    (896, 640, 640, 128, 1),     # odd number of M tiles: the last pair has one masked tile
    (1024, 1280, 640, 160, 2),   # split-K 2: cluster (2,1,2)
    (256, 2560, 1280, 256, 4),   # split-K 4: cluster (2,1,4)
])
def test_linear_pair(cuda, m, k, n, bn, splits):
    ops = _ops()
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    bias = _rand((1, n), cuda, 3).float().contiguous()
    out = torch.full((1, 1, m, n), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], w, out, colbias=bias, bn=bn, splits=splits, pair=True)
    ref = x.float().reshape(m, k) @ w.float().t() + bias
    assert_close(out.reshape(m, n), ref, 2e-3, 2e-3, f"pair linear m={m} k={k} n={n} bn={bn} splits={splits}")
    single = torch.empty_like(out)
    ops.igemm([(x, 1)], w, single, colbias=bias, bn=bn, splits=splits)
    assert torch.equal(out, single), "pair and single-CTA kernels differ"


@pytest.mark.parametrize("nb,h,w,cin,cout,stride,bn,splits,relu", [
    (1, 16, 16, 64, 64, 1, 64, 1, False),
    (1, 64, 64, 320, 320, 1, 160, 1, False),    # UNet 64^2 resnet conv
    (1, 64, 64, 320, 320, 1, 160, 4, False),    # ... with the frame program's split-K
    (1, 32, 32, 640, 640, 1, 160, 4, False),
    (1, 16, 16, 1280, 1280, 1, 256, 4, False),
    (1, 64, 64, 320, 320, 2, 160, 1, False),    # stride 2
    (2, 24, 24, 128, 64, 1, 64, 1, True),       # odd extents (partial tiles)
    (1, 256, 256, 64, 64, 1, 64, 1, True),      # 512 M tiles: persistent pairs, two accumulators
    (4, 96, 56, 320, 320, 1, 160, 1, False),    # 768x448 top level at batch 4
    (1, 48, 64, 640, 640, 2, 160, 1, False),    # 384x512: stride 2 to 24x32
    (4, 12, 7, 1280, 1280, 1, 64, 1, False),    # 12x7 level at batch 4: one 12x7 tile (84 of 128 rows) per image
    (1, 384, 256, 64, 64, 1, 64, 1, True),      # TAESD body of a 768x512 frame: persistent pairs, non-square
])
def test_conv3x3_pair(cuda, nb, h, w, cin, cout, stride, bn, splits, relu):
    ops = _ops()
    x = _nhwc16(_rand((nb, cin, h, w), cuda, 1))
    wt = _rand((cout, cin, 3, 3), cuda, 2, 1.0 / math.sqrt(9 * cin)).to(torch.float16)
    bias = _rand((nb, cout), cuda, 3).float().contiguous()
    ho, wo = h // stride, w // stride
    out = torch.full((nb, ho, wo, cout), float("nan"), dtype=torch.float16, device=cuda)
    wp = ops.pack_conv_weight(wt)
    ops.igemm([(x, 9)], wp, out, stride=stride, colbias=bias, relu=relu, bn=bn, splits=splits, pair=True)
    ref = _ref_conv(x, wt, stride) + bias[:, None, None, :]
    if relu:
        ref = ref.relu()
    assert_close(out, ref, 3e-3, 3e-3, f"pair conv3x3 nb={nb} {h}x{w} {cin}->{cout} s{stride} bn={bn} splits={splits}")
    single = torch.empty_like(out)
    ops.igemm([(x, 9)], wp, single, stride=stride, colbias=bias, relu=relu, bn=bn, splits=splits)
    assert torch.equal(out, single), "pair and single-CTA kernels differ"


def test_fused_qkv_pair(cuda):
    """LayerNorm-folded fused q/k/v projection with the transposed V store, on CTA pairs."""
    fused_qkv_case(cuda, pair=True)


def test_geglu_pair(cuda):
    """GEGLU tile = [value half | gate half]: with pairs the leader stages the value rows, the peer the gate rows."""
    ops = _ops()
    m, k, inner = 1024, 320, 1280
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((2 * inner, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    b = _rand((2 * inner,), cuda, 3).float()
    bn, half = 128, 64
    idx = []
    for t in range(inner // half):
        idx += list(range(t * half, (t + 1) * half))
        idx += list(range(inner + t * half, inner + (t + 1) * half))
    idx = torch.tensor(idx, device=cuda)
    out = torch.empty((1, 1, m, inner), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 1)], w[idx].contiguous(), out, colbias=b[idx].reshape(1, -1).contiguous(), geglu=True, bn=bn, n_valid=inner, pair=True)
    h = x.float().reshape(m, k) @ w.float().t() + b
    ref = h[:, :inner] * F.gelu(h[:, inner:])
    assert_close(out.reshape(m, inner), ref, 4e-3, 4e-3, "pair GEGLU")


def test_row_statistics_pair(cuda):
    ops = _ops()
    m, k, n = 4096, 320, 320
    x = _rand((1, 1, m, k), cuda, 1).to(torch.float16)
    w = _rand((n, k), cuda, 2, 1.0 / math.sqrt(k)).to(torch.float16)
    out = torch.empty((1, 1, m, n), dtype=torch.float16, device=cuda)
    st = torch.zeros((m, 2), dtype=torch.int64, device=cuda)
    ops.igemm([(x, 1)], w, out, bn=160, rowstat_out=st, pair=True)
    y = out.reshape(m, n).double()
    want = torch.stack([y.sum(1), (y * y).sum(1)], dim=1)
    assert_close(st.double() / STAT_SCALE, want, 2e-3, 1e-5, "pair row statistics")
