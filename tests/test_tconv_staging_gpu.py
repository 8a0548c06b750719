"""GPU parity of the persistent TAESD convolution (tconv.cu) where its epilogue goes through the shared-memory staging tile:
the residual loaded by TMA tile after tile on the same CTA, and output / residual views whose rows are wider than the 64
channels the kernel writes.  Reference: F.conv2d in fp32 on the same fp16 operands, and the tap-by-tap kernel (igemm.cu),
which performs the same fp32 operations in the same order."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close

pytestmark = pytest.mark.gpu


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


def _nhwc16(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(torch.float16)


@pytest.mark.parametrize("nb,h,w,relu,ldo,ldr", [
    (1, 256, 256, False, 64, 64),    # 512 tiles: several tiles per CTA, each with its residual through the staging tile
    (2, 40, 28, True, 96, 128),      # ragged tiles, output and residual inside wider rows with pitches of their own
    (1, 64, 64, True, 128, 72),
])
def test_tconv_staged_residual_and_pitch(cuda, nb, h, w, relu, ldo, ldr):
    from ai_rtc_agent_b200.host import ops
    x = _nhwc16(_rand((nb, 64, h, w), cuda, 1))
    wt = _rand((64, 64, 3, 3), cuda, 2, 1.0 / math.sqrt(9 * 64)).to(torch.float16)
    bias = _rand((1, 64), cuda, 3).float().contiguous()
    r = _nhwc16(_rand((nb, ldr, h, w), cuda, 4))[..., :64]
    wp = ops.pack_conv_weight(wt)
    out_rows = torch.full((nb, h, w, ldo), float("nan"), dtype=torch.float16, device=cuda)
    out = out_rows[..., :64]
    ops.igemm([(x, 9)], wp, out, colbias=bias, res=r, relu=relu, tconv=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), None, padding=1).permute(0, 2, 3, 1) + bias[:, None, None, :]
    ref = ref + r.float()
    if relu:
        ref = ref.relu()
    assert_close(out, ref, 3e-3, 3e-3, f"tconv nb={nb} {h}x{w} relu={relu} ldo={ldo} ldr={ldr}")
    assert bool(torch.isnan(out_rows[..., 64:]).all()), "tconv wrote past the 64 output channels of a row"
    base = torch.full((nb, h, w, 64), float("nan"), dtype=torch.float16, device=cuda)
    ops.igemm([(x, 9)], wp, base, colbias=bias, res=r, relu=relu)
    assert_close(out, base, 1e-3, 1e-3, "tconv vs tap-by-tap kernel")
