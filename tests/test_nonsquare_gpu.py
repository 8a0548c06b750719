"""The implicit-GEMM kernel at the latent levels of non-square engines, with the plans the engine's tile policy picks.

Every other conv test uses h == w somewhere; here each level has H != W, so a kernel that mixes up the two extents (in its tile
decomposition, its TMA box coordinates or its masking of partial tiles) writes a different image.  The sizes reach tile shapes
no square engine reaches: 768x448 has a 12x7 level (Wo = 7: a 12-row x 7-column tile of 84 pixels), 384x512 puts its 6x8 level
(48 rows) on the swapped path, and the tiny 128x192 engine packs several 2x3 / 4x6 images into one M tile at batch 4.  (The
swapped orientation at 12x7, which the policy does not pick, is a case of test_igemm_gpu.py's swapped-orientation test.)

Inputs have their own statistics per (image, channel) and a per-image column bias (the time embedding); outputs are guarded
(pitch > Cout, sentinel-filled).  References are float64 on the GPU.  Each case also shows that it would catch H and W swapped
(contractions with 3x3 taps) or pixels shifted by one column (1x1 contractions, where the layout of the pixels does not change
the result), and at batch 4 image 0's input or image 0's bias used for every image.

A case is a contraction family (its segment taps and stride) at one level under one plan; cases with the same family, output
extents, batch and plan (bn, splits, swap, mode) run once."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import SENTINEL, assert_discriminates, guarded, hetero

pytestmark = pytest.mark.gpu

SD_CHS = (320, 640, 1280, 1280)
TINY_CHS = (64, 128, 256, 256)    # oracle.unet.tiny_config


def _families(lh, lw, chs):
    """(h, w, [(channels, ntap)], cout, stride) of the contraction families tests/test_plan.py:_unet_shapes lists: 3x3 c -> c,
    3x3 + 1x1 shortcut over a concatenation, 1x1 projection, stride-2 downsample, at every latent level."""
    out = []
    for k, c in enumerate(chs):
        h, w = lh >> k, lw >> k
        skip = chs[max(k - 1, 0)]
        out += [(h, w, [(c, 9)], c, 1), (h, w, [(c, 9), (c, 1), (skip, 1)], c, 1), (h, w, [(c, 1)], c, 1)]
        if k < 3:
            out.append((h, w, [(c, 9)], c, 2))
    return out


def _conv(srcs, ws, stride):
    """float64 NHWC sum over the segments of conv(x, w): 3x3 (padding 1) or 1x1 taps, all at `stride`."""
    acc = 0
    for x, w in zip(srcs, ws):
        y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None, stride=stride, padding=w.shape[-1] // 2)
        acc = acc + y.permute(0, 2, 3, 1)
    return acc


PLANS = ((1, True), (1, False), (2, True))   # (autotile, allow_swap) of the engine's tile policy


def _case(height, width, chs, nb, name):
    return pytest.param(height, width, chs, nb, id=f"{name}-{nb}")


# Beyond the non-square sizes: the sizes the engine accepts at its edges and the tile regimes only they reach
# (tests/test_config_space.py) -- 64 x 64 (1 x 1 deepest level: the 128 x 1 row tile, four 1-pixel images in one M tile, the
# swapped orientation at 2 x 2), 576 (9 x 9 level: 117-row tiles; 18-wide level: a 16-wide tile with 2 valid columns),
# 704 x 320 at batch 5 (11 x 5 level: 2 images per tile, the last one a phantom), 960 x 832 (15 x 13 level) and 1024 at
# batch 3.  Batches 3 and 5 leave a phantom image in the last M tile; batch 16 fills several tiles with images.
CASES = [_case(h, w, chs, nb, name) for (h, w, chs, name) in
         ((384, 512, SD_CHS, "384x512"), (448, 768, SD_CHS, "448x768"), (768, 448, SD_CHS, "768x448"),
          (128, 192, TINY_CHS, "tiny-128x192")) for nb in (1, 4)] + [
    _case(64, 64, SD_CHS, 1, "64"), _case(64, 64, SD_CHS, 4, "64"), _case(64, 64, TINY_CHS, 16, "tiny-64"),
    _case(512, 512, TINY_CHS, 3, "tiny-512"), _case(448, 448, TINY_CHS, 3, "tiny-448"),
    _case(576, 576, TINY_CHS, 1, "tiny-576"), _case(704, 320, TINY_CHS, 5, "tiny-704x320"),
    _case(960, 832, TINY_CHS, 1, "tiny-960x832"), _case(1024, 1024, TINY_CHS, 3, "tiny-1024"),
    _case(128, 128, TINY_CHS, 16, "tiny-128"),
    # extreme aspect ratios: levels a few rows high and 16 or more columns wide put several images into one 16- or 8-wide
    # tile, and take the swapped orientation to 16-wide pixel tiles
    _case(64, 576, TINY_CHS, 3, "tiny-64x576"), _case(64, 1024, SD_CHS, 3, "64x1024"), _case(64, 320, TINY_CHS, 4, "tiny-64x320"),
    _case(64, 768, TINY_CHS, 4, "tiny-64x768"), _case(64, 576, SD_CHS, 1, "64x576"), _case(64, 512, TINY_CHS, 1, "tiny-64x512"),
    _case(192, 768, TINY_CHS, 3, "tiny-192x768"), _case(128, 64, SD_CHS, 1, "128x64"), _case(64, 256, SD_CHS, 1, "64x256"),
]


@pytest.mark.parametrize("height,width,chs,nb", CASES)
def test_igemm_nonsquare_levels(cuda, height, width, chs, nb):
    from ai_rtc_agent_b200.host import ops
    seen = set()
    seed = 0
    for (h, w, segs, cout, stride) in _families(height // 8, width // 8, chs):
        seed += 1
        srcs = [hetero((nb, h, w, c), (0, 3), 100 * seed + i, cuda) for i, (c, _) in enumerate(segs)]
        g = torch.Generator().manual_seed(seed)
        k_total = sum(c * t for c, t in segs)
        ws = [(torch.randn((cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1), generator=g, dtype=torch.float64)
               / math.sqrt(k_total)).half().to(cuda) for c, t in segs]
        wp = torch.cat([ops.pack_conv_weight(wt) for wt in ws], dim=1).contiguous()
        bias = hetero((nb, cout), (0,), 1000 + seed, cuda, offset=2.0, scale=(0.5, 2.0), dtype=torch.float32).contiguous()
        ho, wo = h // stride, w // stride
        # the tail band holds every phantom image a partial last M tile can reach past the batch (< 4 tile-fulls of one image)
        out = guarded((nb * ho * wo, cout), pitch=cout + 64, device=cuda, tail=max(64, 3 * ho * wo))
        o4 = out.view.view(nb, ho, wo, cout)
        src_taps = [(x, t) for x, (_, t) in zip(srcs, segs)]
        for autotile, allow_swap in PLANS:
            info = ops.igemm_engine_plan(src_taps, wp, o4, autotile=autotile, allow_swap=allow_swap, stride=stride, colbias=bias)
            key = (tuple(t for _, t in segs), stride, ho, wo, nb, info.bn, info.splits, info.swap, info.mode)
            if key in seen:
                continue
            seen.add(key)
            out.buf.view(torch.int16).fill_(SENTINEL)   # a second plan must write every element again
            ops.igemm(src_taps, wp, o4, stride=stride, colbias=bias, bn=info.bn, splits=info.splits, swap=bool(info.swap),
                      pair=info.mode == 1)
            what = (f"{height}x{width} nb={nb} level {h}x{w} {[c for c, _ in segs]}->{cout} s{stride} bn={info.bn} "
                    f"splits={info.splits} swap={info.swap} mode={info.mode}")
            out.assert_untouched(what)
            acc = _conv(srcs, ws, stride)
            bd = bias.double()[:, None, None, :]
            ref = acc + bd
            if any(t == 9 for _, t in segs) and h != w:
                hw_swapped = _conv([x.reshape(nb, w, h, -1) for x in srcs], ws, stride).reshape(nb, ho, wo, cout) + bd
                assert_discriminates(o4, ref, hw_swapped, 4e-3, 3e-3, what, "H and W swapped")
            elif any(t == 9 for _, t in segs) and h > 1:   # square level: H and W swapped = the image transposed
                transposed = _conv([x.transpose(1, 2) for x in srcs], ws, stride).transpose(1, 2) + bd
                assert_discriminates(o4, ref, transposed, 4e-3, 3e-3, what, "H and W swapped")
            elif ho * wo > 1:   # a 1x1 contraction gives the same pixels whichever way they are laid out
                assert_discriminates(o4, ref, ref.roll(1, 2 if wo > 1 else 1), 4e-3, 3e-3, what, "pixels shifted by one")
            if nb > 1:
                assert_discriminates(o4, ref, acc + bd[:1], 4e-3, 3e-3, what, "image 0's bias for every image")
                first = _conv([x[:1].expand_as(x) for x in srcs], ws, stride) + bd
                assert_discriminates(o4, ref, first, 4e-3, 3e-3, what, "image 0's input for every image")
    families = {}
    for k in seen:
        families[k[:2]] = families.get(k[:2], 0) + 1
    print(f"{height}x{width} nb={nb}: {len(seen)} cases; per (taps, stride): {families}")
    assert len(families) == 4, f"a contraction family never ran: {families}"
