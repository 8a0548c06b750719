"""A handful of representative launches for `ncu --set full` (one GPU, short)."""
import math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ai_rtc_agent_b200.host import ops
dev = torch.device("cuda:0")
torch.manual_seed(0)
def rnd(*s, scale=1.0): return (torch.randn(*s, device=dev) * scale).half()
which = sys.argv[1:] or ["taesd", "tconv", "unet64", "unet64bn160", "unet64pair", "unet32pair", "unet16", "geglu", "attn", "gn"]
for rep in range(2):
    if "taesd" in which:   # TAESD 512^2 64->64 conv + bias + relu + residual
        x = rnd(1, 512, 512, 64); w = ops.pack_conv_weight(rnd(64, 64, 3, 3, scale=1/24)); b = torch.randn(1, 64, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, relu=True, res=x)
    if "tconv" in which:   # the same convolution through the persistent halo-tile kernel (resident weights)
        x = rnd(1, 512, 512, 64); w = ops.pack_conv_weight(rnd(64, 64, 3, 3, scale=1/24)); b = torch.randn(1, 64, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, relu=True, res=x, tconv=True)
    if "unet64bn160" in which:  # UNet 64^2 320->320 resnet conv as the engine plans it: 160-wide tiles + cluster split-K 4
        x = rnd(1, 64, 64, 320); w = ops.pack_conv_weight(rnd(320, 320, 3, 3, scale=1/54)); b = torch.randn(1, 320, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, bn=160, splits=4)
    if "unet64pair" in which:   # ... and as the throughput policy plans it: CTA pairs (2-CTA clusters), 160-wide tiles, no split-K
        x = rnd(1, 64, 64, 320); w = ops.pack_conv_weight(rnd(320, 320, 3, 3, scale=1/54)); b = torch.randn(1, 320, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, bn=160, pair=True)
    if "unet32pair" in which:   # UNet 32^2 1280->640 (up block, K = 11520) on CTA pairs
        x = rnd(1, 32, 32, 1280); w = ops.pack_conv_weight(rnd(640, 1280, 3, 3, scale=1/107)); b = torch.randn(1, 640, device=dev)
        y = torch.empty(1, 32, 32, 640, device=dev, dtype=torch.float16); ops.igemm([(x, 9)], w, y, colbias=b, bn=160, pair=True)
    if "geglu" in which:   # 64^2 GEGLU feed-forward: 4096 x 2560 x 320, persistent over M tiles
        x = rnd(1, 1, 4096, 320); w = rnd(2560, 320, scale=1/18); b = torch.randn(1, 2560, device=dev)
        y = torch.empty(1, 1, 4096, 1280, device=dev, dtype=torch.float16); ops.igemm([(x, 1)], w, y, colbias=b, geglu=True, bn=128, n_valid=1280)
    if "unet64" in which:  # UNet 64^2 320->320 resnet conv
        x = rnd(1, 64, 64, 320); w = ops.pack_conv_weight(rnd(320, 320, 3, 3, scale=1/54)); b = torch.randn(1, 320, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, bn=64)
    if "unet16" in which:  # UNet 16^2 1280->1280 conv, split-K 4
        x = rnd(1, 16, 16, 1280); w = ops.pack_conv_weight(rnd(1280, 1280, 3, 3, scale=1/107)); b = torch.randn(1, 1280, device=dev)
        y = torch.empty_like(x); ops.igemm([(x, 9)], w, y, colbias=b, bn=64, splits=4)
    if "attn" in which:    # 64^2 self-attention, 5 heads x 64
        qk = rnd(4096, 640); vt = rnd(320, 4096); o = torch.empty(4096, 320, device=dev, dtype=torch.float16)
        ops.attention(qk[:, :320], qk[:, 320:], vt, o, nb=1, heads=5, sq=4096, skv=4096, d_real=64, dp=64, k_bstride=4096, vt_bstride=4096)
    if "gn" in which:
        x = rnd(1, 64, 64, 320); g = torch.ones(320, device=dev); bb = torch.zeros(320, device=dev); y = torch.empty_like(x)
        ops.groupnorm(x, None, g, bb, y)
    torch.cuda.synchronize()
print("done")
