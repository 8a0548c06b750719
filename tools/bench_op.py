"""Event-timed micro-benchmarks of individual launches (L2-warm, 50 iterations each)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ai_rtc_agent_b200.host import ops
dev = torch.device("cuda:0")
torch.manual_seed(0)
def rnd(*s, scale=1.0): return (torch.randn(*s, device=dev) * scale).half()
def timeit(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1000
def timeit_graph(fn, n):
    """n calls captured into one CUDA graph (no host planning/launch cost in the timed region)"""
    for _ in range(3): fn()
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g, stream=st):
            for _ in range(n): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3): g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (3 * n) * 1000
def conv_case(nb, h, w, cin, cout, bn, splits, res=False, relu=False):
    x = rnd(nb, h, w, cin); wt = ops.pack_conv_weight(rnd(cout, cin, 3, 3, scale=(9*cin) ** -0.5)); b = torch.randn(1, cout, device=dev)
    y = torch.empty(nb, h, w, cout, device=dev, dtype=torch.float16)
    if splits > 1:
        nfl = ops.capi.lib().b2sd_igemm_partial_floats(splits, nb*h*w, cout)
    us = timeit(lambda: ops.igemm([(x, 9)], wt, y, colbias=b, bn=bn, splits=splits, res=x if res else None, relu=relu))
    fl = 2.0 * nb * h * w * cout * cin * 9
    print(f"conv {nb}x{h}x{w} {cin}->{cout} bn={bn} splits={splits}: {us:8.1f} us  {fl/us/1e6:7.1f} TF/s")

def conv_cold(nb, h, w, cin, cout, bn, splits, swap, taps=9, res=True, pair=False):
    """weights rotate over > 2x L2 so every launch streams them from HBM like the real frame does"""
    wbytes = cout * cin * taps * 2
    ncopy = max(2, min(64, int(300e6 // wbytes) + 1))
    x = rnd(nb, h, w, cin)
    if taps == 9: wts = [ops.pack_conv_weight(rnd(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)) for _ in range(ncopy)]
    else: wts = [rnd(cout, cin, scale=cin ** -0.5) for _ in range(ncopy)]
    b = torch.randn(1, cout, device=dev); r = rnd(nb, h, w, cout) if res else None
    y = torch.empty(nb, h, w, cout, device=dev, dtype=torch.float16)
    it = [0]
    def fn():
        it[0] += 1
        ops.igemm([(x, taps)], wts[it[0] % ncopy], y, colbias=b, bn=bn, splits=splits, res=r, swap=swap, pair=pair)
    us = timeit_graph(fn, 2 * ncopy)
    fl = 2.0 * nb * h * w * cout * cin * taps
    print(f"{'swap' if swap else ('pair' if pair else 'base')} taps={taps} {nb}x{h}x{w} {cin}->{cout} bn={bn} splits={splits}: {us:8.1f} us  {fl/us/1e6:7.1f} TF/s  {wbytes/us/1e3:7.1f} GB/s(w)", flush=True)
if "gn" in sys.argv:
    for args in [(1, 64, 64, 320), (1, 64, 64, 640, 320), (1, 64, 64, 320, 320), (1, 32, 32, 640), (1, 32, 32, 1280, 640), (1, 16, 16, 1280), (1, 16, 16, 1280, 1280), (1, 8, 8, 1280, 1280), (4, 64, 64, 320)]:
        xa = rnd(*args[:4]); cb = args[4] if len(args) > 4 else 0; xb = rnd(args[0], args[1], args[2], cb) if cb else None
        c = args[3] + cb; g = torch.ones(c, device=dev); b = torch.zeros(c, device=dev); y = torch.empty(args[0], args[1], args[2], c, device=dev, dtype=torch.float16)
        print(f"groupnorm {args}: {timeit_graph(lambda: ops.groupnorm(xa, xb, g, b, y), 20):7.2f} us per launch (chain of 20 in a graph)", flush=True)
    sys.exit(0)
if "pairsweep" in sys.argv:
    # CTA pairs (2-CTA clusters, multicast weight tile) against the single-CTA kernel, same tile / split-K, weights streamed from HBM
    print("B2_STAGE_KB =", os.environ.get("B2_STAGE_KB", "default"))
    for (h, cin, cout, taps) in [(64, 320, 320, 9), (64, 640, 320, 9), (64, 960, 320, 9), (64, 320, 320, 1), (64, 320, 1280, 1), (64, 1280, 320, 1),
                                 (32, 640, 640, 9), (32, 1280, 640, 9), (32, 1920, 640, 9), (32, 640, 640, 1), (32, 2560, 640, 1),
                                 (16, 1280, 1280, 9), (16, 2560, 1280, 9), (16, 1280, 1280, 1), (16, 5120, 1280, 1)]:
        mt = (h * h + 127) // 128
        for bn in [64, 128, 160, 256]:
            if cout % bn: continue
            for sp in [1, 2, 4]:
                ctas = mt * (cout // bn) * sp
                if ctas > 600 or ctas < 32 or sp * 4 > cin * taps // 64: continue
                for pair in (False, True):
                    try: conv_cold(1, h, h, cin, cout, bn, sp, False, taps, pair=pair)
                    except Exception as e: print("fail", h, cin, cout, bn, sp, pair, str(e)[:80])
    sys.exit(0)
if "tilesweep" in sys.argv:
    print("B2_STAGE_KB =", os.environ.get("B2_STAGE_KB", "default"))
    for (h, cin, cout, taps) in [(64, 320, 320, 9), (64, 640, 320, 9), (64, 960, 320, 9), (64, 320, 320, 1), (64, 1280, 320, 1),
                                 (32, 640, 640, 9), (32, 1280, 640, 9), (32, 640, 640, 1), (32, 2560, 640, 1),
                                 (16, 1280, 1280, 9), (16, 2560, 1280, 9), (16, 1280, 1280, 1), (16, 5120, 1280, 1), (8, 1280, 1280, 9)]:
        mt = (h * h + 127) // 128
        for bn in [64, 128, 160, 256]:
            if cout % bn: continue
            for sp in [1, 2, 4, 8]:
                ctas = mt * (cout // bn) * sp
                if ctas > 320 or ctas < 48 or sp * 4 > cin * taps // 64: continue
                try: conv_cold(1, h, h, cin, cout, bn, sp, False, taps)
                except Exception as e: print("fail", h, cin, cout, bn, sp, str(e)[:80])
    sys.exit(0)
if "boundstudy" in sys.argv:
    print("B2_DBG_MODE =", os.environ.get("B2_DBG_MODE", "0"), "(0 normal, 1 no TMA after first ring pass, 2 no MMAs; needs the "
          "bound-study build: make -C ai-rtc-agent_b200/csrc boundstudy; B200SD_LIB=ai-rtc-agent_b200/libb200sd_bs.so)")
    for (h, cin, cout, taps, bn, sp, sw) in [(64, 320, 320, 9, 64, 1, False), (64, 320, 320, 9, 160, 1, False), (64, 320, 320, 9, 128, 1, True), (64, 320, 320, 9, 256, 2, True),
                                             (32, 640, 640, 9, 64, 2, False), (32, 640, 640, 9, 256, 4, True),
                                             (16, 1280, 1280, 9, 64, 4, False), (16, 1280, 1280, 9, 256, 8, True), (16, 1280, 1280, 9, 128, 4, True),
                                             (8, 1280, 1280, 9, 64, 8, False), (8, 1280, 1280, 9, 64, 8, True),
                                             (64, 320, 320, 1, 64, 1, False), (16, 1280, 1280, 1, 64, 4, False), (16, 1280, 1280, 1, 128, 4, True)]:
        conv_cold(1, h, h, cin, cout, bn, sp, sw, taps)
    sys.exit(0)
if "swapsweep" in sys.argv:
    for (h, cin, cout, taps) in [(64, 320, 320, 9), (64, 320, 320, 1), (64, 1280, 320, 1), (32, 640, 640, 9), (32, 640, 640, 1), (32, 2560, 640, 1),
                                 (16, 1280, 1280, 9), (16, 1280, 1280, 1), (16, 5120, 1280, 1), (8, 1280, 1280, 9), (8, 2560, 1280, 9)]:
        rows = h * h
        base = {64: [(64, 1)], 32: [(64, 2), (128, 2)], 16: [(64, 4), (128, 8)], 8: [(64, 8)]}[h]
        for bn, sp in base:
            try: conv_cold(1, h, h, cin, cout, bn, sp, False, taps)
            except Exception as e: print("fail base", h, cin, cout, bn, sp, str(e)[:80])
        sbn = 256 if rows >= 256 else 64
        for bn in ([256, 128] if rows >= 256 else [64]):
            for sp in [1, 2, 4, 8]:
                ctas = ((rows + bn - 1) // bn) * ((cout + 127) // 128) * sp
                if ctas > 320 or (ctas < 40 and sp < 8): continue
                try: conv_cold(1, h, h, cin, cout, bn, sp, True, taps)
                except Exception as e: print("fail swap", h, cin, cout, bn, sp, str(e)[:80])
    sys.exit(0)
import itertools
if "sweep" in sys.argv:
    for (h, c) in [(64, 320), (32, 640), (16, 1280), (8, 1280)]:
        for bn, sp in itertools.product([64, 128, 160, 256], [1, 2, 4, 8]):
            if c % bn: continue
            try: conv_case(1, h, h, c, c, bn, sp)
            except Exception as e: print("fail", h, c, bn, sp, str(e)[:80])
    sys.exit(0)
for args in [(1,512,512,64,64,64,1,True,True), (1,256,256,64,64,64,1,True,True), (1,64,64,320,320,64,1), (1,64,64,320,320,160,1),
             (1,32,32,640,640,64,1), (1,32,32,640,640,64,2), (1,32,32,640,640,128,2), (1,16,16,1280,1280,64,1), (1,16,16,1280,1280,64,4),
             (1,16,16,1280,1280,128,8), (1,16,16,1280,1280,256,8), (1,8,8,1280,1280,64,8), (1,8,8,1280,1280,64,16), (1,16,16,2560,1280,64,4)]:
    conv_case(*args)

def gn_case(nb, h, w, c, cb=0):
    xa = rnd(nb, h, w, c); xb = rnd(nb, h, w, cb) if cb else None
    g = torch.ones(c + cb, device=dev); b = torch.zeros(c + cb, device=dev); y = torch.empty(nb, h, w, c + cb, device=dev, dtype=torch.float16)
    us = timeit_graph(lambda: ops.groupnorm(xa, xb, g, b, y), 20)
    print(f"groupnorm {nb}x{h}x{w}x{c}+{cb}: {us:7.1f} us  ({(xa.numel() + (xb.numel() if cb else 0)) * 4 / us / 1e3:6.1f} GB/s r+w)")
def ln_case(rows, c):
    x = rnd(rows, c); g = torch.ones(c, device=dev); b = torch.zeros(c, device=dev); y = torch.empty_like(x)
    us = timeit(lambda: ops.layernorm(x, g, b, y))
    print(f"layernorm {rows}x{c}: {us:7.1f} us")
def attn_case(nb, heads, seq, skv=None):
    skv = skv or seq
    qk = rnd(nb * seq, 2 * heads * 64); vt = rnd(heads * 64, nb * max(skv, 128)); o = torch.empty(nb * seq, heads * 64, device=dev, dtype=torch.float16)
    k = qk[:, heads * 64:]
    us = timeit(lambda: ops.attention(qk[:, :heads * 64], k, vt[:, :nb * skv] if skv == seq else vt[:, :skv], o, nb=nb, heads=heads, sq=seq, skv=skv,
                                      d_real=64, dp=64, k_bstride=seq if skv == seq else 0, vt_bstride=seq if skv == seq else 0))
    fl = 4.0 * nb * heads * seq * skv * 64
    print(f"attention nb={nb} heads={heads} seq={seq} skv={skv}: {us:7.1f} us {fl/us/1e6:7.1f} TF/s")
def lin_case(m, k, n, bn=0, geglu=False):
    x = rnd(1, 1, m, k); w = rnd(n * (2 if geglu else 1), k, scale=k ** -0.5); b = torch.randn(1, n * (2 if geglu else 1), device=dev)
    y = torch.empty(1, 1, m, n, device=dev, dtype=torch.float16)
    us = timeit(lambda: ops.igemm([(x, 1)], w, y, colbias=b, bn=bn, geglu=geglu, n_valid=n))
    fl = 2.0 * m * k * n * (2 if geglu else 1)
    print(f"linear m={m} k={k} n={n} bn={bn} geglu={geglu}: {us:7.1f} us {fl/us/1e6:7.1f} TF/s")
def head_case():
    fr = torch.randint(0, 256, (1, 512, 512, 3), dtype=torch.uint8, device=dev); w = rnd(64, 3, 3, 3); b = torch.randn(64, device=dev)
    y = torch.empty(1, 512, 512, 64, device=dev, dtype=torch.float16)
    print(f"smallconv head 512x512 3->64: {timeit(lambda: ops.smallconv(fr, w, b, y, flags=1)):7.1f} us")
    x = rnd(1, 64, 64, 4); w2 = rnd(320, 4, 3, 3); b2 = torch.randn(320, device=dev); y2 = torch.empty(1, 64, 64, 320, device=dev, dtype=torch.float16)
    print(f"smallconv conv_in 64x64 4->320: {timeit(lambda: ops.smallconv(x, w2, b2, y2)):7.1f} us")
if "attnbalance" in sys.argv:
    for heads in [1, 2, 4, 5, 8, 9, 10]:
        attn_case(1, heads, 4096)
    for heads in [5, 10, 18, 20]:
        attn_case(1, heads, 1024)
    sys.exit(0)
if "all" in sys.argv or len(sys.argv) == 1:
    gn_case(1, 64, 64, 320); gn_case(1, 64, 64, 640, 320); gn_case(1, 32, 32, 640); gn_case(1, 16, 16, 1280); gn_case(1, 8, 8, 1280, 1280)
    ln_case(4096, 320); ln_case(1024, 640); ln_case(256, 1280); ln_case(64, 1280)
    attn_case(1, 5, 4096); attn_case(1, 10, 1024); attn_case(1, 20, 256); attn_case(1, 20, 64); attn_case(1, 5, 4096, 77); attn_case(1, 20, 256, 77)
    lin_case(4096, 320, 320); lin_case(4096, 320, 640); lin_case(4096, 320, 1280, 128, True); lin_case(4096, 1280, 320); lin_case(1024, 640, 640); lin_case(1024, 640, 2560, 128, True)
    lin_case(1024, 2560, 640); lin_case(256, 1280, 1280); lin_case(256, 1280, 5120, 128, True); lin_case(256, 5120, 1280); lin_case(64, 1280, 1280)
    head_case()
