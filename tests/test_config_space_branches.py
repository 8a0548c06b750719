"""Coverage of the optional branches of the frame program -- the AutoencoderKL (use_tiny_vae=False), the ControlNet and its HED
edge detector -- by the GPU tests, evaluated WITHOUT a GPU.  The method of tests/test_config_space.py, applied to the code paths
those branches reach and the UNet never does:

  * contractions (b2sd_igemm_plan_dry with the flags the engine launches them with): the tile rules of
    tests/test_config_space.py, prefixed "pad0:" for the AutoencoderKL's Downsample2D(padding=0) (igemm_pad0_kernel) and
    "silu:" for the ControlNet conditioning embedding (the SiLU-epilogue instantiations); "hed:tconv" / "hed:igemm" for HED's
    64 -> 64 conv, which switches kernels at TC_TILES_MIN tiles;
  * the AutoencoderKL mid-block attention (attn_d512_kernel, one 512-wide head over sq = H/8 * W/8 tokens): "d512:one-tile"
    (sq < 128: a single query tile, partly masked), "d512:q-tail" (sq % 128 == 64: the last query tile half masked),
    "d512:long" (sq > 9216, longer than any other sequence the tests ran before), "d512:plain";
  * GroupNorm (b2sd_groupnorm_plan_dry) with the AutoencoderKL's 4, 8 and 16 channels per group (the UNet's groups hold 10 to
    80): "gn:clN+cpgK", and "+long-chunk" when the non-cluster kernels run chunks longer than any chunk of the UNet's space;
  * HED's max-pools and hed_fuse: "+strided" when the elementwise grid (16 CTAs of 256 threads per SM) cannot cover the tensor
    in one pass and the grid-stride loop iterates, "+nonsquare" when hed_fuse's vertical and horizontal ratios differ;
  * the ControlNet's conv_in(x) + cond: one conditioning image broadcast into every stream-batch slot (smallconv residual with
    batch stride 0), "cond-res:bs0+T1" / "+odd" / "+even".

Shapes come from the oracle's restatements (oracle/autoencoder_kl.py, oracle/controlnet.py, oracle/hed.py), not from engine.cu.
The ControlNet body has the UNet's down-path shapes and runs them at the UNet's batch: tests/test_config_space.py models those.
The AutoencoderKL, HED and the conditioning embedding run one frame at a time, so only the frame's sides matter for them.

The space is every side 64 .. 1024 in steps of 64 and every stream batch 1 .. 16, with the full-size models' channels.  Every
regime it reaches must be covered by an operator case of tests/test_config_space_branches_gpu.py or by an engine configuration
(SWEEP_BRANCHES there, and the full-size launch audit's entries with these branches); the engine configurations alone must reach
every contraction, attention and batch regime, and each SWEEP_BRANCHES entry must reach one that no other engine configuration
reaches."""
from __future__ import annotations

import ctypes as C
import functools

from ai_rtc_agent_b200.host import capi
from oracle import autoencoder_kl as oakl
from oracle import controlnet as ocn
from oracle import hed as ohed
from oracle import unet as ounet
from tests import test_config_space as CS

ATTN_D512_MAX = 9216            # longest sequence the attention tests ran before this model (768 x 768)
GRID_THREADS = 132 * 16 * 256   # elementwise kernels (maxpool2x2, hed_fuse): at most 16 CTAs of 256 threads per SM
BRANCH_CLASSES = ("contraction", "attention", "groupnorm", "hed", "batch")


# ---- regimes -----------------------------------------------------------------------------------------------------------------
def d512_regime(sq):
    tags = [t for t, on in (("one-tile", sq < 128), ("q-tail", sq >= 128 and sq % 128), ("long", sq > ATTN_D512_MAX)) if on]
    return "d512:" + ("+".join(tags) or "plain")


@functools.lru_cache(maxsize=None)
def _gn_plan(ca, cb, hw):
    cl, th, ppc = C.c_int(), C.c_int(), C.c_int()
    assert capi.lib().b2sd_groupnorm_plan_dry(ca, cb, 32, hw, C.byref(cl), C.byref(th), C.byref(ppc)) == 0
    return cl.value, ppc.value


@functools.lru_cache(maxsize=None)
def unet_max_chunk():
    """the longest chunk of the non-cluster GroupNorm kernels in the UNet's space (its largest level, 1024 x 1024)"""
    out = 0
    for side in CS.SIDES:
        for k, c in enumerate(CS.SD_CHS):
            hw = (side // 8 >> k) ** 2
            for ca, cb in ((c, 0), (c, CS.SD_CHS[max(k - 1, 0)]), (c, c), (c, CS.SD_CHS[min(k + 1, 3)])):
                cl, ppc = _gn_plan(ca, cb, hw)
                if cl == 0:
                    out = max(out, ppc)
    return out


def gn_regime(c, hw):
    cl, ppc = _gn_plan(c, 0, hw)
    return f"gn:cl{cl}+cpg{c // 32}" + ("+long-chunk" if cl == 0 and ppc > unet_max_chunk() else "")


def maxpool_regime(h, w, c):
    return "hed:maxpool" + ("+strided" if (h // 2) * (w // 2) * (c // 2) > GRID_THREADS else "")


def fuse_regime(h, w):
    tags = [t for t, on in (("strided", h * w > GRID_THREADS), ("nonsquare", h != w)) if on]
    return "+".join(["hed:fuse"] + tags)


def cond_res_regime(nb):
    return "cond-res:bs0+" + ("T1" if nb == 1 else ("odd" if nb % 2 else "even"))


def hed_conv64_regime(h, w):
    return "hed:tconv" if -(-h // 16) * -(-w // 8) >= CS.TC_TILES_MIN else "hed:igemm"


# ---- the branches' families (from the oracle) ------------------------------------------------------------------------------
def kl_contractions(height, width):
    """(nb, h, w, srcs, cout, stride, geglu, allow_swap, flags) of the AutoencoderKL on one height x width frame"""
    ch, lpb = oakl.FULL.block_out_channels, oakl.FULL.layers_per_block
    out = []

    def resnet(h, w, ci, co):   # conv1; conv2 with the 1x1 shortcut as a second K segment, or the identity as a residual
        out.append((1, h, w, ((ci, 9),), co, 1, False, True, 0))
        out.append((1, h, w, ((co, 9), (ci, 1)) if ci != co else ((co, 9),), co, 1, False, True, 0))

    prev = ch[0]
    for i, c in enumerate(ch):                                   # encoder
        h, w = height >> i, width >> i
        for j in range(lpb):
            resnet(h, w, prev if j == 0 else c, c)
        if i < len(ch) - 1:
            out.append((1, h, w, ((c, 9),), c, 2, False, True, capi.IG_PAD0))
        prev = c
    lh, lw = height // 8, width // 8
    for _ in range(2):                                            # encoder and decoder mid blocks
        resnet(lh, lw, ch[-1], ch[-1])
        out.append((1, 1, lh * lw, ((ch[-1], 1),), 3 * ch[-1], 1, False, False, 0))   # [q | k | v] on the tokens
        out.append((1, 1, lh * lw, ((ch[-1], 1),), ch[-1], 1, False, False, 0))       # to_out.0
    out.append((1, lh, lw, ((ch[-1], 9),), oakl.FULL.latent_channels, 1, False, True, 0))   # conv_out (+ quant_conv)
    rev = list(reversed(ch))
    prev = rev[0]
    for i, c in enumerate(rev):                                   # decoder
        h, w = lh << i, lw << i
        for j in range(lpb + 1):
            resnet(h, w, prev if j == 0 else c, c)
        if i < len(rev) - 1:
            out.append((1, 2 * h, 2 * w, ((c, 9),), c, 1, False, True, 0))   # the conv after upsample2x
        prev = c
    out.append((1, height, width, ((rev[-1], 9),), 3, 1, False, True, 0))      # conv_out
    return out


def kl_groupnorms(height, width):
    """(channels, hw) of every GroupNorm of the AutoencoderKL"""
    ch, lpb = oakl.FULL.block_out_channels, oakl.FULL.layers_per_block
    out = set()
    prev = ch[0]
    for i, c in enumerate(ch):
        hw = (height >> i) * (width >> i)
        out |= {(prev, hw), (c, hw)}
        prev = c
    lhw = (height // 8) * (width // 8)
    out.add((ch[-1], lhw))                                        # mid blocks, attention, encoder conv_norm_out
    prev = ch[-1]
    for i, c in enumerate(reversed(ch)):
        hw = (height // 8 << i) * (width // 8 << i)
        out |= {(prev, hw), (c, hw)}
        prev = c
    out.add((ch[0], height * width))                              # decoder conv_norm_out
    return out


def hed_convs(height, width):
    """(h, w, cin, cout) of HED's twelve 3x3 convs (block 1's first conv, on the u8 frame, is a small conv)"""
    out = []
    for b, (cin, cout, n) in enumerate(ohed.BLOCKS):
        for k in range(1 if b == 0 else 0, n):
            out.append((height >> b, width >> b, cin if k == 0 else cout, cout))
    return out


def _pad64(c):
    return -(-c // 64) * 64


def embedding_contractions(height, width, c0):
    """the conditioning embedding's six SiLU convs on their 64-column padded inputs, and conv_out (no activation)"""
    e = ocn.EMBED_CHANNELS
    out, h, w = [], height, width
    for i in range(len(e) - 1):
        out.append((1, h, w, ((_pad64(e[i]), 9),), e[i], 1, False, False, capi.IG_SILU))
        out.append((1, h, w, ((_pad64(e[i]), 9),), e[i + 1], 2, False, False, capi.IG_SILU))
        h, w = h // 2, w // 2
    out.append((1, h, w, ((e[-1], 9),), c0, 1, False, False, 0))
    return out


def zero_convs(nb, lh, lw, cfg=ounet.SD15):
    """the 1x1 zero convs on the ControlNet's down features and mid block, at the stream batch, with the UNet tensor as residual"""
    ch, lpb = cfg.block_out_channels, cfg.layers_per_block
    feats = [(ch[0], 0)]
    for i, c in enumerate(ch):
        feats += [(c, i)] * lpb + ([(c, i + 1)] if i < len(ch) - 1 else [])
    assert [c for c, _ in feats] == ocn.down_residual_channels(cfg)
    feats.append((ch[-1], len(ch) - 1))
    return [(nb, lh >> k, lw >> k, ((c, 1),), c, 1, False, False, 0) for c, k in feats]


def _regimes_of(families, autotiles):
    return {CS._planned(*f[:8], a, f[8]) for f in families for a in autotiles}


def frame_branch_regimes(height, width, kl, cn, hed, autotiles=(1, 2)):
    """the regimes of the branches that run once per frame (they depend on the frame's sides only)"""
    out = {k: set() for k in BRANCH_CLASSES}
    if kl:
        out["contraction"] |= _regimes_of(kl_contractions(height, width), autotiles)
        out["groupnorm"] |= {gn_regime(c, hw) for c, hw in kl_groupnorms(height, width)}
        out["attention"].add(d512_regime((height // 8) * (width // 8)))
    if cn:
        out["contraction"] |= _regimes_of(embedding_contractions(height, width, CS.SD_CHS[0]), autotiles)
    if hed:
        convs = hed_convs(height, width)
        fams = [(1, h, w, ((ci, 9),), co, 1, False, False, 0) for h, w, ci, co in convs]
        h0, w0 = height, width
        if hed_conv64_regime(h0, w0) == "hed:tconv":   # the 64 -> 64 conv of block 1 runs on the halo-tile kernel
            fams = [f for f in fams if not (f[1] == h0 and f[3] == ((64, 9),) and f[4] == 64)]
        out["contraction"] |= _regimes_of(fams, autotiles) | {hed_conv64_regime(h0, w0)}
        out["hed"] |= {maxpool_regime(height >> k, width >> k, ohed.BLOCKS[k][1]) for k in range(len(ohed.BLOCKS) - 1)}
        out["hed"].add(fuse_regime(height, width))
    return out


def branch_regimes(nb, height, width, kl=False, cn=False, hed=False, autotiles=(1, 2)):
    out = {k: set(v) for k, v in frame_branch_regimes(height, width, kl, cn, hed, autotiles).items()}
    if cn:
        out["contraction"] |= _regimes_of(zero_convs(nb, height // 8, width // 8), autotiles)
        out["batch"].add(cond_res_regime(nb))
    return out


@functools.lru_cache(maxsize=None)
def space_branch_regimes():
    out = {k: set() for k in BRANCH_CLASSES}
    for height in CS.SIDES:
        for width in CS.SIDES:
            for k, v in frame_branch_regimes(height, width, True, True, True).items():
                out[k] |= v
            for nb in CS.BATCHES:
                out["contraction"] |= _regimes_of(zero_convs(nb, height // 8, width // 8), (1, 2))
                out["batch"].add(cond_res_regime(nb))
    return out


# ---- the GPU lists ---------------------------------------------------------------------------------------------------------
def engine_branch_regimes(cfg):
    """the branch regimes of a full-size engine configuration (dict of SWEEP_BRANCHES / the launch audit)"""
    h, w = (cfg["hw"], cfg["hw"]) if isinstance(cfg["hw"], int) else cfg["hw"]
    at = (2,) if cfg.get("concurrency", 1) >= 4 else (1,)
    return branch_regimes(len(cfg["tl"]), h, w, kl=cfg.get("kl", False), cn=cfg.get("cn", False), hed=cfg.get("hed", False),
                          autotiles=at)


def _branch_engine_entries():
    from tests import test_config_space_branches_gpu as B
    from tests import test_launch_audit_gpu as LA
    out = [("branch sweep", p.id, engine_branch_regimes(p.values[0])) for p in B.SWEEP_BRANCHES]
    out += [("launch audit full size", p.id, engine_branch_regimes(p.values[0])) for p in LA._FULL
            if any(p.values[0].get(k) for k in ("kl", "cn", "hed"))]
    return out


def _branch_operator_entries():
    from tests import test_config_space_branches_gpu as B
    out = [("attention d512", f"sq{sq}", {"attention": {d512_regime(sq)}}) for sq in B.D512_TOKENS]
    for h, w, c in B.PAD0_CASES:
        out.append(("igemm pad0", f"{h}x{w}x{c}", {"contraction": _regimes_of([(1, h, w, ((c, 9),), c, 2, False, True, capi.IG_PAD0)],
                                                                                (1, 2))}))
    for h, w, c in B.GN_CASES:
        out.append(("groupnorm", f"{h}x{w}x{c}", {"groupnorm": {gn_regime(c, h * w)}}))
    for height, width in B.HED_CASES:
        regs = {maxpool_regime(height >> k, width >> k, ohed.BLOCKS[k][1]) for k in range(len(ohed.BLOCKS) - 1)}
        out.append(("hed maxpool + fuse", f"{height}x{width}", {"hed": regs | {fuse_regime(height, width)}}))
    for height, width in B.EMBEDDING_CASES:
        out.append(("silu embedding", f"{height}x{width}",
                    {"contraction": _regimes_of([f for f in embedding_contractions(height, width, CS.SD_CHS[0]) if f[8]], (1, 2))}))
    for nb in B.COND_RES_BATCHES:
        out.append(("cond residual", f"T{nb}", {"batch": {cond_res_regime(nb)}}))
    return out


def _flat(regs):
    return {r for v in regs.values() for r in v}


def test_branch_regime_signature():
    """the new regimes read back from the planners"""
    assert d512_regime(64) == "d512:one-tile" and d512_regime(192) == "d512:q-tail" and d512_regime(4096) == "d512:plain"
    assert d512_regime(16384) == "d512:long" and d512_regime(13 * 13 * 64) == "d512:q-tail+long"   # 832 x 832
    assert unet_max_chunk() == 128                    # 16384 pixels of the 1024 x 1024 UNet in 128 chunks
    assert gn_regime(128, 1024 * 1024) == "gn:cl0+cpg4+long-chunk"     # 8192 pixels per chunk
    assert gn_regime(512, 8 * 8) == "gn:cl1+cpg16"
    assert CS._planned(1, 64, 64, ((128, 9),), 128, 2, False, True, 1, capi.IG_PAD0).startswith("pad0:")
    d, _ = CS._desc(1, 64, 64, [(64, 9)], 16, flags=capi.IG_SILU)
    info = capi.IgemmPlanInfo()
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 1, 0, C.byref(info)) == 0 and info.bn <= 128, "SiLU kernels: N tile <= 128"
    d, _ = CS._desc(1, 64, 64, [(512, 9)], 512, stride=2, flags=capi.IG_PAD0)
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 2, 1, C.byref(info)) == 0
    assert info.bn in (64, 128, 256) and info.mode == 0 and not info.swap, "pad0 kernels: single CTAs, N tile 64 / 128 / 256"
    assert hed_conv64_regime(64, 64) == "hed:igemm" and hed_conv64_regime(512, 512) == "hed:tconv"
    assert len(hed_convs(512, 512)) == 12
    assert fuse_regime(1024, 960) == "hed:fuse+strided+nonsquare" and maxpool_regime(64, 64, 64) == "hed:maxpool"


def test_gpu_lists_cover_the_branches():
    space = space_branch_regimes()
    ops = _branch_operator_entries()
    engines = _branch_engine_entries()
    unet_engines = CS._engine_entries()
    print(f"\nbranch regimes of the accepted space ({len(_flat(space))}):")
    for k in BRANCH_CLASSES:
        print(f"  {k:12s} {', '.join(sorted(space[k]))}")
    covered = set().union(*(_flat(r) for _, _, r in ops + engines + unet_engines))
    missing = sorted(_flat(space) - covered)
    assert not missing, f"branch regimes no GPU test reaches: {missing}"

    def eng(regs):
        return {r for k in CS.ENGINE_CLASSES for r in regs.get(k, ())}
    space_eng = eng(space)
    reached = set().union(*(eng(r) for _, _, r in engines + unet_engines))
    missing = sorted(space_eng - reached)
    assert not missing, f"branch regimes no engine configuration reaches: {missing}"
    unet_reached = set().union(*(eng(r) for _, _, r in unet_engines))
    dead = []
    for i, (lst, name, regs) in enumerate(engines):
        others = unet_reached.union(*(eng(r) for j, (_, _, r) in enumerate(engines) if j != i))
        only = sorted((eng(regs) & space_eng) - others)
        print(f"  {lst:24s} {name:34s} only it reaches: {', '.join(only) or '-'}")
        if lst == "branch sweep" and not only:
            dead.append(name)
    assert not dead, f"branch sweep configurations that reach no regime of their own: {dead}"
    assert len(_flat(space)) <= 80, "a regime should name a code branch, not a shape"
