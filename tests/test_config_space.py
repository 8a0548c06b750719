"""Coverage of the engine's accepted configuration space by the GPU tests, evaluated WITHOUT a GPU.

The engine accepts any stream batch T from 1 to 16 and any height and width that are multiples of 64 (b2sd_create).  Much of
what can go wrong at a configuration nobody ran is index and mask arithmetic that depends on those numbers: the implicit-GEMM
pixel tile (how many images, rows and columns one 128-row M tile holds, and which tiles are partial), the attention masks of
short or ragged token counts, the GroupNorm launch shape.  A *regime* is a coarse signature of such a decision that names the
code branch it reaches, independent of channel counts:

  * contraction (from the planner's tile shape tw x th x tn, b2sd_igemm_plan_dry at autotile 1 and 2): the tw rule -- "row"
    (Ho == Nb == 1: one row of 128 pixels / tokens), "wo" (tw = Wo <= 16), "16", "8", "16p" (16 with a partial last column
    tile) -- with "swap:" for the swapped orientation, and the flags short (< 128 rows per tile), multi (tn > 1 images per
    tile), pw / ph / pn (partial last tile in w / h / n: pn is a phantom image past the batch);
  * self-attention (from nb and the token count sq): one token, 2 to 7 tokens, per-image V^T (sq % 8 != 0 with nb > 1), a KV tail tile that
    reaches into the next image (sq % 128 != 0 with nb > 1), sq > 9216;
  * GroupNorm (from b2sd_groupnorm_plan_dry): cluster of 1 / 2 / 4 / 8 CTAs or the non-cluster kernels (cl0), hw < 8;
  * stream batch: 1 (no stream-batch state), the largest batch 16, odd and even batches in between.

The space is every side 64 .. 1024 in steps of 64 and every batch 1 .. 16, with the UNet's contraction families
(test_plan._unet_shapes, linears on tokens as the engine runs them) and the TAESD body.  Every regime it reaches must be
covered by some GPU test case: the operator-level cases (tests/test_nonsquare_gpu.py, tests/test_ops_gpu.py) and the engine
configurations (tests/test_config_space_gpu.py, the full-size launch audit).  The engine configurations alone must reach every
contraction, attention and stream-batch regime, so that the frame program around each kernel runs there too, and each
configuration of the sweep must reach one that no other engine configuration reaches, so none of them is dead weight.
tests/test_config_space_gpu.py ties this model to the real frame program: the regimes the launch audit records for a
configuration include the ones predicted here."""
from __future__ import annotations

import ctypes as C
import functools

import pytest

from ai_rtc_agent_b200.host import capi
from tests.test_plan import _desc, _unet_shapes

SD_CHS = (320, 640, 1280, 1280)
TINY_CHS = (64, 128, 256, 256)      # oracle.unet.tiny_config
SIDES = range(64, 1025, 64)
BATCHES = range(1, 17)
TC_TILES_MIN = 2 * 132   # a stride-1 TAESD conv runs the halo-tile kernel from 2 x SMs tiles of 16 x 8 pixels on (engine.cu)
ATTN_MAX = 9216          # longest self-attention sequence of the reference models' usual sizes (768 x 768, level 0)


# ---- regimes -------------------------------------------------------------------------------------------------------------------
def contraction_regime(nb, ho, wo, tw, th, tn, swap):
    if ho == 1 and nb == 1:
        rule = "row"
    elif swap:
        rule = "16" if tw == 16 else "8x8"
    elif tw == wo:
        rule = "wo"
    elif tw == 8:
        rule = "8"
    else:
        rule = "16" if wo % 16 == 0 else "16p"
    flags = [f for f, on in (("short", not swap and tw * th * tn < 128), ("multi", tn > 1), ("pw", wo % tw), ("ph", ho % th),
                             ("pn", nb % tn)) if on]
    return ("swap:" if swap else "") + "+".join([rule] + flags)


def attention_regime(nb, sq):
    tags = [t for t, on in (("sq=1", sq == 1), ("sq<8", 1 < sq < 8), ("vt-per-image", nb > 1 and sq % 8), ("kv-tail", nb > 1 and sq % 128),
                            ("long", sq > ATTN_MAX)) if on]
    return "attn:" + ("+".join(tags) or "plain")


def batch_regime(nb):
    """the stream batch (scheduler step, stream-batch state copies, per-slot time biases): one slot without state, the largest
    batch b2sd_create accepts, and odd / even batches in between"""
    return "batch:1" if nb == 1 else ("batch:16" if nb == 16 else ("batch:odd" if nb % 2 else "batch:even"))


def groupnorm_regime(ca, cb, hw):
    cl, th, ppc = C.c_int(), C.c_int(), C.c_int()
    assert capi.lib().b2sd_groupnorm_plan_dry(ca, cb, 32, hw, C.byref(cl), C.byref(th), C.byref(ppc)) == 0
    return f"gn:cl{cl.value}" + ("+hw<8" if hw < 8 else "")


def variant_prefix(flags):
    """the kernel variant of a contraction with these epilogue flags: "pad0:" (igemm_pad0_kernel, the tap origin at the output
    pixel), "silu:" (the SiLU-epilogue instantiations), "" (the plain kernels)"""
    return "pad0:" if flags & capi.IG_PAD0 else ("silu:" if flags & capi.IG_SILU else "")


@functools.lru_cache(maxsize=None)
def _planned(nb, h, w, srcs, cout, stride, geglu, allow_swap, autotile, flags=0):
    d, _ = _desc(nb, h, w, list(srcs), cout, stride=stride, geglu=geglu, flags=flags)
    info = capi.IgemmPlanInfo()
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), autotile, int(allow_swap), C.byref(info)) == 0, capi.lib().b2sd_last_error()
    return variant_prefix(flags) + contraction_regime(d.nb, d.ho, d.wo, info.tw, info.th, info.tn, info.swap)


def plan_regime(info, nb, ho, wo):
    """regime of a plan the C ABI returned (b2sd_igemm_plan_dry, or a launch record of the audit)"""
    return contraction_regime(nb, ho, wo, info.tw, info.th, info.tn, info.swap)


# ---- the frame program's families --------------------------------------------------------------------------------------------
def contraction_families(chs, nb, lh, lw, taesd=True):
    """(nb, h, w, srcs, cout, stride, geglu, allow_swap) of the UNet's contraction families (single-source 1x1 families are the
    transformer's linears: the engine runs them on nb*h*w tokens), plus the TAESD body convolutions that run as implicit GEMMs
    (stride 2, and stride 1 below the halo-tile kernel's threshold) on one frame of lh*8 x lw*8."""
    out = []
    for (b, (h, w), srcs, cout, stride, geglu, allow_swap) in _unet_shapes(list(chs), nb, lh, lw):
        if len(srcs) == 1 and srcs[0][1] == 1:
            b, h, w = 1, 1, b * h * w
        out.append((b, h, w, tuple(srcs), cout, stride, geglu, allow_swap))
    if taesd:
        for k in range(4):
            h, w = lh * 8 >> k, lw * 8 >> k
            if -(-h // 16) * -(-w // 8) < TC_TILES_MIN:
                out.append((1, h, w, ((64, 9),), 64, 1, False, False))
            if k < 3:
                out.append((1, h, w, ((64, 9),), 64, 2, False, False))
    return out


def _levels(lh, lw):
    return [(lh >> k, lw >> k) for k in range(4)]


def config_regimes(chs, nb, height, width, taesd=True, autotiles=(1, 2)):
    """{"contraction": set, "attention": set, "groupnorm": set, "batch": set} an engine configuration reaches"""
    lh, lw = height // 8, width // 8
    con = {_planned(*f, a) for f in contraction_families(chs, nb, lh, lw, taesd) for a in autotiles}
    att = {attention_regime(nb, h * w) for h, w in _levels(lh, lw)}   # levels 0..2 and the mid block at level 3
    gn = set()
    for k, (h, w) in enumerate(_levels(lh, lw)):
        c, prev, nxt = chs[k], chs[max(k - 1, 0)], chs[min(k + 1, 3)]
        for ca, cb in {(prev, 0), (c, 0), (c, prev), (c, c), (c, nxt)}:   # resnet norm1 / norm2, transformer norm, up concats
            gn.add(groupnorm_regime(ca, cb, h * w))
    return {"contraction": con, "attention": att, "groupnorm": gn, "batch": {batch_regime(nb)}}


# ---- the GPU lists ---------------------------------------------------------------------------------------------------------
def _engine_entries():
    """(list, id, regimes) of every engine configuration the GPU tests run"""
    from tests import test_config_space_gpu as S
    from tests import test_launch_audit_gpu as LA
    out = []
    for lst, params in (("config sweep", S.SWEEP), ("launch audit full size", LA._FULL)):
        for p in params:
            cfg = p.values[0]
            full = lst != "config sweep" or cfg.get("full", False)
            out.append((lst, p.id, engine_regimes(cfg, full)))
    return out


def engine_regimes(cfg, full):
    """the regimes of an engine configuration of the GPU tests (dict of _engine / tests/test_launch_audit_gpu.py)"""
    h, w = (cfg["hw"], cfg["hw"]) if isinstance(cfg["hw"], int) else cfg["hw"]
    at = (2,) if cfg.get("concurrency", 1) >= 4 else (1,)
    return config_regimes(SD_CHS if full else TINY_CHS, len(cfg["tl"]), h, w, taesd=not cfg.get("kl"), autotiles=at)


def _operator_entries():
    """(list, id, regimes) of the operator-level GPU cases"""
    from tests import test_nonsquare_gpu as NS
    from tests import test_ops_gpu as O
    out = []
    for p in NS.CASES:
        height, width, chs, nb = p.values
        regs = set()
        for (h, w, segs, cout, stride) in NS._families(height // 8, width // 8, chs):
            for autotile, allow_swap in NS.PLANS:
                regs.add(_planned(nb, h, w, tuple(segs), cout, stride, False, allow_swap, autotile))
        out.append(("igemm nonsquare", p.id, {"contraction": regs}))
    for name, seqs in (("attention", [(c[0], c[2]) for c in O.SELF_ATTENTION_CASES]),
                       ("attention batch tail", [(4, sq) for sq in O.BATCH_TAIL_SEQS]),
                       ("attention padded V^T", [(O._padded_vt_batch(sq), sq) for sq in O.PADDED_VT_SEQS])):
        for nb, sq in seqs:
            out.append((name, f"nb{nb}-sq{sq}", {"attention": {attention_regime(nb, sq)}}))
    for case in O.GN_PATH_CASES:
        _, _, nb, h, w, ca, cb, _ = case
        out.append(("groupnorm paths", f"{nb}-{h}x{w}-{ca}+{cb}", {"groupnorm": {groupnorm_regime(ca, cb, h * w)}}))
    return out


def space_regimes():
    """every regime of the accepted space: SD-1.5 / SD-Turbo channels, sides 64..1024, batches 1..16, autotile 1 and 2"""
    out = {"contraction": set(), "attention": set(), "groupnorm": set(), "batch": set()}
    for height in SIDES:
        for width in SIDES:
            for nb in BATCHES:
                for k, v in config_regimes(SD_CHS, nb, height, width).items():
                    out[k] |= v
    return out


def _flat(regs):
    return {r for v in regs.values() for r in v}


def test_regime_signature():
    """the tile rules the planner picks, read back from its plan (tw / th / tn are the planner's, not restated here)"""
    def reg(nb, h, w, srcs, cout, **kw):
        d, _ = _desc(nb, h, w, srcs, cout, **kw)
        info = capi.IgemmPlanInfo()
        assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 1, 0, C.byref(info)) == 0
        return (info.tw, info.th, info.tn), plan_regime(info, d.nb, d.ho, d.wo)
    assert reg(1, 1, 4096, [(320, 1)], 320) == ((128, 1, 1), "row")
    assert reg(1, 1, 77, [(320, 1)], 320) == ((128, 1, 1), "row+pw")              # tokens of one 128-row tile, 77 valid
    assert reg(3, 8, 8, [(1280, 9)], 1280) == ((8, 8, 2), "wo+multi+pn")          # T = 3 at 512: a phantom image
    assert reg(3, 7, 7, [(1280, 9)], 1280) == ((7, 7, 2), "wo+short+multi+pn")    # T = 3 at 448
    assert reg(5, 11, 5, [(640, 9)], 640) == ((5, 11, 2), "wo+short+multi+pn")   # T = 5 at 704 x 320, level 2
    assert reg(1, 13, 13, [(1280, 9)], 1280) == ((13, 9, 1), "wo+short+ph")       # 832: 117 rows per tile
    assert reg(1, 64, 64, [(320, 9)], 320) == ((16, 8, 1), "16")
    assert reg(1, 9, 18, [(1280, 9)], 1280) == ((16, 8, 1), "16p+pw+ph")           # 576 x 1152-class: last column tile 2 wide
    assert reg(1, 24, 24, [(640, 9)], 640) == ((8, 16, 1), "8+ph")
    assert reg(1, 1, 1, [(1280, 9)], 1280) == ((128, 1, 1), "row+pw")             # 64 x 64 at the deepest level
    assert reg(4, 1, 1, [(1280, 9)], 1280) == ((1, 1, 4), "wo+short+multi")       # four 1-pixel images in one M tile
    d, _ = _desc(1, 8, 8, [(1280, 9)], 1280)
    info = capi.IgemmPlanInfo()
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 1, 1, C.byref(info)) == 0 and info.swap
    assert (info.tw, info.th, info.tn) == (8, 8, 1) and plan_regime(info, 1, 8, 8) == "swap:8x8"
    assert attention_regime(3, 1) == "attn:sq=1+vt-per-image+kv-tail"
    assert attention_regime(3, 4) == "attn:sq<8+vt-per-image+kv-tail"
    assert attention_regime(1, 16384) == "attn:long"
    assert attention_regime(4, 4096) == "attn:plain"
    assert groupnorm_regime(1280, 0, 1) == "gn:cl1+hw<8"


ENGINE_CLASSES = ("contraction", "attention", "batch")   # what the launch audit records and tests/test_config_space_gpu.py ties


def test_gpu_lists_cover_the_configuration_space():
    space = space_regimes()
    ops = _operator_entries()
    engines = _engine_entries()
    n_space = {k: len(v) for k, v in space.items()}
    print(f"\nregimes of the accepted space: {n_space}")
    covered = set().union(*(_flat(r) for _, _, r in ops + engines))
    missing = sorted(_flat(space) - covered)
    assert not missing, f"regimes no GPU test reaches: {missing}"
    # The frame program itself, not only its kernels one by one: the engine configurations (launch-audited, and the sweep's
    # also run against the oracle) together reach every contraction, attention and stream-batch regime of the space.
    def eng(regs):
        return {r for k in ENGINE_CLASSES for r in regs.get(k, ())}
    space_eng = eng(space)
    missing = sorted(space_eng - set().union(*(eng(r) for _, _, r in engines)))
    assert not missing, f"regimes no engine configuration reaches: {missing}"
    # Each configuration of the sweep earns its GPU time: a regime that no other engine configuration reaches.  (The
    # full-size audit entries are also there for frame resizing, which this model does not describe; the ControlNet, HED and
    # AutoencoderKL branches are modelled by tests/test_config_space_branches.py.)
    dead = []
    for i, (lst, name, regs) in enumerate(engines):
        others = set().union(*(eng(r) for j, (_, _, r) in enumerate(engines) if j != i))
        only = sorted((eng(regs) & space_eng) - others)
        print(f"  {lst:24s} {name:34s} only it reaches: {', '.join(only) or '-'}")
        if lst == "config sweep" and not only:
            dead.append(name)
    assert not dead, f"sweep configurations that reach no regime of their own: {dead}"
    assert len(_flat(space)) <= 80, "a regime should name a code branch, not a shape"
