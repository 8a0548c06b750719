"""Precision of the fp16-output kernels to the last fp16 place (tests/ulp.py), on top of the tolerance tests.

Exact-arithmetic cases: operands are small integers times powers of two, so every product and partial sum is exact in fp32
in any summation order (all partial sums stay below 2^24) and the stored result must equal round16(float64) bit for bit.
The contractions run with every plan the engine's planner picks at the engine's shapes, with outputs steered into
[2048, 65504) (spacing 2..32: odd sums are exact ties), the subnormal range, and across 65504 / 65520.

Floor cases: random data at the shapes and edges where kernels go wrong, judged by the per-element floor of tests/ulp.py:
bounded error, correct rounding of the well-conditioned elements, no bias."""
import math

import pytest
import torch

from tests import launch_ref as R
from tests import ulp as U
from tests.test_ops_gpu import GN_OCCUPANCY_DEPENDENT
from tests.test_plan import _desc, _plan, _unet_shapes
from tests.util import offset_heavy_rows

pytestmark = pytest.mark.gpu

SD_CHS = (320, 640, 1280, 1280)


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _ints(shape, lo, hi, seed, scale=1.0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi + 1, shape, generator=g).double() * scale).half().to(device)


# ---- exact-arithmetic contractions -------------------------------------------------------------------------------------------
# (x scale, w scale, bias): (i) outputs ~ 8192 +- a few hundred: spacing 8, odd multiples of 4 are ties; (ii) products
# int * 2^-25, outputs |sum| * 2^-25 < 2^-14: subnormal, odd sums are ties; (iii) outputs 65504 - 160 .. 65504 + 160 with
# spacing 32: finite, rounded down to 65504, exact ties at 65520 and inf beyond.
RANGES = {"ties": (1.0, 1.0, 8192.0), "subnormal": (2.0 ** -13, 2.0 ** -12, 0.0), "overflow": (1.0, 1.0, 65504.0)}


def _exact_operands(srcs_shape, k, n_rows, rng, seed):
    """integer sources (values in [-3, 3] times the range's scale), weights [n_rows, k] (integers in [-2, 2]) scaled so the
    sum of |products| stays below 2^23 / scale, and the bias"""
    xs, ws, bias = RANGES[rng]
    srcs = [_ints(s, -3, 3, seed + i, xs) for i, s in enumerate(srcs_shape)]
    # few nonzero weights per column keeps the output spread (and so |sum|) near 100 even at K = 23040
    g = torch.Generator().manual_seed(seed + 100)
    w = torch.randint(-2, 3, (n_rows, k), generator=g).double()
    keep = torch.rand((n_rows, k), generator=g) < min(1.0, 256.0 / k)
    w = (w * keep * ws).half().cuda().contiguous()
    return srcs, w, bias


def _run_exact(ops, nb, ho, wo, srcs, w, cout, stride, bias, plan, *, res=None, relu=False, pad0=False, tconv=False,
               acc_scale=1.0, res_scale=1.0):
    out = torch.full((nb, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    colbias = torch.full((1, cout), bias, dtype=torch.float32, device="cuda")
    ops.igemm(srcs, w, out, stride=stride, colbias=colbias, res=res, relu=relu, pad0=pad0, tconv=tconv, acc_scale=acc_scale,
              res_scale=res_scale, **plan)
    d = ops._igemm_desc(srcs, w, out, stride=stride, colbias=colbias, res=res, relu=relu, pad0=pad0, tconv=tconv,
                        acc_scale=acc_scale, res_scale=res_scale, **plan)
    dd = R.as_dict(d)
    acc = R.contraction_acc(dd, [t for t, _ in srcs], w)
    ref = R.epilogue(dd, acc, colbias.reshape(-1), None if res is None else res.reshape(-1, cout))
    return out.reshape(-1, cout), ref


def _planner_choices(nb, lh, lw, autotile):
    """(bn, splits, swap, pair) the host-only planner picks for every non-GEGLU contraction family at this engine size,
    from descriptors built without tensors (tests/test_plan.py)"""
    out = set()
    for b, (rh, rw), srcs_c, cout, stride, geglu, allow_swap in _unet_shapes(SD_CHS, nb, lh, lw):
        if not geglu:
            info = _plan(_desc(b, rh, rw, srcs_c, cout, stride=stride)[0], autotile, int(allow_swap))
            out.add((info.bn, info.splits, bool(info.swap), info.mode == 1))
    return out


def _engine_shapes():
    """(nb, lh, lw, autotile): the 512 x 512 engine at stream batch 1 and 4 and the 256 x 256 one, both tile policies"""
    return [(1, 64, 64, 1), (1, 64, 64, 2), (4, 32, 32, 1), (4, 32, 32, 2), (4, 16, 16, 1)]



@pytest.mark.parametrize("rng", list(RANGES))
@pytest.mark.parametrize("nb,lh,lw,autotile", _engine_shapes())
def test_exact_contraction_engine_plans(cuda, nb, lh, lw, autotile, rng):
    """Every contraction family of the SD UNet (convs, concat + shortcut segments, linears, stride-2 downsamplers) with the
    plan the engine's tile policy picks (bn, split-K, orientation, CTA pairs): bit-exact round16 of the float64 sum.  GEGLU
    (erf in the epilogue) is left to the floor cases."""
    ops = _ops()
    plans = set()
    for i, (b, (rh, rw), srcs_c, cout, stride, geglu, allow_swap) in enumerate(_unet_shapes(SD_CHS, nb, lh, lw)):
        if geglu:
            continue
        k = sum(c * t for c, t in srcs_c)
        shapes = [(b, rh, rw, c) for c, _ in srcs_c]
        srcs, w, bias = _exact_operands(shapes, k, cout, rng, 17 * i + 3)
        ho, wo = rh // stride, rw // stride
        probe = torch.empty((b, ho, wo, cout), dtype=torch.float16, device=cuda)
        info = ops.igemm_engine_plan(list(zip(srcs, [t for _, t in srcs_c])), w, probe, autotile=autotile,
                                     allow_swap=allow_swap, stride=stride,
                                     colbias=torch.zeros((1, cout), dtype=torch.float32, device=cuda))
        plan = dict(bn=info.bn, splits=info.splits, swap=bool(info.swap), pair=info.mode == 1)
        plans.add(tuple(plan.values()))
        got, ref = _run_exact(ops, b, ho, wo, list(zip(srcs, [t for _, t in srcs_c])), w, cout, stride, bias, plan)
        U.assert_bit_exact(got, ref, f"{rng}: {srcs_c} -> {cout} s{stride} at {b}x{rh}x{rw}, plan {plan}")
    print(f"nb={nb} {lh}x{lw} autotile={autotile} {rng}: plans (bn, splits, swap, pair) {sorted(plans)}")
    assert plans == _planner_choices(nb, lh, lw, autotile), "the plans run are not the planner's choices at these shapes"


# plans the engine's policy does not pick at the shapes above but the planner accepts: the other split-K factors on both
# orientations, CTA pairs with split-K, N tiles that are odd multiples of 16 (48, 80, 112, 240), and the 160 / 256 families
EXPLICIT = [
    dict(bn=48, splits=1, swap=False, pair=False), dict(bn=80, splits=2, swap=False, pair=False),
    dict(bn=112, splits=4, swap=False, pair=False), dict(bn=240, splits=1, swap=False, pair=False),
    dict(bn=64, splits=8, swap=False, pair=False), dict(bn=128, splits=2, swap=False, pair=False),
    dict(bn=256, splits=4, swap=False, pair=False), dict(bn=160, splits=1, swap=False, pair=False),
    dict(bn=64, splits=8, swap=True, pair=False), dict(bn=128, splits=2, swap=True, pair=False),
    dict(bn=256, splits=1, swap=True, pair=False), dict(bn=128, splits=4, swap=False, pair=True),
    dict(bn=160, splits=2, swap=False, pair=True), dict(bn=32, splits=1, swap=False, pair=True),
]


@pytest.mark.parametrize("rng", list(RANGES))
@pytest.mark.parametrize("plan", EXPLICIT, ids=lambda p: "bn{bn}-s{splits}{}{}".format("-swap" if p["swap"] else "",
                                                                                        "-pair" if p["pair"] else "", **p))
def test_exact_contraction_explicit_plans(cuda, plan, rng):
    """A 3x3 conv over two concatenated sources plus a 1x1 shortcut segment (1280 + 640 channels at 16 x 16, batch 2) with
    residual: bit-exact on every split-K factor, orientation, CTA pair and N tile family."""
    ops = _ops()
    nb, h, w_, cout = 2, 16, 16, 640
    srcs_c = [(1280, 9), (640, 9), (640, 1)]
    k = sum(c * t for c, t in srcs_c)
    srcs, w, bias = _exact_operands([(nb, h, w_, c) for c, _ in srcs_c], k, cout, rng, 5)
    xs = RANGES[rng][0]
    res = _ints((nb, h, w_, cout), -8, 8, 9, xs * 2.0 ** -12 if rng == "subnormal" else 1.0)
    got, ref = _run_exact(ops, nb, h, w_, list(zip(srcs, [t for _, t in srcs_c])), w, cout, 1, bias, plan, res=res)
    U.assert_bit_exact(got, ref, f"{rng}: concat + shortcut + residual, plan {plan}")


@pytest.mark.parametrize("rng", list(RANGES))
@pytest.mark.parametrize("case", ["linear", "conv-s2", "pad0", "relu-res-scaled", "tconv", "tconv-relu-res"])
def test_exact_contraction_epilogues(cuda, case, rng):
    """Linear over tokens, stride-2 3x3, the pad0 (padding after the last row / column) 3x3, ReLU with a residual under
    power-of-two acc_scale / res_scale, and the TAESD tconv kernel with its staged residual epilogue: bit-exact."""
    ops = _ops()
    kw, stride, pad0, tconv, nb, h, w_, cin, cout, ntap = {}, 1, False, False, 1, 32, 32, 320, 320, 9
    if case == "linear":
        nb, h, w_, cin, cout, ntap = 1, 1, 4096, 640, 640, 1
    elif case == "conv-s2":
        stride = 2
    elif case == "pad0":
        stride, pad0, kw = 2, True, dict(bn=128)
    elif case.startswith("tconv"):
        tconv, h, w_, cin, cout = True, 64, 64, 64, 64
    srcs, w, bias = _exact_operands([(nb, h, w_, cin)], cin * ntap, cout, rng, 11)
    ho, wo = h // stride, w_ // stride
    res, relu = None, False
    scales = {}
    if case in ("relu-res-scaled", "tconv-relu-res"):
        relu = True
        res = _ints((nb, ho, wo, cout), -8, 8, 12, RANGES[rng][0] * 2.0 ** -12 if rng == "subnormal" else 1.0)
        if case == "relu-res-scaled":
            scales = dict(acc_scale=0.5, res_scale=2.0)
    got, ref = _run_exact(ops, nb, ho, wo, [(srcs[0], ntap)], w, cout, stride, bias, kw, res=res, relu=relu, pad0=pad0,
                          tconv=tconv, **scales)
    U.assert_bit_exact(got, ref, f"{rng}: {case}")


def test_exact_transposed_v_store(cuda):
    """The fused q | k | v projection writing its V block transposed through out2 (the V^T store of the self-attention
    program), without the LayerNorm fold: q | k and V^T both bit-exact, in guarded buffers wider than their data."""
    from tests.util import guarded
    ops = _ops()
    m, c = 4096, 320
    x = _ints((1, 1, m, c), -3, 3, 1)
    w = _ints((3 * c, c), -2, 2, 2).contiguous()
    bias = torch.full((1, 3 * c), 8192.0, device=cuda)
    qk = guarded((m, 2 * c), pitch=2 * c + 64, device=cuda)
    vt = guarded((c, m), pitch=m + 64, device=cuda)
    ops.igemm([(x, 1)], w, qk.view[None, None], colbias=bias, n_valid=3 * c, out2=vt.view, col2=2 * c, bn=160)
    qk.assert_untouched("q | k")
    vt.assert_untouched("V^T")
    ref = x.double().reshape(m, c) @ w.double().t() + 8192.0
    U.assert_bit_exact(qk.view, ref[:, :2 * c], "q | k")
    U.assert_bit_exact(vt.view, ref[:, 2 * c:].t(), "V^T through out2")


def test_exact_swapped_vt_store(cuda):
    """V^T = Wv X^T with the weights on the M side (the swapped-operand store the prompt program uses): bit-exact."""
    ops = _ops()
    tokens, c = 1024, 320
    x = _ints((tokens, c), -3, 3, 1).contiguous()
    wv = _ints((1, 1, c, c), -2, 2, 2)
    out = torch.empty((1, 1, c, tokens), dtype=torch.float16, device=cuda)
    ops.igemm([(wv, 1)], x, out, bn=128, colbias=torch.full((1, tokens), 8192.0, device=cuda))
    ref = wv.double().reshape(c, c) @ x.double().t() + 8192.0
    U.assert_bit_exact(out.reshape(c, tokens), ref, "V^T swapped-operand GEMM")


@pytest.mark.parametrize("splits,pair", [(1, False), (4, False), (1, True)])
def test_exact_row_statistics(cuda, splits, pair):
    """The LayerNorm row-statistics producer: with integer outputs its int64 fixed-point sums equal sum(y) * 2^20 and
    sum(y^2) * 2^20 exactly (each fp32 partial is an exact integer below 2^24)."""
    ops = _ops()
    m, k, n = 1024, 320, 1280
    x = _ints((1, 1, m, k), -1, 1, 3)
    w = _ints((n, k), -1, 1, 4).contiguous()
    out = torch.empty((1, 1, m, n), dtype=torch.float16, device=cuda)
    st = torch.zeros((m, 2), dtype=torch.int64, device=cuda)
    ops.igemm([(x, 1)], w, out, splits=splits, pair=pair, bn=160, rowstat_out=st)
    y = out.reshape(m, n).double()
    assert torch.equal(y, x.double().reshape(m, k) @ w.double().t())
    want = torch.stack([y.sum(1), (y * y).sum(1)], 1) * R.STAT_SCALE
    assert torch.equal(st.double(), want), f"{int((st.double() != want).sum())} row sums differ"


# ---- exact attention ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("skv", [64, 256])
@pytest.mark.parametrize("d,dp", [(40, 64), (64, 64), (80, 128), (160, 192)])
@pytest.mark.parametrize("cross", [False, True])
def test_exact_attention_uniform_softmax(cuda, d, dp, skv, cross):
    """q = 0: every valid key gets P = 1, l = skv (a power of two), and the output is exactly the mean of V, so it must be
    round16 of it bit for bit.  Keys and values past skv hold poison (a large key that q = 0 ignores, values of 1000) that
    only the mask keeps out; self-attention packs three images with their own V."""
    ops = _ops()
    heads, nb = 2, 3
    sq = 128
    rows = skv + 64                                # poison rows past skv
    kimg = 1 if cross else nb
    q = torch.zeros((nb * sq, heads * dp), dtype=torch.float16, device=cuda)
    k = _ints((kimg * rows, heads * dp), -4, 4, 1)
    v = _ints((kimg, heads, rows, dp), -1000, 1000, 2)
    for b in range(kimg):
        v[b, :, skv:] = 1000.0
    v[..., d:] = 0
    vt = v.permute(1, 3, 0, 2).reshape(heads * dp, kimg * rows).contiguous()
    out = torch.full((nb * sq, heads * d), float("nan"), dtype=torch.float16, device=cuda)
    bs = 0 if cross else rows
    ops.attention(q, k, vt, out, nb=nb, heads=heads, sq=sq, skv=skv, d_real=d, dp=dp, k_bstride=bs, vt_bstride=bs)
    mean = v[:, :, :skv, :d].double().mean(2).reshape(kimg, 1, heads * d)    # [image, 1, heads * d]
    ref = mean.expand(kimg, sq, heads * d).reshape(-1, heads * d)
    if cross:
        ref = ref.repeat(nb, 1)
    U.assert_bit_exact(out, ref, f"uniform attention d={d}/{dp} skv={skv} {'cross' if cross else 'self'}")


# ---- floor cases: contractions -----------------------------------------------------------------------------------------------
GAMMA = {"contraction": 4.0, "attention": 4.0, "norm": 4.0, "elementwise": 4.0}


def _contraction_floor(ops, srcs, w, out, what, colbias=None, res=None, geglu=False, silu=False, n_valid=None, plan=None,
                       rowstat_in=None, colsum=None, ln_c=0, min_well=1000):
    """min_well = 0 where every budget is, by construction, wider than 0.05 ulp (K in the tens of thousands, cancellation,
    the folded LayerNorm's mu colsum term, the GEGLU and SiLU activations): there (a) and the mean bias are what is checked."""
    plan = plan or {}
    kw = dict(colbias=colbias, res=res, geglu=geglu, silu=silu, n_valid=n_valid, rowstat_in=rowstat_in, colsum=colsum,
              ln_c=ln_c)
    ops.igemm(srcs, w, out, **kw, **plan)
    d = R.as_dict(ops._igemm_desc(srcs, w, out, **kw, **plan))
    ts = [t for t, _ in srcs]
    acc = R.contraction_acc(d, ts, w)
    rs = None if rowstat_in is None else rowstat_in
    nv = d["n_valid"]
    cb = None if colbias is None else colbias.reshape(-1)
    rr = None if res is None else res.reshape(-1, nv)
    ref = R.epilogue(d, acc, cb, rr, rs, colsum)
    S = R.contraction_acc(d, [t.abs() for t in ts], w.abs())
    B = U.contraction_budget(d, acc, S, cb, rr, rs, colsum, ref, GAMMA["contraction"])
    got = out.reshape(-1, out.shape[-1])[:, :nv]
    return U.assert_floor(got, ref, B, what, min_well)


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def test_floor_largest_k(cuda):
    """3x3 over 2560 concatenated channels (K = 23040, the SD-1.5 up-block conv at 8 x 8) plus a 1x1 shortcut segment."""
    ops = _ops()
    xa, xb = _rand((1, 8, 8, 1280), 1).half(), _rand((1, 8, 8, 1280), 2).half()
    w = _rand((1280, 23040 + 1280), 3, 1 / math.sqrt(23040)).half().contiguous()
    out = torch.empty((1, 8, 8, 1280), dtype=torch.float16, device=cuda)
    _contraction_floor(ops, [(xa, 9), (xb, 9), (xa, 1)], w, out, "K=24320 concat conv + shortcut",
                       colbias=_rand((1, 1280), 4).float().contiguous(), min_well=0)


@pytest.mark.parametrize("splits", [1, 4])
def test_floor_cancellation(cuda, splits):
    """Outputs from heavy cancellation: x W + b with b ~ -(x W) on average, so the outputs are ~30x smaller than their terms."""
    ops = _ops()
    m, k, n = 2048, 1280, 640
    x = (_rand((1, 1, m, k), 1) + 2.0).half()
    w = _rand((n, k), 2, 1 / math.sqrt(k)).half().contiguous()
    bias = (-(x.double().reshape(m, k).mean(0) @ w.double().t())).float().reshape(1, n).contiguous()
    out = torch.empty((1, 1, m, n), dtype=torch.float16, device=cuda)
    _contraction_floor(ops, [(x, 1)], w, out, f"cancellation splits={splits}", colbias=bias, plan=dict(splits=splits),
                       min_well=0)


def test_floor_geglu(cuda):
    ops = _ops()
    m, k, inner = 2048, 320, 1280
    x = _rand((1, 1, m, k), 1).half()
    w = _rand((2 * inner, k), 2, 1 / math.sqrt(k)).half().contiguous()
    b = _rand((1, 2 * inner), 3).float().contiguous()
    out = torch.empty((1, 1, m, inner), dtype=torch.float16, device=cuda)
    _contraction_floor(ops, [(x, 1)], w, out, "GEGLU", colbias=b, geglu=True, n_valid=inner, plan=dict(bn=128), min_well=0)


def test_floor_silu(cuda):
    ops = _ops()
    x = _rand((2, 32, 32, 128), 1).half()
    w = _rand((256, 9 * 128), 2, 1 / math.sqrt(9 * 128)).half().contiguous()
    out = torch.empty((2, 32, 32, 256), dtype=torch.float16, device=cuda)
    _contraction_floor(ops, [(x, 9)], w, out, "SiLU conv", colbias=_rand((1, 256), 3).float().contiguous(), silu=True,
                       plan=dict(bn=128), min_well=0)


@pytest.mark.parametrize("geglu", [False, True])
def test_floor_layernorm_folded_offset_heavy(cuda, geglu):
    """LayerNorm folded into the consumer (rstd (x W'^T - mu colsum) + bias') over rows 30..100 standard deviations off zero."""
    ops = _ops()
    m, k = 1024, 320
    n = 2560 if geglu else 640
    x = offset_heavy_rows(m, k, cuda).reshape(1, 1, m, k)
    w = (_rand((n, k), 2, 1 / math.sqrt(k)) * (1 + 0.1 * _rand((k,), 3))[None]).half().contiguous()
    colsum = w.float().sum(1).contiguous()
    xd = x.reshape(m, k).double()
    st = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1).mul(R.STAT_SCALE).round().to(torch.int64).contiguous()
    b = _rand((1, n), 4).float().contiguous()
    out = torch.empty((1, 1, m, n // 2 if geglu else n), dtype=torch.float16, device=cuda)
    _contraction_floor(ops, [(x, 1)], w, out, f"LN-folded {'GEGLU' if geglu else 'linear'} offset-heavy", colbias=b,
                       geglu=geglu, n_valid=n // 2 if geglu else None, plan=dict(bn=128), rowstat_in=st, colsum=colsum, ln_c=k,
                       min_well=0)


# ---- floor cases: attention --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,dp", [(40, 64), (64, 64), (80, 128), (160, 192), (512, 512)])
@pytest.mark.parametrize("cross", [False, True])
def test_floor_attention(cuda, d, dp, cross):
    """Budget: the accumulation term over the d-long dot products and the skv-long P.V sum, plus 2^-11 sum_j p_j |v_j|: P is
    rounded to fp16 before P.V (DESIGN 4.4), which moves each p_j by at most 2^-11 of itself."""
    ops = _ops()
    if d == 512 and cross:
        pytest.skip("the d = 512 attention is the VAE's single-head self-attention")
    heads = 1 if d == 512 else 2
    nb, sq = 2, 1024
    skv = 77 if cross else sq
    kimg = 1 if cross else nb
    q = torch.zeros((nb * sq, heads * dp), dtype=torch.float16, device=cuda)
    k = torch.zeros((kimg * skv, heads * dp), dtype=torch.float16, device=cuda)
    for h in range(heads):
        q[:, h * dp:h * dp + d] = _rand((nb * sq, d), 1 + h).half()
        k[:, h * dp:h * dp + d] = _rand((kimg * skv, d), 3 + h).half()
    cols = -(-kimg * skv // 8) * 8
    vt = torch.zeros((heads * dp, cols), dtype=torch.float16, device=cuda)
    for h in range(heads):
        vt[h * dp:h * dp + d, :kimg * skv] = _rand((d, kimg * skv), 5 + h).half()
    vt = vt[:, :kimg * skv]
    out = torch.empty((nb * sq, heads * d), dtype=torch.float16, device=cuda)
    bs = 0 if cross else skv
    a = dict(nb=nb, heads=heads, sq=sq, skv=skv, d_real=d, dp=dp, k_bstride=bs, vt_bstride=bs)
    ops.attention(q, k, vt, out, **a)
    ref = R.attention_ref(a, q, k, vt)
    pv = R.attention_ref(a, q, k, vt.abs())          # sum_j p_j |v_j|
    B = U.budget(pv, max(skv, d), GAMMA["attention"]) + 2.0 ** -11 * pv
    # every element's budget exceeds 0.05 ulp (the P rounding term): (a) and the bias of the mean are what is checked
    U.assert_floor(out, ref, B, f"attention d={d}/{dp} {'cross' if cross else 'self'}", min_well=0)


# ---- floor cases: norms ------------------------------------------------------------------------------------------------------
SIGMAS = [0, 3, 10, 30, 100]


def _norm_min_well(ratio):
    """At 100 standard deviations the apply step's |mu| term puts nearly every budget above 0.05 ulp, so (a) and the mean
    carry the check there; (a) is what statistics summed without a pilot fail by hundreds of ulps."""
    return 1000 if ratio < 100 else 0


def _offset_groups(nb, h, w, c, ratio, seed):
    """NHWC fp16 whose groups have |mean| / std = ratio (alternating sign, std ~1)"""
    g = torch.Generator().manual_seed(seed)
    gm = (torch.randint(0, 2, (nb, 1, 1, 32, 1), generator=g).double() * 2 - 1) * ratio
    x = gm + 0.3 * torch.randn((nb, 1, 1, 32, c // 32), generator=g, dtype=torch.float64) \
        + torch.randn((nb, h, w, 32, c // 32), generator=g, dtype=torch.float64)
    return x.reshape(nb, h, w, c).half().cuda()


# (path, nb, h, w, ca, cb): cluster of 1 / 8 / 4 CTAs, fused, statistics + apply (see test_ops_gpu.GN_PATH_CASES)
GN_FLOOR_CASES = [("cluster", 1, 16, 16, 1280, 0), ("cluster", 1, 64, 64, 640, 320), ("fused", 1, 96, 96, 640, 0),
                  ("stats+apply", 1, 96, 96, 640, 320), ("cluster", 2, 32, 32, 1280, 640)]


@pytest.mark.parametrize("ratio", SIGMAS)
@pytest.mark.parametrize("path,nb,h,w,ca,cb", GN_FLOOR_CASES)
def test_floor_groupnorm(cuda, path, nb, h, w, ca, cb, ratio):
    ops = _ops()
    c = ca + cb
    x = _offset_groups(nb, h, w, c, ratio, 7)
    gamma = (1 + 0.2 * _rand((c,), 3)).float()
    beta = (0.2 * _rand((c,), 4)).float()
    for silu in (False, True):
        y = torch.full((nb, h, w, c), float("nan"), dtype=torch.float16, device=cuda)
        _, ran = ops.groupnorm(x[..., :ca].contiguous(), x[..., ca:].contiguous() if cb else None, gamma, beta, y,
                               silu=silu, return_path=True)
        g = {"nb": nb, "hw": h * w, "groups": 32, "eps": 1e-5, "silu": silu}
        xf = x.reshape(nb * h * w, c)
        ref = R.groupnorm_ref(g, xf, None, gamma, beta)
        xg = xf.double().reshape(nb, h * w, 32, c // 32)
        mean = xg.mean(dim=(1, 3), keepdim=True)
        rstd = 1 / torch.sqrt(xg.var(dim=(1, 3), unbiased=False, keepdim=True) + 1e-5)
        B = U.norm_budget(xg, mean, rstd, gamma.double().reshape(1, 1, 32, -1), beta.double().reshape(1, 1, 32, -1),
                         silu)
        U.assert_floor(y.reshape(nb * h * w, c), ref, U.budget(B.reshape(nb * h * w, c), 1, GAMMA["norm"]),
                       f"groupnorm[{ran}] {nb}x{h}x{w} {ca}+{cb} silu={silu} |mean|/std={ratio}", _norm_min_well(ratio))
    if ran != path:
        assert (path, nb, h, w, ca, cb) in GN_OCCUPANCY_DEPENDENT, f"ran the {ran} path, the planner's choice is {path}"
        pytest.skip(f"this device's occupancy selected the {ran} path, not {path} (the floor was verified)")


@pytest.mark.parametrize("ratio", SIGMAS)
@pytest.mark.parametrize("rows,c", [(4096, 320), (1024, 1280)])
def test_floor_layernorm(cuda, rows, c, ratio):
    ops = _ops()
    g = torch.Generator().manual_seed(13)
    sign = torch.ones(rows, dtype=torch.float64)
    sign[1::2] = -1
    x = (ratio * sign[:, None] + torch.randn((rows, c), generator=g, dtype=torch.float64)).half().cuda()
    gamma = (1 + 0.1 * _rand((c,), 2)).float()
    beta = (0.1 * _rand((c,), 3)).float()
    y = torch.empty_like(x)
    ops.layernorm(x, gamma, beta, y)
    ref = R.layernorm_ref({"eps": 1e-5}, x, gamma, beta)
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    B = U.norm_budget(xd, mean, rstd, gamma.double()[None], beta.double()[None], False)
    U.assert_floor(y, ref, U.budget(B, 1, GAMMA["norm"]), f"layernorm {rows}x{c} |mean|/std={ratio}", _norm_min_well(ratio))


# ---- floor cases: smallconv heads, lcm_step ----------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, 2 | 4])
def test_floor_smallconv(cuda, flags):
    """UNet conv_in (4 -> 320) and the TAESD decoder head (tanh(z/3)*3, ReLU)."""
    ops = _ops()
    z = (_rand((2, 32, 32, 4), 1) * 2).half()
    wt = _rand((320, 4, 3, 3), 2, 1 / 6.0).half()
    b = _rand((320,), 3).float()
    y = torch.empty((2, 32, 32, 320), dtype=torch.float16, device=cuda)
    ops.smallconv(z, wt, b, y, flags=flags)
    a = {"nb": 2, "h": 32, "w": 32, "cin": 4, "cout": 320, "in_h": 32, "in_w": 32, "flags": flags}
    wk = wt.permute(2, 3, 1, 0).reshape(36, 320).float()           # [tap][c] x cout
    ref = R.smallconv_ref(a, z, wk, bias=b)
    S = R.smallconv_ref(dict(a, flags=0), R.smallconv_input(a, z).abs().half(), wk.abs(), bias=b.abs())
    U.assert_floor(y.reshape(-1, 320), ref, U.budget(S, 37, GAMMA["elementwise"]), f"smallconv flags={flags}")


def test_floor_lcm_step(cuda):
    ops = _ops()
    T, h, w = 4, 64, 64
    x, eps, noise = (_rand((T, h, w, 4), s).half() for s in (1, 2, 3))
    coef = torch.tensor([0.9, 0.7, 0.5, 0.3, 0.4, 0.7, 0.85, 0.95, 0.01, 0.02, 0.05, 0.1, 0.99, 0.98, 0.95, 0.9],
                        dtype=torch.float32, device=cuda)
    x0 = x.clone()
    out = torch.empty((1, h, w, 4), dtype=torch.float16, device=cuda)
    ops.lcm_step(x0, eps, noise, coef, out)
    a = {"T": T, "do_add_noise": 1}
    f = lambda t: t.reshape(T, h * w, 4)   # noqa: E731
    ref_out, ref_x = R.lcm_step_ref(a, f(x), f(eps), f(noise), coef)
    c = coef.double().reshape(4, T)
    S0 = (c[3] / c[0])[:, None, None] * (f(x).double().abs() + c[1][:, None, None] * f(eps).double().abs()) \
        + c[2][:, None, None] * f(x).double().abs()
    Sx = S0.clone()
    Sx[1:] = c[0][1:, None, None] * S0[:-1] + c[1][1:, None, None] * f(noise).double().abs()[1:]
    U.assert_floor(out.reshape(h * w, 4), ref_out, U.budget(S0[T - 1], 6, GAMMA["elementwise"]), "lcm_step x0")
    U.assert_floor(f(x0)[1:], ref_x[1:], U.budget(Sx[1:], 8, GAMMA["elementwise"]), "lcm_step re-noised slots")


def test_exact_post_f16(cuda):
    """The float entry's tail: y * 2 - 1 in fp16 (the product is exact, the difference rounds once), NCHW, read through a
    pitch wider than 3 channels: bit-exact round16(2 y - 1)."""
    ops = _ops()
    g = torch.Generator().manual_seed(4)
    y = (torch.randn((2, 48, 40, 8), generator=g) * 0.6 + 0.5).half().cuda()
    y[0, 0, :5, 0] = torch.tensor([0.0, 2 ** -24, 0.5 + 2 ** -12, 40000.0, -40000.0], dtype=torch.float16)
    out = torch.full((2, 3, 48, 40), float("nan"), dtype=torch.float16, device=cuda)
    ops.post_f16(y, out)
    U.assert_bit_exact(out, y[..., :3].double().permute(0, 3, 1, 2) * 2 - 1, "post_f16")
