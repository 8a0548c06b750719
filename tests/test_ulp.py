"""The fp16 measuring stick (tests/ulp.py), without a GPU: round16 / ulp16 / err_ulp pinned bit for bit at binade edges, ties,
subnormals and the overflow threshold, and the floor shown to fail on each named wrong result while the correctly rounded
result of the same fp32 computation passes (the pattern of assert_discriminates: prove the check can fail without planting
the bug in a kernel)."""
import math

import numpy as np
import pytest
import torch

from tests import ulp as U

T = lambda *v: torch.tensor(v, dtype=torch.float64)   # noqa: E731


def bits(x: torch.Tensor) -> list:
    return x.to(torch.float16).view(torch.int16).tolist()


def test_round16_points():
    cases = [
        (1.0, 1.0), (1.0 + 2 ** -11, 1.0), (1.0 + 3 * 2 ** -11, 1.0 + 2 ** -9),                  # ties to even
        (1.0 + 2 ** -11 + 2 ** -40, 1.0 + 2 ** -10),                                            # torch's CPU cast gives 1.0
        (2047.5, 2048.0), (2048.0 + 1.0, 2048.0), (2048.0 + 3.0, 2052.0), (2049.0 + 2 ** -30, 2050.0),
        (65504.0, 65504.0), (65519.0, 65504.0), (65519.999, 65504.0), (65520.0, math.inf), (1e6, math.inf),
        (-65520.0, -math.inf), (-65519.0, -65504.0),
        (2 ** -24, 2 ** -24), (2 ** -25, 0.0), (2 ** -25 + 2 ** -60, 2 ** -24), (3 * 2 ** -25, 2 ** -23),   # subnormal ties
        (5 * 2 ** -25, 2 ** -23), (2 ** -14 - 2 ** -25, 2 ** -14), (2 ** -14 - 3 * 2 ** -26, 2 ** -14 - 2 ** -24),
        (0.0, 0.0), (-0.0, -0.0), (-(2 ** -26), -0.0),
    ]
    x = T(*[c[0] for c in cases])
    want = T(*[c[1] for c in cases])
    got = U.round16(x)
    assert torch.equal(got, want), [(a, g, w) for a, g, w in zip(x.tolist(), got.tolist(), want.tolist()) if g != w]
    assert bits(got) == bits(want)   # signed zeros included
    assert torch.isnan(U.round16(T(math.nan))).all()


def test_round16_matches_numpy_single_rounding():
    """numpy converts float64 to float16 in one rounding; round16 must agree on every binade, subnormals, ties and overflow."""
    g = torch.Generator().manual_seed(3)
    e = torch.randint(-27, 17, (200000,), generator=g).double()
    m = 1 + torch.rand(200000, generator=g, dtype=torch.float64)
    x = m * torch.pow(2.0, e) * (torch.randint(0, 2, (200000,), generator=g) * 2 - 1)
    # exact ties and near-ties at every binade, and the region around 65504 / 65520
    k = torch.randint(0, 1024, (20000,), generator=g).double()
    eb = torch.randint(-24, 16, (20000,), generator=g).double()
    ties = (2 * k + 1) * torch.pow(2.0, eb - 11)
    x = torch.cat([x, ties, ties * (1 + 2 ** -40), ties * (1 - 2 ** -40), torch.linspace(65400, 65600, 4001, dtype=torch.float64)])
    with np.errstate(over="ignore"):
        ref = torch.from_numpy(x.numpy().astype(np.float16).astype(np.float64))
    got = U.round16(x)
    bad = got != ref
    assert not bad.any(), list(zip(x[bad][:8].tolist(), got[bad][:8].tolist(), ref[bad][:8].tolist()))


def test_ulp16_points():
    cases = [
        (1.0, 2 ** -10), (1.999999, 2 ** -10), (2.0, 2 ** -9), (2047.999, 1.0), (2048.0, 2.0), (-2048.0, 2.0),
        (32767.9, 16.0), (32768.0, 32.0), (65504.0, 32.0), (65519.0, 32.0), (65520.0, 32.0), (1e9, 32.0),
        (2 ** -14, 2 ** -24), (2 ** -14 - 2 ** -30, 2 ** -24), (2 ** -20, 2 ** -24), (2 ** -24, 2 ** -24), (0.0, 2 ** -24),
        (2 ** -13 - 2 ** -40, 2 ** -24), (2 ** -13, 2 ** -23),
    ]
    got = U.ulp16(T(*[c[0] for c in cases]))
    assert got.tolist() == [c[1] for c in cases]
    # the spacing of every finite fp16 binade equals the distance to the next representable value
    h = torch.arange(0, 0x7BFF, dtype=torch.int32).to(torch.int16).view(torch.float16)
    nxt = torch.arange(1, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16)
    assert torch.equal(U.ulp16(h.double()), nxt.double() - h.double())


def test_err_ulp_points():
    got = T(1.0, 1.0 + 2 ** -10, 2048.0, math.inf, 65504.0, math.inf, -math.inf, math.nan, 0.0)
    ref = T(1.0, 1.0, 2049.0, 7e4, 7e4, 100.0, 7e4, 1.0, 2 ** -24)
    assert U.err_ulp(got, ref).tolist() == [0.0, 1.0, -0.5, 0.0, math.inf, math.inf, math.inf, math.inf, -1.0]


# ---- the floor fails on each named wrong result --------------------------------------------------------------------------------
def _rtz(v: torch.Tensor) -> torch.Tensor:
    """fp16 round toward zero of float64 values (saturating at 65504)."""
    u = U.ulp16(v)
    return (torch.trunc(v / u) * u).clamp(-U.FP16_MAX, U.FP16_MAX)


def _rha(v: torch.Tensor) -> torch.Tensor:
    """fp16 round to nearest, ties away from zero."""
    u = U.ulp16(v)
    r = torch.floor(v.abs() / u + 0.5) * u
    return torch.copysign(torch.where(r > U.FP16_MAX, torch.full_like(r, math.inf), r), v)


def _contraction(kind: str, seed: int = 5, n: int = 512, m: int = 256, k: int = 320):
    """A linear layer's operands (fp16 x [n, k], fp16 w [k, m], fp32 bias [m]) and its float64 reference, budget (S from the
    magnitudes, n = k + 1 terms) and fp32 accumulator (torch's CPU fp32 matmul: a real fp32 summation order).
    kind: "random" (O(1) outputs), "ties" (integer operands, outputs in [16384, 32768) where the spacing is 16 and one output
    in 16 is an exact tie), "subnormal" (outputs below 2^-14), "overflow" (outputs around 65504 / 65520)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "ties":
        x = torch.randint(-15, 16, (n, k), generator=g).half()
        w = torch.randint(-15, 16, (k, m), generator=g).half()
        bias = torch.full((m,), 24576.0)
    else:
        x = torch.randn((n, k), generator=g).half()
        w = (torch.randn((k, m), generator=g) / math.sqrt(k)).half()
        bias = torch.randn((m,), generator=g).float()
        if kind == "subnormal":
            x = (x.float() * 2 ** -9).half()
            w = (w.float() * 2 ** -9).half()
            bias = bias * 2 ** -20
        elif kind == "overflow":
            x = (x.float() * 64).half()
            w = (w.float() * 64).half()
            bias = torch.full((m,), 65504.0) - 2048.0
    ref = x.double() @ w.double() + bias.double()
    S = x.double().abs() @ w.double().abs() + bias.double().abs()
    acc = x.float() @ w.float()
    return x, w, bias, ref, U.budget(S, k + 1, 4.0), acc


def _wrong_results(kind):
    x, w, bias, ref, B, acc = _contraction(kind)
    v = (acc + bias).double()                            # the fp32 pre-rounding value (fp32 add of the bias)
    k = x.shape[1]
    parts = [(x[:, i:i + k // 4].float() @ w[i:i + k // 4].float()).half().float() for i in range(0, k, k // 4)]
    return ref, B, U.round16(v), {
        "round toward zero": _rtz(v),
        "round half away from zero": _rha(v),
        "fp16 rounding before the bias add": U.round16(acc.half().float().double() + bias.double()),   # v in fp32 again
        "fp16 split-K partials": U.round16((sum(parts) + bias).double()),
        "bf16 intermediate": U.round16(v.float().bfloat16().double()),
        "subnormal outputs flushed to zero": torch.where(U.round16(v).abs() < U.FP16_MIN_NORMAL, torch.zeros_like(v), U.round16(v)),
        "satfinite": U.round16(v).clamp(-U.FP16_MAX, U.FP16_MAX),
        "-0.25 ulp bias": U.round16(v - 0.25 * U.ulp16(v)),
    }


# which wrong results each data set can show (e.g. a flush-to-zero only changes subnormal outputs)
DISCRIMINATES = {
    "random": ["round toward zero", "fp16 rounding before the bias add", "fp16 split-K partials", "bf16 intermediate",
               "-0.25 ulp bias"],
    "ties": ["round half away from zero", "round toward zero", "-0.25 ulp bias"],
    "subnormal": ["subnormal outputs flushed to zero", "round toward zero", "bf16 intermediate"],
    "overflow": ["satfinite"],
}


@pytest.mark.parametrize("kind", list(DISCRIMINATES))
def test_floor_passes_correct_rounding_and_fails_each_wrong_result(kind):
    ref, B, good, wrongs = _wrong_results(kind)
    s = U.floor_stats(good, ref, B)
    assert not U.floor_failures(s), (kind, U.floor_failures(s), s)
    if kind == "overflow":
        assert torch.isinf(U.round16(ref)).any() and torch.isfinite(U.round16(ref)).any()
    if kind == "subnormal":
        assert (U.round16(ref).abs() < U.FP16_MIN_NORMAL).double().mean() > 0.9
    if kind == "ties":
        assert torch.equal(good, U.round16(ref)), "integer operands: the fp32 sum is exact, so the result is bit-exact"
    for name in DISCRIMINATES[kind]:
        bad = U.floor_failures(U.floor_stats(wrongs[name], ref, B))
        assert bad, f"{kind}: the floor cannot tell '{name}' from a correctly rounded result"


def test_bit_exact_check():
    ref = T(2049.0, 2051.0, 3 * 2 ** -25, 7e4)
    U.assert_bit_exact(torch.tensor([2048.0, 2052.0, 2 ** -23, math.inf]).half(), ref, "ties")
    with pytest.raises(AssertionError):
        U.assert_bit_exact(torch.tensor([2050.0, 2052.0, 2 ** -23, math.inf]).half(), ref, "half away")
    with pytest.raises(AssertionError):
        U.assert_bit_exact(torch.tensor([2048.0, 2052.0, 2 ** -23, 65504.0]).half(), ref, "satfinite")


def _simulated_norm(x16: torch.Tensor, centred: bool) -> torch.Tensor:
    """What a GroupNorm / LayerNorm kernel stores for one group x16 (fp16 [n], gamma 1, beta 0), with fp32 statistics summed
    as the kernels sum them: 32-term runs per thread, then a tree; of x - x[0] (centred) or of raw x."""
    x = x16.float()
    p = x[0] if centred else torch.zeros((), dtype=torch.float32)
    d = (x - p).reshape(-1, 32)
    s = torch.zeros(d.shape[0], dtype=torch.float32)
    q = torch.zeros_like(s)
    for i in range(32):
        s, q = s + d[:, i], q + d[:, i] * d[:, i]
    n = float(x.numel())
    m = s.sum() / n
    rstd = torch.rsqrt(torch.clamp_min(q.sum() / n - m * m, 0.0) + 1e-5)
    return ((x - (p + m)) * rstd).half()


@pytest.mark.parametrize("ratio", [0, 10, 100])
def test_floor_fails_uncentred_norm_statistics(ratio):
    """The single-pass E[x^2] - mean^2 of raw fp32 sums (what every GroupNorm path and layernorm_kernel computed before
    their statistics were centred on a pilot) loses ~(mean/std)^2 of fp32's precision: the floor fails it from 10 standard
    deviations on, and passes the centred computation."""
    g = torch.Generator().manual_seed(9)
    x = (ratio + torch.randn(10240, generator=g, dtype=torch.float64)).half()
    xd = x.double()
    mean, rstd = xd.mean(), 1 / torch.sqrt(xd.var(unbiased=False) + 1e-5)
    ref = (xd - mean) * rstd
    one, zero = torch.ones(()), torch.zeros(())
    B = U.budget(U.norm_budget(xd, mean, rstd, one.double(), zero.double(), False), 1, 4.0)
    min_well = 1000 if ratio < 100 else 0
    assert not U.floor_failures(U.floor_stats(_simulated_norm(x, True), ref, B), min_well)
    bad = U.floor_failures(U.floor_stats(_simulated_norm(x, False), ref, B), min_well)
    assert bool(bad) == (ratio >= 10), bad
