"""The fp16 measuring stick: correct rounding of a float64 reference, the fp16 ulp at a value, signed errors in ulps, and the
per-element precision floor a kernel's fp16 output must meet.

A kernel that reads fp16 operands, accumulates in fp32 and stores fp16 has two error sources: the fp32 arithmetic, bounded
per element by a budget B (below), and the one final rounding to fp16, at most half an ulp.  The floor checks both, so it
tells a last-bit difference (a reordered fp32 sum) from a larger one (a second rounding, a truncation, a narrower
intermediate, a systematic bias), which a tolerance several ulps wide cannot.

Why not torch's cast: torch's CPU float64 -> float16 conversion goes through float32 and so rounds twice
(1 + 2^-11 + 2^-40 becomes 1.0 instead of 1 + 2^-10); round16 rounds once, on any device."""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest): the relative error of one fp32 operation
FP16_MAX = 65504.0
FP16_OVERFLOW = 65520.0   # the midpoint between 65504 and 2^16: from here on round-to-nearest-even gives inf
FP16_MIN_NORMAL = 2.0 ** -14
FP16_SUBNORMAL_ULP = 2.0 ** -24


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """float64 fp16 spacing of the binade that contains x: 2^(e-10) for |x| in [2^e, 2^(e+1)), e >= -14; 2^-24 below 2^-14
    (subnormals, and zero); 32 at and above 65504 (the last finite binade's spacing, also used beyond the overflow threshold).
    The binade comes from frexp, which is exact, so x just below a power of two gets the smaller spacing."""
    x = x.double()
    _, e = torch.frexp(x.abs())                      # |x| = m * 2^e, m in [0.5, 1): binade exponent e - 1
    e = (e - 1).clamp(-14, 15)
    u = torch.ldexp(torch.ones_like(x), e - 10)
    return torch.where(x == 0, torch.full_like(x, FP16_SUBNORMAL_ULP), u)


def round16(x: torch.Tensor) -> torch.Tensor:
    """IEEE round-to-nearest-even of float64 to fp16 in one rounding, returned as float64: ties to even, subnormals kept
    (spacing 2^-24), |x| >= 65520 -> +-inf, NaN stays NaN, the sign of zero kept."""
    x = x.double()
    u = ulp16(x)
    q = torch.round(x.abs() / u) * u                 # x / u is exact (power-of-two scaling); torch.round: half to even
    q = torch.where(q > FP16_MAX, torch.full_like(q, math.inf), q)
    return torch.copysign(q, x)


def err_ulp(got: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """(got - ref) / ulp16(ref), float64.  Where round16(ref) is +-inf the error is 0 when got is that same inf and inf
    otherwise; a got that is inf or NaN where round16(ref) is finite is an infinite error."""
    got, ref = got.double(), ref.double().to(got.device)
    r = round16(ref)
    e = (got - ref) / ulp16(ref)
    e = torch.where(torch.isinf(r), torch.where(got == r, torch.zeros_like(e), torch.full_like(e, math.inf)), e)
    return torch.where(torch.isfinite(r) & ~torch.isfinite(got), torch.full_like(e, math.inf), e)


def budget(S: torch.Tensor, n: float, gamma: float) -> torch.Tensor:
    """B = gamma * 2^-24 * sqrt(n) * S: the fp32 arithmetic error allowed in an element made of n terms whose magnitudes sum
    to S.  Each fp32 addition contributes an independent rounding of at most 2^-24 of a partial sum that is at most S, so
    the accumulated error is a random walk of standard deviation ~2^-24 * sqrt(n) * S / sqrt(3), and gamma (fixed per kernel
    class) covers the tail over ~10^6 elements and the few operations of the epilogue.  The worst case n * 2^-24 * S is
    much looser and would hide the defects the floor is there to find."""
    return gamma * U32 * math.sqrt(max(n, 1)) * S.double()


# ---- the floor ---------------------------------------------------------------------------------------------------------------
# (a) bound: |got - ref| <= 1 ulp16(ref) + B.  The kernel's fp32 value v is within B of ref and is rounded once, so
#     |got - v| <= 0.5 ulp16(v).  ulp16(v) is at most 2 ulp16(ref) (v may sit in the next binade up), hence 1 ulp + B.
#     A second rounding, a truncation or a bf16 intermediate breaks it wherever B is small.
# (b) rounding: of the well-conditioned elements (B <= 0.05 ulp16(ref)), at least 99.5 % equal round16(ref).  Such an
#     element is rounded the other way only when ref lies within its actual fp32 error (typically B / gamma) of a rounding
#     midpoint; a kernel that rounds once sees a few tenths of a percent of those.  A second rounding or a round-toward-
#     zero changes ~25 % to 50 % of them.
# (c) bias: the mean signed error is within 0.02 ulp of zero, plus 4 standard errors of the sample mean, and the rms error of
#     the well-conditioned elements is at most 0.35 ulp.  Correct rounding has mean 0 and rms 1/sqrt(12) = 0.289 (the
#     rounding error is uniform in [-0.5, 0.5] ulp); the accumulation noise of a well-conditioned element adds at most
#     ~0.03 in quadrature.  A systematic -0.25 ulp bias, or a truncation, moves the mean by 0.25 ulp or more.  References on
#     a coarse lattice (fp16 inputs far from zero, normalised) need not fill each ulp uniformly, so the rms may also reach
#     that of round16(ref) itself on the same elements plus 0.06 (0.35 - 0.289).
WELL_CONDITIONED = 0.05
MIN_CORRECTLY_ROUNDED = 0.995
MAX_MEAN = 0.02
MAX_RMS = 0.35


@dataclass
class FloorStats:
    n: int                  # elements checked
    n_well: int             # well-conditioned elements (B <= 0.05 ulp)
    rounded: float          # fraction of the well-conditioned elements equal to round16(ref)
    excess: float           # max over elements of (|got - ref| - 1 ulp - B) / ulp16(ref): <= 0 passes (a)
    mean: float             # mean signed error over all finite elements, ulps
    mean_tol: float         # what (c) allows the mean to be
    rms: float              # rms error of the well-conditioned elements, ulps
    rms_ideal: float        # rms error of round16(ref) on the same elements
    ill: float              # fraction of elements with B > 1 ulp

    def row(self, name: str) -> str:
        return (f"{name:<34} {self.n:>10d} {100 * self.rounded:>8.3f}% {self.excess:>+9.3f} {self.mean:>+8.4f} "
                f"{self.rms:>6.3f} {100 * self.ill:>6.2f}%")


TABLE_HEADER = (f"{'class':<34} {'elements':>10} {'rounded':>9} {'excess':>9} {'mean':>8} {'rms':>6} {'ill':>7}")


class FloorAccumulator:
    """Gathers the floor's figures over many launches of one class (the frame-program audit) without keeping their elements."""

    def __init__(self):
        self.n = self.n_well = self.n_fin = 0
        self.correct = 0
        self.excess = -math.inf
        self.sum_e = self.sum_e2 = self.sum_w2 = self.sum_ideal2 = 0.0
        self.n_ill = 0

    def add(self, got: torch.Tensor, ref: torch.Tensor, B) -> None:
        got = got.detach().double()
        ref = ref.detach().double().to(got.device)
        B = torch.broadcast_to(torch.as_tensor(B).detach().double().to(got.device), ref.shape).flatten()
        got, ref = got.flatten(), ref.flatten()
        u = ulp16(ref)
        r = round16(ref)
        e = err_ulp(got, ref)
        b = B / u
        infref = torch.isinf(r)
        excess = torch.where(infref, torch.where(got == r, torch.full_like(e, -1.0), torch.full_like(e, math.inf)),
                             e.abs() - 1.0 - b)
        excess = excess.nan_to_num(nan=math.inf, posinf=math.inf)
        fin = torch.isfinite(e) & ~infref
        well = fin & (b <= WELL_CONDITIONED)
        self.n += got.numel()
        self.n_well += int(well.sum())
        self.n_fin += int(fin.sum())
        self.correct += int((got[well] == r[well]).sum())
        if excess.numel():
            self.excess = max(self.excess, float(excess.max()))
        ef = e[fin]
        self.sum_e += float(ef.sum())
        self.sum_e2 += float(ef.pow(2).sum())
        self.sum_w2 += float(e[well].pow(2).sum())
        self.sum_ideal2 += float(err_ulp(r[well], ref[well]).pow(2).sum())
        self.n_ill += int((b > 1.0).sum())

    def stats(self) -> "FloorStats":
        nf, nw = max(self.n_fin, 1), max(self.n_well, 1)
        mean = self.sum_e / nf
        sd = math.sqrt(max(self.sum_e2 / nf - mean * mean, 0.0))
        return FloorStats(n=self.n, n_well=self.n_well, rounded=self.correct / nw if self.n_well else 1.0,
                          excess=self.excess if self.n else -1.0, mean=mean,
                          mean_tol=MAX_MEAN + 4.0 * sd / math.sqrt(nf), rms=math.sqrt(self.sum_w2 / nw),
                          rms_ideal=math.sqrt(self.sum_ideal2 / nw), ill=self.n_ill / max(self.n, 1))


def floor_stats(got: torch.Tensor, ref: torch.Tensor, B: torch.Tensor) -> FloorStats:
    """The figures the floor judges, for fp16 results `got` against float64 references `ref` with per-element budgets B."""
    acc = FloorAccumulator()
    acc.add(got, ref, B)
    return acc.stats()


def floor_failures(s: FloorStats, min_well: int = 1000) -> list:
    """The criteria that `s` fails, as readable strings (empty: the floor holds).  (b) and (c) need at least `min_well`
    well-conditioned elements to say anything; with fewer they are reported as failures, so a case cannot pass vacuously."""
    out = []
    if s.excess > 0:
        out.append(f"(a) an element is {s.excess:.3f} ulp beyond 1 ulp + budget")
    if s.n_well < min_well:
        out.append(f"only {s.n_well} well-conditioned elements (need {min_well})")
    else:
        if s.rounded < MIN_CORRECTLY_ROUNDED:
            out.append(f"(b) {100 * s.rounded:.3f}% correctly rounded (need {100 * MIN_CORRECTLY_ROUNDED:.1f}%)")
        if s.rms > max(MAX_RMS, s.rms_ideal + MAX_RMS - 0.289):
            out.append(f"(c) rms {s.rms:.4f} ulp (max {max(MAX_RMS, s.rms_ideal + MAX_RMS - 0.289):.4f})")
    if abs(s.mean) > s.mean_tol:
        out.append(f"(c) mean signed error {s.mean:+.4f} ulp (max {s.mean_tol:.4f})")
    return out


def assert_floor(got, ref, B, what: str, min_well: int = 1000) -> FloorStats:
    """Fail unless fp16 `got` meets the floor against float64 `ref` with per-element budget B; prints the table row."""
    s = floor_stats(got, ref, B)
    print(s.row(what))
    bad = floor_failures(s, min_well)
    assert not bad, f"{what}: fp16 precision floor not met: " + "; ".join(bad) + f"\n{TABLE_HEADER}\n{s.row(what)}"
    return s


def assert_bit_exact(got: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    """got (fp16) equals round16(ref) bit for bit (+-0 told apart only where ref is not zero)."""
    got = got.detach()
    exp = round16(ref.detach().double().to(got.device)).to(torch.float16)
    g16, e16 = got.to(torch.float16).view(torch.int16), exp.view(torch.int16)
    same = (g16 == e16) | ((got == 0) & (exp == 0))
    if not bool(same.all()):
        idx = (~same).nonzero()
        k = tuple(idx[0].tolist())
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.numel()} elements differ from round16(float64); first at "
                             f"{k}: got {got[k].item()!r}, expected {exp[k].item()!r} (reference {ref[k].item()!r})")


# ---- budgets of the normalisations ---------------------------------------------------------------------------------------
NORM_DEPTH = 128   # the norm kernels add at most ~128 terms in sequence (per-thread runs, then shuffle / shared-memory trees)
NORM_PILOT = 3.0   # |mean - pilot| / std the statistics budget allows: the pilot is one sample of the group / row


def norm_budget(x, mean, rstd, gamma, beta, silu):
    """Per-element budget, in units of 2^-24 (pass it to ulp.budget with n = 1).  x [..., c] float64; mean / rstd
    broadcastable.  The apply step (x - mu) rstd gamma + beta has terms of size |gamma| rstd (|x| + |mu|) and |beta| (three
    operations).  The statistics are sums of x - p and (x - p)^2 about a pilot p; summed NORM_DEPTH deep, their relative
    error is ~2^-24 sqrt(NORM_DEPTH) of sum (x - p)^2 = n (var + (mu - p)^2), so rstd is off by that times
    (1 + ((mu - p)/std)^2) and the mean by 2^-24 sqrt(NORM_DEPTH) |mu - p|.  A kernel that sums raw x has (mu/std)^2 in place
    of ((mu - p)/std)^2: 10^4 at 100 standard deviations, which the floor catches."""
    t = (x - mean) * rstd
    S = gamma.abs() * rstd * (x.abs() + mean.abs()) + beta.abs()
    stats = gamma.abs() * (t.abs() * (1 + NORM_PILOT ** 2) + NORM_PILOT) * math.sqrt(NORM_DEPTH)
    pre = t * gamma + beta
    if silu:
        sg = torch.sigmoid(pre)
        slope = (sg * (1 + pre * (1 - sg))).abs()
        return slope * (S * math.sqrt(3) + stats) + 4 * (pre * sg).abs()
    return S * math.sqrt(3) + stats


# ---- budgets of the contractions -------------------------------------------------------------------------------------------
def contraction_budget(d, acc, S, colbias, res, rowstat_in, colsum, ref, gamma):
    """B of a contraction's stored result [rows, n_valid], from its descriptor d (tests/launch_ref.py), its float64
    accumulator acc and the same sum over |operands| S ([rows, n_gemm]); colbias is the bias row it adds (one image's, with
    no batch stride), res / rowstat_in its rows, ref the reference.  Terms: S, |bias|, |res_scale res|, and the LayerNorm
    fold's rstd (S + |mu colsum|); GEGLU: each factor's error times the other factor (|gelu'| <= 1.13); SiLU: |silu'| <= 1.1,
    plus a few fp32 ulps of the result for expf / erff and the division."""
    from tests import launch_ref as R
    k = sum(nt * c for _, _, nt, c in R.k_segments(d))
    if colsum is not None:
        mu, rstd = R.ln_stats(rowstat_in, d["ln_c"], d["ln_eps"])
        S = rstd * (S + (mu * colsum.double()[None, :S.shape[1]]).abs())
    if colbias is not None:
        S = S + colbias.double().abs()[None, :S.shape[1]]
    if d["flags"] & R.IG_GEGLU:
        bn = d["bn"]
        pre = R.epilogue(dict(d, flags=0, acc_scale=1.0), acc, colbias, None, rowstat_in, colsum).reshape(acc.shape[0], -1, bn)
        Sv = S.reshape(acc.shape[0], -1, bn)
        half = bn // 2
        val, gate = pre[:, :, :half], pre[:, :, half:]
        S = (Sv[:, :, :half] * R.gelu_erf(gate).abs() + 1.13 * Sv[:, :, half:] * val.abs()
             + 4 * ref.reshape(val.shape).abs()).reshape(acc.shape[0], -1)
    else:
        S = S * abs(d["acc_scale"])
        if res is not None:
            S = S + abs(d["res_scale"]) * res.double().abs()
        if d["flags"] & R.IG_SILU:
            S = 1.1 * S + 4 * ref.abs()
    return budget(S, k + 3, gamma)
