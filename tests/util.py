"""Shared helpers for the parity tests."""
import math

import torch


def describe_mismatch(got: torch.Tensor, ref: torch.Tensor, tol_abs: float, tol_rel: float) -> str:
    """Compact remote-debuggable summary: error stats + where (row%8 / col%64 patterns) it is wrong."""
    got = got.float().cpu()
    ref = ref.float().cpu()
    err = (got - ref).abs()
    bad = err > (tol_abs + tol_rel * ref.abs())
    lines = [f"shape={tuple(got.shape)} max_err={err.max().item():.4g} ref_absmax={ref.abs().max().item():.4g} "
             f"bad={bad.sum().item()}/{bad.numel()} nan_got={torch.isnan(got).sum().item()}"]
    if bad.any():
        idx = bad.nonzero()
        lines.append("first bad idx: " + str(idx[:6].tolist()))
        for k in range(min(6, idx.shape[0])):
            t = tuple(idx[k].tolist())
            lines.append(f"  {t}: got={got[t].item():.5g} ref={ref[t].item():.5g}")
        flat = bad.reshape(-1, bad.shape[-1])
        rows_bad = flat.any(dim=1)
        cols_bad = flat.any(dim=0)
        lines.append(f"rows bad {rows_bad.sum().item()}/{rows_bad.numel()} cols bad {cols_bad.sum().item()}/{cols_bad.numel()}")
        rb = rows_bad.nonzero().flatten()
        cb = cols_bad.nonzero().flatten()
        lines.append("bad rows (first 24): " + str(rb[:24].tolist()))
        lines.append("bad cols (first 24): " + str(cb[:24].tolist()))
    return "\n".join(lines)


def assert_close(got, ref, tol_abs, tol_rel, what=""):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    err = (got - ref).abs()
    ok = bool((err <= tol_abs + tol_rel * ref.abs()).all()) and not bool(torch.isnan(got).any())
    assert ok, what + "\n" + describe_mismatch(got, ref, tol_abs, tol_rel)


# ---- discriminating inputs, guard bands and wrong references ------------------------------------------------------------------
def hetero(shape, dims, seed, device, offset=3.0, scale=(0.1, 4.0), dtype=torch.float16):
    """randn(shape) in which every index of the dimensions `dims` (e.g. (0, 3) = every (batch item, channel) of an NHWC tensor,
    (0,) = every row of a token matrix) gets its own offset, uniform in [-offset, offset], and its own scale, log-uniform in
    `scale`.  Each GroupNorm group, LayerNorm row and batch item then has clearly different statistics, so a kernel that applies
    the statistics of the wrong one is off by O(1) rather than by sampling noise.  Seeded, drawn on the CPU, rounded to `dtype`."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    pshape = [shape[d] if d in dims else 1 for d in range(len(shape))]
    off = (torch.rand(pshape, generator=g, dtype=torch.float64) * 2 - 1) * offset
    lo, hi = math.log(scale[0]), math.log(scale[1])
    sc = torch.exp(lo + (hi - lo) * torch.rand(pshape, generator=g, dtype=torch.float64))
    x = torch.randn(shape, generator=g, dtype=torch.float64) * sc + off
    return x.to(dtype).to(device)


def offset_heavy_rows(rows, c, device, seed=12):
    """fp16 [rows, c] whose row means are 30..100 standard deviations from zero (alternating sign, std ~1)."""
    g = torch.Generator().manual_seed(seed)
    mags = torch.linspace(30, 100, rows, dtype=torch.float64)[torch.randperm(rows, generator=g)]
    sign = torch.ones(rows, dtype=torch.float64)
    sign[1::2] = -1
    coff = 0.5 * (torch.rand((1, c), generator=g, dtype=torch.float64) * 2 - 1)
    x = (sign * mags)[:, None] + coff + torch.randn((rows, c), generator=g, dtype=torch.float64)
    return x.half().to(device)


SENTINEL = 0x7D5A   # an fp16 NaN with a payload no arithmetic produces (kernels write the canonical 0x7E00 / 0x7FFF)


class Guarded:
    """An output allocation [lead + rows + tail, pitch] filled with the SENTINEL bit pattern; `view` is the [rows, cols] window
    a kernel may write (pitch > cols leaves spare columns, as in the engine's strided buffers).  assert_untouched() checks, bit
    for bit, the bands of rows before and after the window and the spare columns [cols, pitch) of every row."""

    def __init__(self, rows, cols, pitch=None, device="cuda", lead=8, tail=64):
        pitch = cols if pitch is None else pitch
        assert pitch >= cols and pitch % 8 == 0
        self.rows, self.cols, self.pitch, self.lead = rows, cols, pitch, lead
        self.buf = torch.empty((lead + rows + tail, pitch), dtype=torch.float16, device=device)
        self.buf.view(torch.int16).fill_(SENTINEL)
        self.view = self.buf[lead:lead + rows, :cols]

    def assert_untouched(self, what=""):
        bits = self.buf.view(torch.int16)
        mask = torch.ones_like(bits, dtype=torch.bool)
        mask[self.lead:self.lead + self.rows, :self.cols] = False
        bad = (bits != SENTINEL) & mask
        if bad.any():
            idx = bad.nonzero()
            idx[:, 0] -= self.lead
            raise AssertionError(f"{what}: {int(bad.sum())} guard elements written outside the [{self.rows}, {self.cols}] window "
                                 f"(pitch {self.pitch}); first (row, col) relative to the window: {idx[:8].tolist()}")


def guarded(shape, pitch=None, device="cuda", lead=8, tail=64):
    """Guarded output for a [rows, cols] result (shape may have leading unit dimensions folded into rows)."""
    rows = math.prod(shape[:-1])
    return Guarded(rows, shape[-1], pitch, device, lead, tail)


def assert_discriminates(got, ref, wrong_ref, tol_abs, tol_rel, what="", bug=""):
    """got matches ref within tol_abs + tol_rel*|ref|, AND the plausible wrong answer `wrong_ref` (the result a kernel with the
    named bug would produce, built in plain torch) is off from ref by at least 10x that tolerance somewhere.  The second half
    proves the test would fail on that bug without planting the bug in a kernel."""
    got = got.detach().double()
    ref = ref.detach().double().to(got.device)
    wrong = wrong_ref.detach().double().to(got.device)
    assert_close(got, ref, tol_abs, tol_rel, what)
    margin = ((wrong - ref).abs() / (tol_abs + tol_rel * ref.abs())).nan_to_num(nan=float("inf"))
    worst = margin.max().item()
    assert worst >= 10.0, (f"{what}: the wrong reference '{bug}' differs from the reference by at most {worst:.2f}x the "
                           "tolerance; the test cannot tell that bug apart")
