"""The fp16 precision floor (tests/ulp.py) on the launches of a real frame: every contraction, attention, GroupNorm, LayerNorm,
smallconv and scheduler step of the frame program, on the activations the engine really produces.

The launch audit's machinery (tests/test_launch_audit_gpu.py: Auditor, _engine, _audit) runs the frame and its tolerance
checks; PrecisionAuditor adds, after each launch, the floor's figures per class.  References are float64.  A contraction of
more than 4096 output rows is checked on a deterministic sample of at least 4096 of them (the first and last row of every
image, the rows on each side of every 128-row tile edge, seeded random rows): their input patches are gathered and summed in
float64, which keeps the largest launches affordable without falling back to an fp32 reference.

The norm budget assumes the statistics are centred within NORM_PILOT standard deviations of the mean (ulp.norm_budget); the
table also reports, per norm launch class, the largest |mean - pilot| / std met, so the pilot is tested on real activations."""
from __future__ import annotations

import collections

import pytest
import torch

from tests import launch_ref as R
from tests import test_launch_audit_gpu as LA
from tests import ulp as U

pytestmark = pytest.mark.gpu

GAMMA = 4.0
SAMPLE = 4096
CLASSES = ("contraction", "contraction+ln", "geglu", "geglu+ln", "attention", "norm", "smallconv", "lcm_step")
# classes whose budgets are, by construction, wider than 0.05 ulp almost everywhere (the LayerNorm fold's |mu colsum| term,
# the GEGLU product, P rounded to fp16): (a) and the mean are what is checked there
MIN_WELL = {"contraction+ln": 0, "geglu": 0, "geglu+ln": 0, "attention": 0}


def sample_rows(d, device) -> torch.Tensor:
    """The output rows a large contraction is checked on (all rows when there are at most SAMPLE)."""
    rows = R.rows_of(d)
    if rows <= SAMPLE:
        return torch.arange(rows, device=device)
    per = d["ho"] * d["wo"]
    img = torch.arange(d["nb"], device=device) * per
    edges = torch.arange(0, rows, 128, device=device)
    pick = torch.cat([img, img + per - 1, edges, (edges - 1).clamp_min(0)])
    g = torch.Generator().manual_seed(rows)
    pick = torch.cat([pick, torch.randint(0, rows, (SAMPLE,), generator=g).to(device)])
    return torch.unique(pick)


def rows_acc(d, srcs, w, idx, absolute=False) -> torch.Tensor:
    """float64 sum over segments / taps / channels of src * w for the output rows idx: [len(idx), n_gemm].  Each row's input
    patch is gathered as the kernel reads it (3x3 taps around stride * (y, x), zero outside the image; pad0: taps at
    stride * (y, x) + (dy, dx), zero past the last row / column)."""
    ng = R.n_gemm(d)
    W = w[:ng].double()
    if W.shape[0] < ng:
        W = torch.cat([W, W.new_zeros(ng - W.shape[0], W.shape[1])])
    if absolute:
        W = W.abs()
    per = d["ho"] * d["wo"]
    b, rem = idx // per, idx % per
    y, x = rem // d["wo"], rem % d["wo"]
    st = d["stride"]
    org = 0 if d["flags"] & R.IG_PAD0 else -1
    out = torch.zeros(len(idx), ng, dtype=torch.float64, device=idx.device)
    for s, k0, nt, c in R.k_segments(d):
        X = srcs[s]
        n, h, wd, _ = X.shape
        if nt == 1:
            if d["nb"] * d["ho"] == 1 and n * h == 1:   # Linear over tokens
                p = X.reshape(-1, c)[x].double()
            else:
                p = X[b, y * st, x * st].double()
        else:
            taps = []
            for dy in range(3):
                for dx in range(3):
                    iy, ix = y * st + dy + org, x * st + dx + org
                    ok = ((iy >= 0) & (iy < h) & (ix >= 0) & (ix < wd)).double()[:, None]
                    taps.append(X[b, iy.clamp(0, h - 1), ix.clamp(0, wd - 1)].double() * ok)
            p = torch.stack(taps, 1).reshape(len(idx), 9 * c)
        if absolute:
            p = p.abs()
        out += p @ W[:, k0:k0 + nt * c].T
    return out


class PrecisionAuditor(LA.Auditor):
    def __init__(self):
        super().__init__()
        self.floor = collections.defaultdict(U.FloorAccumulator)
        self.pilot = collections.defaultdict(float)   # norm: the largest |mean - pilot| / std

    def _after_igemm(self, rec, kind, label, s):
        super()._after_igemm(rec, kind, label, s)
        d = R.as_dict(rec.igemm)
        cls = LA._kind_class(kind, d)
        rows, ng, nv = R.rows_of(d), R.n_gemm(d), d["n_valid"]
        c_main = d["col2"] if d["out2"] else nv
        got = LA._dev(d["out"], rows, c_main, d["ldc"])
        got2 = LA._dev(d["out2"], nv - d["col2"], rows, d["ld2"]) if d["out2"] else None
        idx = sample_rows(d, got.device)
        per = d["ho"] * d["wo"]
        for img in torch.unique(idx // per).tolist():
            for part in torch.split(idx[idx // per == img], 1024):
                acc = rows_acc(d, s["src"], s["w"], part)
                S = rows_acc(d, s["src"], s["w"], part, absolute=True)
                cb = s["colbias"]
                if cb is not None and d["colbias_bstride"]:
                    cb = cb[img * d["colbias_bstride"]:img * d["colbias_bstride"] + ng]
                de = dict(d, colbias_bstride=0)
                res = s["res"][part] if s["res"] is not None else None
                rs = s["rowstat_in"][part] if s["rowstat_in"] is not None else None
                ref = R.epilogue(de, acc, cb, res, rs, s["colsum"])
                B = U.contraction_budget(de, acc, S, cb, res, rs, s["colsum"], ref, GAMMA)
                self.floor[cls].add(got[part], ref[:, :c_main], B[:, :c_main])
                if got2 is not None:
                    self.floor[cls].add(got2[:, part].T, ref[:, c_main:], B[:, c_main:])

    def _after_attn(self, rec, kind, label, s):
        super()._after_attn(rec, kind, label, s)
        a = R.as_dict(rec.attn)
        ref = R.attention_ref(a, s["q"], s["k"], s["vt"])
        pv = R.attention_ref(a, s["q"], s["k"], s["vt"].abs())          # sum_j p_j |v_j|
        got = LA._dev(a["out"], a["nb"] * a["sq"], a["heads"] * a["d_real"], a["ldo"])
        B = U.budget(pv, max(a["skv"], a["dp"]), GAMMA) + 2.0 ** -11 * pv
        self.floor["attention"].add(got, ref, B)

    def _norm(self, key, x, mean, var, gamma, beta, eps, silu, pilot, got, ref):
        rstd = 1 / torch.sqrt(var + eps)
        self.pilot[key] = max(self.pilot[key], float(((mean - pilot).abs() / var.sqrt().clamp_min(1e-30)).max()))
        B = U.budget(U.norm_budget(x, mean, rstd, gamma, beta, silu), 1, GAMMA)
        self.floor["norm"].add(got, ref, B.reshape(ref.shape))

    def _after_groupnorm(self, rec, kind, label, s):
        super()._after_groupnorm(rec, kind, label, s)
        g = R.as_dict(rec.groupnorm)
        x = s["xa"].double() if s["xb"] is None else torch.cat([s["xa"].double(), s["xb"].double()], 1)
        nb, hw, G = g["nb"], g["hw"], g["groups"]
        c = x.shape[1]
        xg = x.reshape(nb, hw, G, c // G)
        mean = xg.mean(dim=(1, 3), keepdim=True)
        var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
        pilot = xg[:, :1, :, :1]                     # the group's first channel at the image's first pixel
        ref = R.groupnorm_ref(g, s["xa"], s["xb"], s["gamma"], s["beta"])
        got = LA._dev(g["y"], nb * hw, c, g["ldy"])
        self._norm("groupnorm", xg, mean, var, s["gamma"].double().reshape(1, 1, G, -1), s["beta"].double().reshape(1, 1, G, -1),
                   g["eps"], bool(g["silu"]), pilot, got, ref)

    def _after_layernorm(self, rec, kind, label, s):
        super()._after_layernorm(rec, kind, label, s)
        l = R.as_dict(rec.layernorm)
        x = s["x"].double()
        mean, var = x.mean(1, keepdim=True), x.var(1, unbiased=False, keepdim=True)
        ref = R.layernorm_ref(l, s["x"], s["gamma"], s["beta"])
        got = LA._dev(l["y"], l["rows"], l["c"], l["ldy"])
        self._norm("layernorm", x, mean, var, s["gamma"].double()[None], s["beta"].double()[None], l["eps"], False, x[:, :1],
                   got, ref)

    def _after_smallconv(self, rec, kind, label, s):
        super()._after_smallconv(rec, kind, label, s)
        a = R.as_dict(rec.smallconv)
        rows = a["nb"] * a["h"] * a["w"]
        ref = R.smallconv_ref(a, s["x"], s["wt"], s["bias"], s["res"], s["in_off"])
        # S: the same convolution of |the transformed input| with |weights|, plus |bias| and |residual| (n = 9 cin + 2)
        v = R.smallconv_input(a, s["x"], s["in_off"]).abs().half()
        plain = {k: a[k] for k in ("nb", "h", "w", "cin", "cout", "in_h", "in_w")}
        S = R.smallconv_ref(dict(plain, flags=0), v, s["wt"].abs(), None if s["bias"] is None else s["bias"].abs(),
                            None if s["res"] is None else s["res"].abs())
        if a["flags"] & R.SC_OUT_SILU:
            S = 1.1 * S + 4 * ref.abs()
        got = LA._dev(a["y"], rows, a["cout"], a["ldy"])
        self.floor["smallconv"].add(got, ref, U.budget(S, 9 * a["cin"] + 2, GAMMA))

    def _after_lcm_step(self, rec, kind, label, s):
        super()._after_lcm_step(rec, kind, label, s)
        a = R.as_dict(rec.lcm_step)
        T, hw = a["T"], a["hw"]
        noise = s["noise"] if s["noise"] is not None else torch.zeros_like(s["x"])
        X, E, N = (t.reshape(T, hw, 4) for t in (s["x"], s["eps"], noise))
        out, xnew = R.lcm_step_ref(a, X, E, N, s["coef"])
        c = s["coef"].double().reshape(4, T)
        al, be, cs, co = (c[i][:, None, None] for i in range(4))
        S0 = (co / al).abs() * (X.double().abs() + be.abs() * E.double().abs()) + cs.abs() * X.double().abs()
        self.floor["lcm_step"].add(LA._dev(a["out_latent"], hw, 4, 4), out, U.budget(S0[T - 1], 6, GAMMA))
        if T > 1:
            Sx = al[1:].abs() * S0[:-1] + (be[1:].abs() * N.double().abs()[1:] if a["do_add_noise"] else 0.0)
            self.floor["lcm_step"].add(LA._dev(a["x"], T * hw, 4, 4).reshape(T, hw, 4)[1:], xnew[1:], U.budget(Sx, 8, GAMMA))

    def floor_table(self, name):
        lines = [f"precision floor {name}:", "  " + U.TABLE_HEADER]
        lines += ["  " + self.floor[c].stats().row(c) for c in CLASSES if c in self.floor]
        lines.append("  largest |mean - pilot| / std: " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(self.pilot.items())))
        return "\n".join(lines)


def _precision_audit(cuda, name, cfg, full, monkeypatch):
    monkeypatch.setattr(LA, "Auditor", PrecisionAuditor)
    aud = LA._audit(cuda, name, cfg, full)
    print("\n" + aud.floor_table(name))
    bad = {c: U.floor_failures(aud.floor[c].stats(), MIN_WELL.get(c, 1000)) for c in aud.floor}
    bad = {c: f for c, f in bad.items() if f}
    assert not bad, f"{name}: fp16 precision floor not met: {bad}\n{aud.floor_table(name)}"
    assert {"contraction", "attention", "norm", "smallconv", "lcm_step"} <= set(aud.floor), sorted(aud.floor)


@pytest.mark.parametrize("cfg", [pytest.param(dict(turbo=False, tl=LA._T4, hw=192), id="tiny-sd15-T4-192")])
def test_precision_audit_tiny(cuda, request, cfg, monkeypatch):
    _precision_audit(cuda, request.node.callspec.id, cfg, False, monkeypatch)


FULL = [p for p in LA._FULL if p.id in ("sd15-T4-768-c1", "turbo-T1-512-kl", "turbo-T1-1024-c8")]


@pytest.mark.parametrize("cfg", FULL)
def test_precision_audit_full_size(cuda, request, cfg, monkeypatch):
    _precision_audit(cuda, request.node.callspec.id, cfg, True, monkeypatch)
