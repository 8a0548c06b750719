"""Descriptor-driven references of the frame program's launches (contractions, attention, GroupNorm, LayerNorm).

Each reference reads only a launch's descriptor (the C ABI's b2sd_igemm_desc / b2sd_attn_desc / GroupNorm and LayerNorm
arguments, as a dict of field name -> value) and snapshots of the tensors it reads, and computes what the launch must write, in
float64 (fp32 with TF32 off for the largest contractions).  The launch audit (test_launch_audit_gpu.py) checks every launch of
a real frame against them; test_launch_ref.py checks them against plain torch.nn computations.

Also here: the "wrong references" -- the result a kernel with one named bug would produce -- that prove each check could fail."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

IG_RELU, IG_GEGLU, IG_SILU, IG_PAD0, IG_TCONV, IG_PAIR = 1, 2, 8, 16, 64, 128
STAT_SCALE = float(1 << 20)   # fixed point of the LayerNorm row statistics (IG_STAT_SCALE)

# per-class tolerance (atol in units of rms(ref), rtol): the op tests' constants
TOL = {
    "contraction": (3e-3, 3e-3),
    "contraction+ln": (6e-3, 4e-3),
    "geglu+ln": (8e-3, 5e-3),
    "geglu": (3e-3, 3e-3),
    "attention": (2e-3, 4e-3),
    "norm": (3e-3, 2e-3),
}
BIG_FLOP = 20e9   # contractions above this run their reference in fp32 (TF32 off), the rest in float64


def as_dict(struct) -> dict:
    """ctypes Structure -> {field: value} (nested arrays / structures converted recursively)."""
    out = {}
    for name, _ in struct._fields_:
        v = getattr(struct, name)
        if hasattr(v, "_fields_"):
            v = as_dict(v)
        elif hasattr(v, "_length_"):
            v = [as_dict(x) if hasattr(x, "_fields_") else x for x in v]
        out[name] = v
    return out


def n_gemm(d) -> int:
    """GEMM columns of a contraction (GEGLU: value and gate columns)."""
    return 2 * d["n_valid"] if d["flags"] & IG_GEGLU else d["n_valid"]


def rows_of(d) -> int:
    return d["nb"] * d["ho"] * d["wo"]


def k_segments(d) -> List[tuple]:
    """[(segment, k0, ntap, c)] in K order."""
    segs, k0 = [], 0
    for s in range(d["nseg"]):
        c, nt = d["src"][s]["c"], d["ntap"][s]
        segs.append((s, k0, nt, c))
        k0 += nt * c
    return segs


# ---- contraction ------------------------------------------------------------------------------------------------------------
def _seg_conv(x_nhwc: torch.Tensor, wseg: torch.Tensor, ntap: int, stride: int, pad0: bool, ho: int, wo: int) -> torch.Tensor:
    """One K segment: x [N,H,W,C], wseg [n, ntap*C] in [tap][c] order -> [N, ho, wo, n]."""
    n = wseg.shape[0]
    c = x_nhwc.shape[3]
    x = x_nhwc.permute(0, 3, 1, 2)
    if ntap == 9:
        w = wseg.reshape(n, 3, 3, c).permute(0, 3, 1, 2)
        x = F.pad(x, (0, 1, 0, 1)) if pad0 else F.pad(x, (1, 1, 1, 1))
    else:
        w = wseg.reshape(n, c, 1, 1)
    y = F.conv2d(x, w, stride=stride)
    y = y[:, :, :ho, :wo]
    assert y.shape[2] == ho and y.shape[3] == wo, (tuple(y.shape), ho, wo)
    return y.permute(0, 2, 3, 1)


def contraction_acc(d, srcs: List[torch.Tensor], w: torch.Tensor, kmask: Optional[torch.Tensor] = None,
                    dtype=torch.float64) -> torch.Tensor:
    """sum over segments / taps / channels of src * w: [rows, n_gemm] in `dtype`.  srcs[s]: [N,H,W,C] of segment s;
    w: [>= 0 rows, K] packed weights (rows beyond w_rows are zero, as the TMA unit fills them); kmask: optional [K] 0/1 factor
    on the K columns (wrong references that lose part of K)."""
    ng = n_gemm(d)
    W = w[:ng].to(dtype)
    if W.shape[0] < ng:
        W = torch.cat([W, W.new_zeros(ng - W.shape[0], W.shape[1])])
    if kmask is not None:
        W = W * kmask.to(dtype)[None, :W.shape[1]]
    acc = None
    for s, k0, nt, c in k_segments(d):
        x = srcs[s].to(dtype)
        if d["nb"] * d["ho"] == 1 and nt == 1 and x.shape[0] * x.shape[1] == 1:   # Linear over tokens
            y = x.reshape(-1, c)[:d["wo"]] @ W[:, k0:k0 + c].T
        else:
            y = _seg_conv(x, W[:, k0:k0 + nt * c], nt, d["stride"], bool(d["flags"] & IG_PAD0), d["ho"], d["wo"]).reshape(-1, ng)
        acc = y if acc is None else acc + y
    return acc.double()


def ln_stats(rowstat: torch.Tensor, ln_c: int, eps: float):
    """(mean, rstd) [rows, 1] float64 from the fixed-point (sum, sum of squares) int64 [rows, 2]."""
    s = rowstat.double() / STAT_SCALE
    mu = s[:, 0:1] / ln_c
    var = (s[:, 1:2] / ln_c - mu * mu).clamp_min(0.0)
    return mu, 1.0 / torch.sqrt(var + eps)


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def epilogue(d, acc: torch.Tensor, colbias=None, res=None, rowstat_in=None, colsum=None) -> torch.Tensor:
    """acc [rows, n_gemm] -> what the launch stores, [rows, n_valid] float64 (columns >= col2 are the out2 block with out2).
    colbias: float [nb*bstride] or [n_gemm]; res [rows, n_valid]; rowstat_in int64 [rows, 2]; colsum [n_gemm]."""
    rows, ng = acc.shape
    x = acc.double()
    if colsum is not None:
        mu, rstd = ln_stats(rowstat_in, d["ln_c"], d["ln_eps"])
        x = rstd * (x - mu * colsum.double()[None, :ng])
    if colbias is not None:
        cb = colbias.double()
        if d["colbias_bstride"]:
            per_img = d["ho"] * d["wo"]
            b = torch.arange(rows, device=x.device) // per_img
            idx = b[:, None] * d["colbias_bstride"] + torch.arange(ng, device=x.device)[None, :]
            x = x + cb[idx]
        else:
            x = x + cb[None, :ng]
    if d["flags"] & IG_GEGLU:
        bn = d["bn"]
        half = bn // 2
        t = x.reshape(rows, ng // bn, bn)
        return (t[:, :, :half] * gelu_erf(t[:, :, half:])).reshape(rows, ng // 2)
    x = x * d["acc_scale"]
    if res is not None:
        x = x + d["res_scale"] * res.double()
    if d["flags"] & IG_RELU:
        x = x.clamp_min(0.0)
    if d["flags"] & IG_SILU:
        x = x * torch.sigmoid(x)
    return x


def contraction_ref(d, snap: Dict[str, torch.Tensor], kmask=None, bias0=False, stats_shift=False, no_res=False,
                    dtype=torch.float64) -> torch.Tensor:
    """The launch's stored result [rows, n_valid] from the snapshot {"src": [..], "w", "colbias", "res", "rowstat_in",
    "colsum"}.  The keyword arguments build wrong references: kmask (part of K lost), bias0 (image 0's bias for every image),
    stats_shift (the neighbouring row's LayerNorm statistics), no_res (the residual omitted)."""
    acc = contraction_acc(d, snap["src"], snap["w"], kmask, dtype)
    cb = snap.get("colbias")
    if bias0 and cb is not None:
        cb = cb[:n_gemm(d)]
        d = dict(d, colbias_bstride=0)
    rs = snap.get("rowstat_in")
    if stats_shift and rs is not None:
        rs = torch.roll(rs, 1, dims=0)
    return epilogue(d, acc, cb, None if no_res else snap.get("res"), rs, snap.get("colsum"))


def split_k_lost_mask(d, total_kb: int, kb_per_split: int, device) -> torch.Tensor:
    """[K] mask without the last cluster rank's K slice."""
    k = sum(nt * c for _, _, nt, c in k_segments(d))
    m = torch.ones(k, dtype=torch.float64, device=device)
    splits = -(-total_kb // kb_per_split)
    m[(splits - 1) * kb_per_split * 64:] = 0
    return m


def last_block_mask(d, w: torch.Tensor) -> torch.Tensor:
    """[K] mask without the last 64-wide K block whose weights are not all zero (narrow layers pad K with zero weights)."""
    k = sum(nt * c for _, _, nt, c in k_segments(d))
    W = w[:n_gemm(d), :k]
    nz = (W != 0).reshape(W.shape[0], k // 64, 64).any(dim=2).any(dim=0)
    last = int(nz.nonzero().max())
    m = torch.ones(k, dtype=torch.float64, device=w.device)
    m[last * 64:(last + 1) * 64] = 0
    return m


def split_out2(d, y: torch.Tensor):
    """A stored result [rows, n_valid] -> (what goes to `out`, [rows, col2 or n_valid]; what goes to `out2` transposed,
    [n_valid - col2, rows] or None)."""
    if not d["out2"]:
        return y, None
    return y[:, :d["col2"]], y[:, d["col2"]:].T


def rowstat_sums(out_rows: torch.Tensor) -> torch.Tensor:
    """(sum, sum of squares) [rows, 2] float64 of the stored fp16 rows the producer's statistics describe."""
    x = out_rows.double()
    return torch.stack([x.sum(1), (x * x).sum(1)], dim=1)


# ---- attention --------------------------------------------------------------------------------------------------------------
def attention_ref(a, q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, drop_last_block: int = 0, kv_item0=False,
                  dp_scale=False, qchunk: int = 1024) -> torch.Tensor:
    """out [nb*sq, heads*d_real] float64.  q [nb*sq, >= heads*dp], k [k_rows, >= heads*dp] and vt [heads*dp, vt_cols]
    snapshots.  Image b: Q rows b*sq, K rows b*k_bstride, V^T columns b*vt_bstride; heads zero-padded to dp (the dot product
    runs over dp), softmax scale d_real^-0.5.  Wrong references: drop_last_block = KV block size (the last KV block lost),
    kv_item0 (image 0's K/V for every image), dp_scale (dp^-0.5)."""
    nb, heads, sq, skv, dr, dp = a["nb"], a["heads"], a["sq"], a["skv"], a["d_real"], a["dp"]
    scale = (dp if dp_scale else dr) ** -0.5
    nkv = skv
    if drop_last_block:
        nkv = (skv - 1) // drop_last_block * drop_last_block
    out = torch.empty(nb * sq, heads * dr, dtype=torch.float64, device=q.device)
    for b in range(nb):
        bk = 0 if kv_item0 else b
        k0, v0 = bk * a["k_bstride"], bk * a["vt_bstride"]
        for h in range(heads):
            K = k[k0:k0 + nkv, h * dp:(h + 1) * dp].double()
            V = vt[h * dp:h * dp + dr, v0:v0 + nkv].double().T
            for r0 in range(0, sq, qchunk):
                r1 = min(sq, r0 + qchunk)
                Q = q[b * sq + r0:b * sq + r1, h * dp:(h + 1) * dp].double()
                p = torch.softmax((Q @ K.T) * scale, dim=-1)
                out[b * sq + r0:b * sq + r1, h * dr:(h + 1) * dr] = p @ V
    return out


# ---- normalisations ---------------------------------------------------------------------------------------------------------
def groupnorm_ref(g, xa: torch.Tensor, xb: Optional[torch.Tensor], gamma, beta, shift_groups=False) -> torch.Tensor:
    """GroupNorm(+SiLU) over [xa | xb]: xa [nb*hw, ca], xb [nb*hw, cb] or None -> [nb*hw, ca+cb] float64.
    shift_groups: each group normalised with the neighbouring group's statistics (wrong reference)."""
    x = xa.double() if xb is None else torch.cat([xa.double(), xb.double()], dim=1)
    nb, hw, G = g["nb"], g["hw"], g["groups"]
    c = x.shape[1]
    xg = x.reshape(nb, hw, G, c // G)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
    if shift_groups:
        mean, var = torch.roll(mean, 1, dims=2), torch.roll(var, 1, dims=2)
    y = ((xg - mean) / torch.sqrt(var + g["eps"])).reshape(nb * hw, c) * gamma.double()[None] + beta.double()[None]
    if g["silu"]:
        y = y * torch.sigmoid(y)
    return y


def layernorm_ref(l, x: torch.Tensor, gamma, beta, shift_rows=False) -> torch.Tensor:
    """LayerNorm over the c columns of x [rows, c] -> float64; shift_rows: the neighbouring row's statistics (wrong reference)."""
    x = x.double()
    mean = x.mean(dim=1, keepdim=True)
    var = x.var(dim=1, unbiased=False, keepdim=True)
    if shift_rows:
        mean, var = torch.roll(mean, 1, dims=0), torch.roll(var, 1, dims=0)
    return (x - mean) / torch.sqrt(var + l["eps"]) * gamma.double()[None] + beta.double()[None]


# ---- comparison -------------------------------------------------------------------------------------------------------------
def tol_units(got: torch.Tensor, ref: torch.Tensor, atol: float, rtol: float) -> float:
    """max |got - ref| / (atol * rms(ref) + rtol * |ref|); NaN anywhere counts as infinite."""
    got, ref = got.double(), ref.double()
    rms = ref.pow(2).mean().sqrt().clamp_min(1e-30)
    u = ((got - ref).abs() / (atol * rms + rtol * ref.abs())).nan_to_num(nan=float("inf"))
    return u.max().item() if u.numel() else 0.0
