"""Descriptor-driven references of the launches of the frame program and of the prompt / timestep refresh: contractions,
attention, GroupNorm, LayerNorm and the elementwise kernels (smallconv, upsample2x, HED's maxpool2x2 / hed_project / hed_fuse,
lcm_step, post_u8, small_linear, timestep_embedding).

Each reference reads only a launch's descriptor (the C ABI's b2sd_igemm_desc / b2sd_attn_desc / argument structs of the other
kinds, as a dict of field name -> value) and snapshots of the tensors it reads, and computes what the launch must write, in
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
    # fp16 output of an fp32 sum of 27 / 36 products of fp16-rounded inputs: the contraction's constants
    "smallconv": (3e-3, 3e-3),
    # fp32 output, fp32 sums of <= 512 products: ~1e-6 of rms expected, the rest is room for cancellation
    "hed_project": (1e-3, 1e-3),
    # fp16 output (one rounding, 4.9e-4 relative) of a few fp32 multiply-adds
    "lcm_step": (1e-3, 1e-3),
    # fp32 output, fp32 sums of <= 1280 products and an fp32 SiLU: ~1e-6 of rms expected
    "small_linear": (2e-4, 2e-4),
}
# timestep_embedding: absolute error.  The fp32 argument t * freq reaches ~1000, where one ulp is 6e-5, and expf may differ
# from torch's exp by an ulp of the frequency (another ~6e-5 at t ~ 1000).
TEMB_ATOL = 2e-4
SC_IN_U8, SC_IN_TANH3, SC_OUT_RELU, SC_IN_F32_NCHW, SC_IN_F16_NCHW, SC_OUT_SILU, SC_IN_OFFSET = 1, 2, 4, 8, 16, 32, 64
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


def k_block_mask(d, kb0: int, kb1: int, device) -> torch.Tensor:
    """[K] mask without the 64-wide K blocks [kb0, kb1) (a split-K rank's slice, or one block)."""
    k = sum(nt * c for _, _, nt, c in k_segments(d))
    m = torch.ones(k, dtype=torch.float64, device=device)
    m[kb0 * 64:kb1 * 64] = 0
    return m


def nonzero_blocks(d, w: torch.Tensor) -> List[int]:
    """the 64-wide K blocks whose weights are not all zero, in K order"""
    k = sum(nt * c for _, _, nt, c in k_segments(d))
    W = w[:n_gemm(d), :k]
    return (W != 0).reshape(W.shape[0], k // 64, 64).any(dim=2).any(dim=0).nonzero().flatten().tolist()


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


def layernorm_ref(l, x: torch.Tensor, gamma, beta, shift_rows=False, shift_affine=False) -> torch.Tensor:
    """LayerNorm over the c columns of x [rows, c] -> float64; wrong references: shift_rows, the neighbouring row's statistics;
    shift_affine, the neighbouring column's gamma and beta."""
    x = x.double()
    if shift_affine:
        gamma, beta = torch.roll(gamma, 1), torch.roll(beta, 1)
    mean = x.mean(dim=1, keepdim=True)
    var = x.var(dim=1, unbiased=False, keepdim=True)
    if shift_rows:
        mean, var = torch.roll(mean, 1, dims=0), torch.roll(var, 1, dims=0)
    return (x - mean) / torch.sqrt(var + l["eps"]) * gamma.double()[None] + beta.double()[None]


# ---- smallconv -------------------------------------------------------------------------------------------------------------
def nearest_index(n_in: int, n_out: int, device=None, exact_integer=False) -> torch.Tensor:
    """Source index of every output index of a nearest resize n_in -> n_out: torch's rule (F.interpolate, size given)
    min(floor(dst * fp32(n_in / n_out)), n_in - 1) with the product in fp32; exact_integer: floor(dst * n_in / n_out), the
    rule the two differ from wherever n_out has an odd factor (wrong reference)."""
    dst = torch.arange(n_out, device=device)
    if exact_integer:
        return dst * n_in // n_out
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    return (dst.float() * scale.to(device)).floor().long().clamp_max(n_in - 1)


def smallconv_input(a, x: torch.Tensor, in_off: Optional[torch.Tensor] = None) -> torch.Tensor:
    """What the kernel convolves: x [nb, in_h, in_w, cin] (u8 or fp16 NHWC) or [nb, cin, in_h, in_w] (the NCHW flags) ->
    the transformed input (u8 / 255, u8 - offset, tanh(z/3)*3 or fp16 as is) in fp32, rounded to fp16, as float64
    [nb, in_h, in_w, cin]."""
    f = a["flags"]
    if f & (SC_IN_F32_NCHW | SC_IN_F16_NCHW):
        x = x.permute(0, 2, 3, 1)
    v = x.float()
    if f & SC_IN_OFFSET:
        v = (v * 255.0 if f & (SC_IN_F32_NCHW | SC_IN_F16_NCHW) else v) - in_off.float()[None, None, None, :]
    elif f & SC_IN_U8:
        v = v * torch.tensor(1.0 / 255.0, dtype=torch.float32)
    elif f & SC_IN_TANH3 and not f & (SC_IN_F32_NCHW | SC_IN_F16_NCHW):
        v = torch.tanh(v * torch.tensor(1.0 / 3.0, dtype=torch.float32)) * 3.0
    return v.half().double()


def smallconv_ref(a, x: torch.Tensor, wt: torch.Tensor, bias=None, res=None, in_off=None, mirrored=False,
                  exact_integer=False, res_item0=False, no_res=False, offset_after_pad=False) -> torch.Tensor:
    """b2sd_smallconv_args -> [nb * h * w, cout] float64.  x: the source as smallconv_input takes it; wt fp32 [cin*9][cout]
    (k = tap*cin + c, tap = 3*dy + dx); bias [cout]; res [nb or 1, h*w, cout] (item n's residual, read at n * res_bstride:
    the audit snapshots each item there); in_off [3].  Wrong references: mirrored (3x3 taps flipped), exact_integer (the
    integer resize rule), res_item0 (item 0's residual for every item), no_res (residual omitted), offset_after_pad (the
    offset also subtracted from the zero padding)."""
    nb, h, w, cin, cout = a["nb"], a["h"], a["w"], a["cin"], a["cout"]
    v = smallconv_input(a, x, in_off)
    iy = nearest_index(a["in_h"], h, v.device, exact_integer)
    ix = nearest_index(a["in_w"], w, v.device, exact_integer)
    v = v[:, iy][:, :, ix].permute(0, 3, 1, 2)                                   # [nb, cin, h, w]
    if offset_after_pad:   # pad the raw frame with zeros, then subtract the offset: the border sees -in_off
        off = in_off.float().half().double().to(v.device)[None, :, None, None]
        v = F.pad(v + off, (1, 1, 1, 1)) - off
    else:
        v = F.pad(v, (1, 1, 1, 1))
    W = wt.double().reshape(3, 3, cin, cout).permute(3, 2, 0, 1)                # OIHW
    if mirrored:
        W = W.flip(2, 3)
    y = F.conv2d(v, W).permute(0, 2, 3, 1).reshape(nb, h * w, cout)
    if bias is not None:
        y = y + bias.double()[None, None, :cout]
    if res is not None and not no_res:
        r = res.double()
        if r.shape[0] == 1 or res_item0:
            r = r[:1].expand(nb, -1, -1)
        y = y + r[:, :, :cout]
    if a["flags"] & SC_OUT_RELU:
        y = y.clamp_min(0.0)
    if a["flags"] & SC_OUT_SILU:
        y = y * torch.sigmoid(y)
    return y.reshape(nb * h * w, cout)


# ---- resampling -------------------------------------------------------------------------------------------------------------
def upsample2x_ref(x: torch.Tensor, shifted=False) -> torch.Tensor:
    """x [nb, h, w, c] -> [nb, 2h, 2w, c], nearest (output row y reads source row y // 2); shifted: (y + 1) // 2 (wrong
    reference)."""
    nb, h, w, c = x.shape
    iy, ix = torch.arange(2 * h, device=x.device) // 2, torch.arange(2 * w, device=x.device) // 2
    if shifted:
        iy =((torch.arange(2 * h, device=x.device) + 1) // 2).clamp_max(h - 1)
        ix = ((torch.arange(2 * w, device=x.device) + 1) // 2).clamp_max(w - 1)
    return x[:, iy][:, :, ix]


def maxpool2x2_ref(x: torch.Tensor, average=False, shifted=False) -> torch.Tensor:
    """x [nb, h, w, c] -> [nb, h/2, w/2, c] 2x2/2 max-pool; wrong references: average pooling, the window shifted by one pixel
    (rows and columns 2y+1, 2y+2, clamped)."""
    nb, h, w, c = x.shape
    t = x.permute(0, 3, 1, 2).double()
    if shifted:
        t = F.pad(t[:, :, 1:, 1:], (0, 1, 0, 1), mode="replicate")
    y = F.avg_pool2d(t, 2) if average else F.max_pool2d(t, 2)
    return y.permute(0, 2, 3, 1).to(x.dtype)


# ---- HED --------------------------------------------------------------------------------------------------------------------
def hed_project_ref(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, no_bias=False, swap_pairs=False) -> torch.Tensor:
    """x [npix, c] fp16, w [c], bias [1] -> [npix] float64 = x . w + bias; wrong references: bias omitted, each channel pair's
    weights swapped."""
    W = w.double()
    if swap_pairs:
        W = W.reshape(-1, 2).flip(1).reshape(-1)
    y = x.double() @ W
    return y if no_bias else y + bias.double()[0]


def _bilinear(m: torch.Tensor, h: int, w: int, align_corners=False) -> torch.Tensor:
    """m [hk, wk] -> [h, w] float64 bilinear: half-pixel centres, negative source coordinates clamped to 0, the far
    neighbour clamped to the last row / column (F.interpolate(align_corners=False), cv2.INTER_LINEAR)."""
    hk, wk = m.shape
    m = m.double()

    def axis(n_out, n_in):
        o = torch.arange(n_out, dtype=torch.float64, device=m.device)
        if align_corners:
            s = o * ((n_in - 1) / (n_out - 1)) if n_out > 1 else o * 0
        else:
            s = ((o + 0.5) * (n_in / n_out) - 0.5).clamp_min(0.0)
        i0 = s.floor().long().clamp_max(n_in - 1)
        i1 = (i0 + 1).clamp_max(n_in - 1)
        return i0, i1, s - i0.double()

    y0, y1, fy = axis(h, hk)
    x0, x1, fx = axis(w, wk)
    top = m[y0][:, x0] * (1 - fx)[None] + m[y0][:, x1] * fx[None]
    bot = m[y1][:, x0] * (1 - fx)[None] + m[y1][:, x1] * fx[None]
    return top * (1 - fy)[:, None] + bot * fy[:, None]


def hed_fuse_value(maps: List[torch.Tensor], h: int, w: int, align_corners=False) -> torch.Tensor:
    """The edge value before the u8 cast, float64 [h, w]: clamp(sigmoid(mean of the bilinear-upsampled maps) * 255, 0, 255)."""
    s = sum(_bilinear(m, h, w, align_corners) for m in maps) / len(maps)
    return (torch.sigmoid(s) * 255.0).clamp(0.0, 255.0)


def hed_fuse_ref(maps: List[torch.Tensor], h: int, w: int, align_corners=False, rounding=False) -> torch.Tensor:
    """u8 [h, w] edge map (truncation, as numpy's astype(uint8)); wrong references: align_corners=True, rounding."""
    v = hed_fuse_value(maps, h, w, align_corners)
    return (v.round() if rounding else v.floor()).to(torch.uint8)


def hed_fuse_mismatch(got_u8: torch.Tensor, maps: List[torch.Tensor], h: int, w: int):
    """(number of pixels that differ from the reference, whether every difference is +-1 at a value within 1e-3 of an
    integer): the kernel's fp32 sum may fall on the other side of an integer than the float64 one."""
    v = hed_fuse_value(maps, h, w)
    d = got_u8.to(v.device).long() - v.floor().long()
    bad = d != 0
    near = (v - v.round()).abs() <= 1e-3
    return int(bad.sum()), bool(((d.abs() <= 1) & near)[bad].all())


# ---- scheduler step ---------------------------------------------------------------------------------------------------------
def lcm_step_ref(a, x: torch.Tensor, eps: torch.Tensor, noise: torch.Tensor, coef: torch.Tensor, swap_cskip_cout=False,
                 own_x0=False):
    """x, eps, noise [T, hw, 4]; coef [4 * T] (alpha, beta, c_skip, c_out) -> (out_latent [hw, 4], the new x [T, hw, 4]) float64.
    x0[i] = c_out[i] (x[i] - beta[i] eps[i]) / alpha[i] + c_skip[i] x[i]; out_latent = x0[T-1]; slot i+1 of x becomes
    alpha[i+1] x0[i] + beta[i+1] noise[i+1] (without the noise term when do_add_noise = 0), slot 0 is left alone.
    Wrong references: c_skip / c_out swapped, slot i re-noised from its own x0."""
    T = a["T"]
    c = coef.double().reshape(4, T)
    al, be, cs, co = c[0], c[1], c[2], c[3]
    if swap_cskip_cout:
        cs, co = co, cs
    X, E, N = x.double(), eps.double(), noise.double()
    x0 = co[:, None, None] * (X - be[:, None, None] * E) / al[:, None, None] + cs[:, None, None] * X
    new = X.clone()
    if T > 1:
        src = x0[1:] if own_x0 else x0[:-1]
        new[1:] = al[1:, None, None] * src + (be[1:, None, None] * N[1:] if a["do_add_noise"] else 0.0)
    return x0[T - 1], new


# ---- post_u8 ----------------------------------------------------------------------------------------------------------------
def post_u8_ref(a, y: torch.Tensor, rounding=False, bgr=False) -> torch.Tensor:
    """y [nb * h * w, 3] fp16 -> u8 [nb, 3, h, w]: x*2-1, x/2+0.5, clamp(0,1), *255, clamp(0,255), truncation, every operation
    rounded to fp16 (each is exact in float64, so rounding the float64 result is the fp16 operation).  Wrong references:
    rounding instead of truncation, BGR channel order."""
    def r(t):
        return t.half().double()
    v = y.double()
    v = r(r(v * 2.0) - 1.0)
    v = r(r(v * 0.5) + 0.5)
    v = v.clamp(0.0, 1.0)
    v = r(v * 255.0).clamp(0.0, 255.0)
    u = (v.round() if rounding else v.floor()).to(torch.uint8)
    if bgr:
        u = u.flip(1)
    return u.reshape(a["nb"], a["h"], a["w"], 3).permute(0, 3, 1, 2)


# ---- prepare-time: time embedding -------------------------------------------------------------------------------------------
def small_linear_ref(a, x: torch.Tensor, w: torch.Tensor, bias=None, no_silu=False, no_bias=False, slot0=False) -> torch.Tensor:
    """x [nb, >= k] fp32, w [n, k] fp16, bias [n] -> [nb, n] float64 = bias + act(x) W^T, act = SiLU when silu_in.  Wrong
    references: SiLU omitted, bias omitted, slot 0's input for every slot."""
    v = x[:, :a["k"]].double()
    if slot0:
        v = v[:1].expand_as(v)
    if a["silu_in"] and not no_silu:
        v = v * torch.sigmoid(v)
    y = v @ w.double().T
    if bias is not None and not no_bias:
        y = y + bias.double()[None]
    return y


def timestep_embedding_ref(t: torch.Tensor, dim: int, sin_first=False, half_minus_one=False) -> torch.Tensor:
    """t [nb] fp32 -> [nb, dim] float64 [cos | sin](t * freq), freq_j = exp(-ln(1e4) j / half) rounded to fp32 (as diffusers
    and the oracle compute it in fp32).  Wrong references: [sin | cos] order, exponent over half - 1."""
    half = dim // 2
    j = torch.arange(half, dtype=torch.float64, device=t.device)
    freq = torch.exp(-math.log(10000.0) * j / (half - 1 if half_minus_one else half)).float().double()
    arg = t.double()[:, None] * freq[None]
    c, s = torch.cos(arg), torch.sin(arg)
    return torch.cat([s, c] if sin_first else [c, s], dim=1)


# ---- comparison -------------------------------------------------------------------------------------------------------------
def tol_units(got: torch.Tensor, ref: torch.Tensor, atol: float, rtol: float) -> float:
    """max |got - ref| / (atol * rms(ref) + rtol * |ref|); NaN anywhere counts as infinite."""
    got, ref = got.double(), ref.double()
    rms = ref.pow(2).mean().sqrt().clamp_min(1e-30)
    u = ((got - ref).abs() / (atol * rms + rtol * ref.abs())).nan_to_num(nan=float("inf"))
    return u.max().item() if u.numel() else 0.0
