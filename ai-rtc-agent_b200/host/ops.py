"""Thin torch-tensor wrappers over the operator-level C ABI (used by tests and tools; the per-frame
engine calls the same kernels from C++ without going through Python)."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import capi


_SCRATCH = {}  # split-K workspaces kept alive between calls (stream-ordered reuse)


def pack_conv_weight(w_oihw: torch.Tensor) -> torch.Tensor:
    """[O,I,kh,kw] -> [O, kh*kw*I] fp16 with K order [tap][c] (tap = ky*kw + kx)."""
    o, i, kh, kw = w_oihw.shape
    return w_oihw.permute(0, 2, 3, 1).reshape(o, kh * kw * i).contiguous().to(torch.float16)


def _pitch(t: torch.Tensor) -> int:
    """elements between consecutive pixels of an NHWC view: the stride of its innermost dimension with more than one index
    (torch gives a size-1 dimension an arbitrary stride, e.g. W = 1 in the 1 x 1 output of a stride-2 conv)"""
    n, h, w, _ = t.shape
    return t.stride(2) if w > 1 or (h == 1 and n == 1) else (t.stride(1) if h > 1 else t.stride(0))


def _view(t: torch.Tensor) -> capi.ActView:
    assert t.dtype == torch.float16 and t.is_cuda and t.dim() == 4
    n, h, w, c = t.shape
    assert t.stride(3) == 1 and t.stride(2) % 8 == 0
    ld = t.stride(2)
    assert t.stride(1) == w * ld and t.stride(0) == h * w * ld, "NHWC view must be dense in n,h,w"
    return capi.ActView(t.data_ptr(), n, h, w, c, ld)


def igemm(srcs: Sequence[Tuple[torch.Tensor, int]], w: torch.Tensor, out: torch.Tensor, *,
          stride: int = 1, colbias: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
          acc_scale: float = 1.0, res_scale: float = 1.0, relu: bool = False, geglu: bool = False, silu: bool = False,
          bn: int = 0, splits: int = 1, n_valid: Optional[int] = None, timeline: Optional[torch.Tensor] = None, swap: bool = False,
          tconv: bool = False, pair: bool = False, pad0: bool = False,
          rowstat_out: Optional[torch.Tensor] = None, rowstat_in: Optional[torch.Tensor] = None,
          colsum: Optional[torch.Tensor] = None, ln_c: int = 0, ln_eps: float = 1e-5,
          out2: Optional[torch.Tensor] = None, col2: int = 0, acc_scale_b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """srcs: [(NHWC fp16 tensor, ntap)], w: packed fp16 [rows, K]; out: NHWC fp16 [nb,ho,wo,ldc>=n].  pad0: 3x3 taps read input
    (stride*out + tap), the zero padding only after the last row / column (AutoencoderKL's Downsample2D).  acc_scale_b: fp32
    [nb] on the device, a factor of each batch item's contraction term (acc + bias)."""
    d = _igemm_desc(srcs, w, out, stride=stride, colbias=colbias, res=res, acc_scale=acc_scale, res_scale=res_scale, relu=relu,
                    geglu=geglu, silu=silu, bn=bn, splits=splits, n_valid=n_valid, timeline=timeline, swap=swap, tconv=tconv, pair=pair,
                    pad0=pad0,
                    rowstat_out=rowstat_out, rowstat_in=rowstat_in, colsum=colsum, ln_c=ln_c, ln_eps=ln_eps, out2=out2, col2=col2,
                    acc_scale_b=acc_scale_b)
    capi.check(capi.lib().b2sd_op_igemm(C.byref(d), capi.current_stream_ptr()), "b2sd_op_igemm")
    return out


def igemm_engine_plan(srcs, w, out, *, autotile: int = 1, allow_swap: bool = True, **kw) -> capi.IgemmPlanInfo:
    """The tile / split-K / orientation / CTA-pair choice the engine's tile policy makes for this contraction (autotile 1:
    one frame in flight, 2: >= 4 frames in flight), from the host-only planner; no launch.  Pass its bn, splits, swap and
    pair (mode == 1) to igemm() to run the contraction the way the frame program does."""
    d = _igemm_desc(srcs, w, out, **kw)
    info = capi.IgemmPlanInfo()
    capi.check(capi.lib().b2sd_igemm_plan_dry(C.byref(d), autotile, int(allow_swap), C.byref(info)), "b2sd_igemm_plan_dry")
    return info


def _igemm_desc(srcs, w, out, *, stride=1, colbias=None, res=None, acc_scale=1.0, res_scale=1.0, relu=False, geglu=False,
                silu=False, bn=0, splits=1, n_valid=None, timeline=None, swap=False, tconv=False, pair=False, pad0=False, rowstat_out=None,
                rowstat_in=None, colsum=None, ln_c=0, ln_eps=1e-5, out2=None, col2=0, acc_scale_b=None) -> capi.IgemmDesc:
    d = capi.IgemmDesc()
    d.nseg = len(srcs)
    for i, (t, ntap) in enumerate(srcs):
        d.src[i] = _view(t)
        d.ntap[i] = ntap
    assert w.dtype == torch.float16 and w.is_contiguous()
    d.w, d.w_rows, d.w_ld = w.data_ptr(), w.shape[0], w.shape[1]
    d.stride = stride
    nb, ho, wo, _ = out.shape
    d.nb, d.ho, d.wo = nb, ho, wo
    d.bn, d.splits = bn, splits
    d.swap = int(swap)
    d.out, d.ldc = out.data_ptr(), _pitch(out)
    nv = n_valid if n_valid is not None else out.shape[3]
    d.n_valid = nv
    if timeline is not None:
        d.partial = timeline.data_ptr()   # debug: int64 tensor [ctas, 8] receiving globaltimer stamps (tap kernel only)
    if colbias is not None:
        assert colbias.dtype == torch.float32 and colbias.is_contiguous()
        d.colbias = colbias.data_ptr()
        d.colbias_bstride = colbias.shape[1] if colbias.dim() == 2 and colbias.shape[0] > 1 else 0
    if res is not None:
        assert res.dtype == torch.float16
        d.res, d.ldr = res.data_ptr(), _pitch(res)
    d.acc_scale, d.res_scale = acc_scale, res_scale
    if acc_scale_b is not None:
        assert acc_scale_b.dtype == torch.float32 and acc_scale_b.is_cuda and acc_scale_b.numel() >= nb
        d.acc_scale_b = acc_scale_b.data_ptr()
    d.flags = (capi.IG_RELU if relu else 0) | (capi.IG_GEGLU if geglu else 0) | (capi.IG_TCONV if tconv else 0) | (capi.IG_PAIR if pair else 0) \
        | (capi.IG_SILU if silu else 0) | (capi.IG_PAD0 if pad0 else 0)
    if rowstat_out is not None:
        assert rowstat_out.dtype == torch.int64 and rowstat_out.is_contiguous()
        d.rowstat_out = rowstat_out.data_ptr()
    if rowstat_in is not None:
        assert rowstat_in.dtype == torch.int64 and colsum is not None and colsum.dtype == torch.float32 and ln_c > 0
        d.rowstat_in, d.colsum, d.ln_c, d.ln_eps = rowstat_in.data_ptr(), colsum.data_ptr(), ln_c, ln_eps
    if out2 is not None:
        assert out2.dtype == torch.float16 and out2.dim() == 2 and out2.stride(1) == 1
        d.out2, d.ld2, d.col2 = out2.data_ptr(), out2.stride(0), col2
    return d


def _sp():
    return capi.current_stream_ptr()


def attention(q, k, vt, out, *, nb, heads, sq, skv, d_real, dp, k_bstride, vt_bstride):
    """q [nb*sq, >=heads*dp], k [rows, >=heads*dp], vt [heads*dp, cols] (2-D fp16 views), out [nb*sq, heads*d_real]."""
    d = capi.AttnDesc()
    d.q, d.ldq = q.data_ptr(), q.stride(0)
    d.k, d.ldk, d.k_bstride, d.k_rows = k.data_ptr(), k.stride(0), k_bstride, k.shape[0]
    d.vt, d.ldvt, d.vt_bstride, d.vt_cols = vt.data_ptr(), vt.stride(0), vt_bstride, vt.shape[1]
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.nb, d.heads, d.sq, d.skv, d.d_real, d.dp = nb, heads, sq, skv, d_real, dp
    capi.check(capi.lib().b2sd_op_attention(C.byref(d), _sp()), "b2sd_op_attention")
    return out


def attention_ip(q, k, vt, out, k_ip, vt_ip, n_ip, *, nb, heads, sq, skv, d_real, dp, k_bstride, vt_bstride):
    """attention() plus IP-Adapter's decoupled image segment: k_ip [64, k.stride(0)] and vt_ip [heads*dp, 64] (fp16, keys past
    n_ip zeroed), n_ip a device int32 tensor of one element (0..64)."""
    d = capi.AttnDesc()
    d.q, d.ldq = q.data_ptr(), q.stride(0)
    d.k, d.ldk, d.k_bstride, d.k_rows = k.data_ptr(), k.stride(0), k_bstride, k.shape[0]
    d.vt, d.ldvt, d.vt_bstride, d.vt_cols = vt.data_ptr(), vt.stride(0), vt_bstride, vt.shape[1]
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.nb, d.heads, d.sq, d.skv, d.d_real, d.dp = nb, heads, sq, skv, d_real, dp
    assert k_ip.shape[0] == 64 and k_ip.stride(0) == k.stride(0) and vt_ip.shape[1] == 64 and vt_ip.stride(0) == 64
    assert n_ip.dtype == torch.int32 and n_ip.is_cuda
    capi.check(capi.lib().b2sd_op_attention_ip(C.byref(d), k_ip.data_ptr(), vt_ip.data_ptr(), n_ip.data_ptr(), _sp()),
               "b2sd_op_attention_ip")
    return out


GN_PATHS = {0: "cluster", 1: "fused", 2: "stats+apply"}


def groupnorm(xa, xb, gamma, beta, y, *, groups=32, eps=1e-5, silu=True, return_path=False):
    """xa/xb: NHWC fp16 (xb may be None); y: NHWC fp16 with C = ca + cb.  return_path: also return the kernel path that ran
    ("cluster", "fused" or "stats+apply", see b2sd_groupnorm_last_path)."""
    nb, h, w, ca = xa.shape
    cb = 0 if xb is None else xb.shape[3]
    capi.check(capi.lib().b2sd_op_groupnorm(
        xa.data_ptr(), ca, xa.stride(2), 0 if xb is None else xb.data_ptr(), cb, 0 if xb is None else xb.stride(2),
        gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), y.stride(2), nb, h * w, groups, eps, int(silu), _sp()),
        "b2sd_op_groupnorm")
    if return_path:
        return y, GN_PATHS[capi.lib().b2sd_groupnorm_last_path()]
    return y


def layernorm(x, gamma, beta, y, eps=1e-5):
    rows, c = x.shape
    capi.check(capi.lib().b2sd_op_layernorm(x.data_ptr(), x.stride(0), gamma.data_ptr(), beta.data_ptr(),
                                            y.data_ptr(), y.stride(0), rows, c, eps, _sp()), "b2sd_op_layernorm")
    return y


def upsample2x(x, y):
    nb, h, w, c = x.shape
    capi.check(capi.lib().b2sd_op_upsample2x(x.data_ptr(), y.data_ptr(), nb, h, w, c, _sp()), "b2sd_op_upsample2x")
    return y


def smallconv(x, w_oihw, bias, y, *, flags=0):
    """x: NHWC fp16 (or u8 when flags&1) [nb,in_h,in_w,cin]; y NHWC fp16 [nb,h,w,cout]."""
    nb, in_h, in_w, cin = x.shape
    _, h, w, cout = y.shape
    capi.check(capi.lib().b2sd_op_smallconv(x.data_ptr(), w_oihw.data_ptr(), 0 if bias is None else bias.data_ptr(),
                                            y.data_ptr(), y.stride(2), nb, h, w, cin, cout, in_h, in_w, flags, _sp()),
               "b2sd_op_smallconv")
    return y


def smallconv_ex(x, w_oihw, bias, y, *, flags=0, res=None, res_bstride=None, in_off=None):
    """smallconv with SiLU output (flags & 32), cout a multiple of 16 (y may be wider: its extra columns are not written) and an
    optional fp16 NHWC residual; res_bstride = elements between its batch items (default: its own; 0 broadcasts item 0)."""
    nb, in_h, in_w, cin = x.shape
    _, h, w, _ = y.shape
    cout = w_oihw.shape[0]
    rp, ldr, bs = 0, 0, 0
    if res is not None:
        assert res.dtype == torch.float16 and res.stride(3) == 1
        rp, ldr = res.data_ptr(), res.stride(2)
        bs = res.stride(0) if res_bstride is None else res_bstride
    capi.check(capi.lib().b2sd_op_smallconv_ex(x.data_ptr(), w_oihw.data_ptr(), bias.data_ptr() if bias is not None else None,
                                               y.data_ptr(), y.stride(2), nb, h, w, cin, cout, in_h, in_w, flags, rp, ldr, bs,
                                               in_off.data_ptr() if in_off is not None else None, _sp()), "b2sd_op_smallconv_ex")
    return y


def maxpool2x2(x, y):
    nb, h, w, c = x.shape
    capi.check(capi.lib().b2sd_op_maxpool2x2(x.data_ptr(), y.data_ptr(), nb, h, w, c, _sp()), "b2sd_op_maxpool2x2")
    return y


def hed_project(x, w, bias, out):
    """x NHWC fp16 [1,h,w,c] (pitch x.stride(2)); w fp32 [c], bias fp32 [1]; out fp32 [h*w]."""
    _, h, ww, c = x.shape
    capi.check(capi.lib().b2sd_op_hed_project(x.data_ptr(), x.stride(2), c, h * ww, w.data_ptr(), bias.data_ptr(), out.data_ptr(),
                                              _sp()), "b2sd_op_hed_project")
    return out


def hed_fuse(maps, out_u8, edge_f16=None):
    """maps: fp32 CUDA tensors [hk, wk]; out_u8: u8 [h, w, 3]."""
    n = len(maps)
    ptrs = (C.c_void_p * n)(*[m.data_ptr() for m in maps])
    hs = (C.c_int * n)(*[m.shape[0] for m in maps])
    ws = (C.c_int * n)(*[m.shape[1] for m in maps])
    capi.check(capi.lib().b2sd_op_hed_fuse(ptrs, hs, ws, n, out_u8.shape[0], out_u8.shape[1], out_u8.data_ptr(),
                                           edge_f16.data_ptr() if edge_f16 is not None else None, _sp()), "b2sd_op_hed_fuse")
    return out_u8


def lcm_step(x, eps, noise, coef, out_latent, do_add_noise=True):
    T, hw = x.shape[0], x.shape[1] * x.shape[2]
    capi.check(capi.lib().b2sd_op_lcm_step(x.data_ptr(), eps.data_ptr(), noise.data_ptr(), coef.data_ptr(),
                                           out_latent.data_ptr(), T, hw, int(do_add_noise), _sp()), "b2sd_op_lcm_step")
    return out_latent


def post_u8(y, out):
    nb, h, w, _ = y.shape
    capi.check(capi.lib().b2sd_op_post_u8(y.data_ptr(), y.stride(2), out.data_ptr(), nb, h, w, _sp()), "b2sd_op_post_u8")
    return out


def post_f16(y, out):
    """y: NHWC fp16 [nb, h, w, >= 3]; out: fp16 NCHW [nb, 3, h, w] = y * 2 - 1 (the float entry's tail)"""
    nb, h, w, _ = y.shape
    capi.check(capi.lib().b2sd_op_post_f16(y.data_ptr(), y.stride(2), out.data_ptr(), nb, h, w, _sp()), "b2sd_op_post_f16")
    return out
