"""GPU parity of the attention and SIMT helper kernels through the C ABI against PyTorch fp32 ops.

Tolerances: fp16 operands, fp32 math; outputs rounded to fp16 once.  Attention additionally rounds
P to fp16 before P.V (as every fp16 flash-attention does): abs 2e-3 on O(1) outputs.

The discriminating tests (hetero inputs, poisoned keys, guarded outputs) compute their references in float64 on the GPU and
check, with assert_discriminates, that a named plausible bug would land well outside the tolerance."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close, assert_discriminates, guarded, hetero, offset_heavy_rows

pytestmark = pytest.mark.gpu


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


SELF_ATTENTION_CASES = [
    (1, 1, 128, 64, 64),     # one q tile, one kv block
    (1, 2, 256, 64, 64),     # two kv blocks: online-softmax rescale, S double buffer
    (1, 5, 4096, 64, 64),    # SD-Turbo 64x64 latent self-attention
    (2, 10, 1024, 64, 64),   # batch 2
    (1, 20, 64, 64, 64),     # 8x8 level: half-empty q tile, masked kv tail
    (1, 4, 576, 64, 64),     # 768-class odd length (tail masking)
    (1, 8, 256, 40, 64),     # SD-1.5 head dim 40 zero-padded to 64
    (1, 8, 256, 80, 128),    # SD-1.5 head dim 80 -> 128
    (2, 8, 384, 160, 192),   # SD-1.5 head dim 160 -> 192 (BKV 64 variant)
    (1, 5, 16384, 64, 64),   # SD-Turbo 1024x1024 level 0: 128 q tiles, 128 kv blocks
    (3, 8, 1024, 40, 64),    # stream batch 3
    (2, 2, 14400, 64, 64),   # 960 x 960 level 0 at batch 2: a long sequence whose last KV tile reaches into the next image
    (1, 8, 4, 40, 64),       # 128 x 128 mid block: 4 tokens, fewer than one 8-column V^T group
]


@pytest.mark.parametrize("nb,heads,seq,d,dp", SELF_ATTENTION_CASES)
def test_self_attention(cuda, nb, heads, seq, d, dp):
    ops = _ops()
    q = _rand((nb, heads, seq, d), cuda, 1).half()
    k = _rand((nb, heads, seq, d), cuda, 2).half()
    v = _rand((nb, heads, seq, d), cuda, 3).half()
    # kernel layouts: q,k [nb*seq, heads*dp] (zero padded per head), vt [heads*dp, nb*seq]
    qp = torch.zeros(nb, seq, heads, dp, dtype=torch.float16, device=cuda)
    kp = torch.zeros_like(qp)
    qp[..., :d] = q.permute(0, 2, 1, 3)
    kp[..., :d] = k.permute(0, 2, 1, 3)
    cols = -(-nb * seq // 8) * 8   # V^T row pitch: a multiple of 8 (16-byte rows for the TMA unit)
    vt = torch.zeros(heads, dp, cols, dtype=torch.float16, device=cuda)
    vt[:, :d, :nb * seq] = v.permute(1, 3, 0, 2).reshape(heads, d, nb * seq)
    out = torch.full((nb * seq, heads * d), float("nan"), dtype=torch.float16, device=cuda)
    ops.attention(qp.reshape(nb * seq, heads * dp), kp.reshape(nb * seq, heads * dp),
                  vt.reshape(heads * dp, cols)[:, :nb * seq], out, nb=nb, heads=heads, sq=seq, skv=seq, d_real=d, dp=dp,
                  k_bstride=seq, vt_bstride=seq)
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float())  # (nb,heads,seq,d)
    ref = ref.permute(0, 2, 1, 3).reshape(nb * seq, heads * d)
    assert_close(out, ref, 2e-3, 4e-3, f"self-attn nb={nb} heads={heads} seq={seq} d={d}/{dp}")


@pytest.mark.parametrize("nb,heads,seq,d,dp,skv", [(1, 5, 4096, 64, 64, 77), (4, 20, 256, 64, 64, 77),
                                                    (2, 8, 1024, 40, 64, 77)])
def test_cross_attention_shared_kv(cuda, nb, heads, seq, d, dp, skv):
    """attn2: keys/values come from the 77-token prompt, identical for every batch item (prompt K/V cache)."""
    ops = _ops()
    q = _rand((nb, heads, seq, d), cuda, 1).half()
    k = _rand((heads, skv, d), cuda, 2).half()
    v = _rand((heads, skv, d), cuda, 3).half()
    qp = torch.zeros(nb, seq, heads, dp, dtype=torch.float16, device=cuda)
    qp[..., :d] = q.permute(0, 2, 1, 3)
    kp = torch.zeros(skv, heads, dp, dtype=torch.float16, device=cuda)
    kp[..., :d] = k.permute(1, 0, 2)
    vt_full = torch.zeros(heads, dp, 128, dtype=torch.float16, device=cuda)  # pitch 128, 77 valid columns
    vt_full[:, :d, :skv] = v.permute(0, 2, 1)
    vt = vt_full.reshape(heads * dp, 128)[:, :skv]
    out = torch.empty((nb * seq, heads * d), dtype=torch.float16, device=cuda)
    ops.attention(qp.reshape(nb * seq, heads * dp), kp.reshape(skv, heads * dp), vt, out, nb=nb, heads=heads, sq=seq,
                  skv=skv, d_real=d, dp=dp, k_bstride=0, vt_bstride=0)
    ref = F.scaled_dot_product_attention(q.float(), k.float()[None], v.float()[None])
    ref = ref.permute(0, 2, 1, 3).reshape(nb * seq, heads * d)
    assert_close(out, ref, 2e-3, 4e-3, f"cross-attn nb={nb} heads={heads} seq={seq}")


# ---- attention under poison: masks, batch strides, padded head dims, peaked softmax -----------------------------------------
ATTN_TOL = (2e-3, 4e-3)


def _bkv(dp):
    return 64 if dp == 192 else 128   # KV block of attn_kernel (the dp = 192 variant halves it)


def _attn64(q, k, v, d):
    """float64 softmax(q k^T / sqrt(d)) v; q [nb,heads,sq,d], k/v [nb or 1,heads,skv,d]; returns [nb*sq, heads*d]."""
    s = q.double() @ k.double().transpose(-1, -2) / math.sqrt(d)
    o = torch.softmax(s, dim=-1) @ v.double()
    return o.permute(0, 2, 1, 3).reshape(q.shape[0] * q.shape[2], -1)


def _q_layout(q, dp):
    """[nb,heads,sq,d] -> the kernel's [nb*sq, heads*dp] (each head zero-padded to dp)."""
    nb, heads, sq, d = q.shape
    qp = torch.zeros(nb, sq, heads, dp, dtype=torch.float16, device=q.device)
    qp[..., :d] = q.permute(0, 2, 1, 3)
    return qp.reshape(nb * sq, heads * dp)


def _vt_layout(v, dp, pitch=None):
    """[nb,heads,skv,d] -> V^T [heads*dp, nb*skv] (key index contiguous), or, for a single batch item, with row pitch `pitch`."""
    nb, heads, skv, d = v.shape
    cols = nb * skv if pitch is None else pitch
    vt = torch.zeros(heads, dp, cols, dtype=torch.float16, device=v.device)
    vt[:, :d, :nb * skv] = v.permute(1, 3, 0, 2).reshape(heads, d, nb * skv)
    return vt.reshape(heads * dp, cols)


BATCH_TAIL_SEQS = [144, 576, 4096 + 64]


@pytest.mark.parametrize("seq", BATCH_TAIL_SEQS)
@pytest.mark.parametrize("d,dp", [(64, 64), (80, 128), (160, 192)])
def test_self_attention_batch_tail_poisoned(cuda, seq, d, dp):
    """Four batch items packed with k_bstride = vt_bstride = seq, as the engine packs them: the tail KV tile of batch item b
    reads the leading keys of item b+1.  Those keys carry a component along a direction that only item b's queries share, so
    their logit for item b's queries is ~+30 (a mask leak moves the output by O(1), not O(1/seq)), while for item b+1 they are
    ordinary keys; their values are raised by 16.  Values get their own offset per (batch item, head).  Catches: the tail not
    masked, a mask one column too wide, item 0's values used for every item (V^T batch stride ignored).  The output is written
    with ldo > heads*d into a guarded buffer."""
    ops = _ops()
    nb, heads = 4, 2
    bkv = _bkv(dp)
    tail = -(-seq // bkv) * bkv - seq        # keys of item b+1 that item b's last tile reads
    q = _rand((nb, heads, seq, d), cuda, 1)
    k = _rand((nb, heads, seq, d), cuda, 2)
    v = hetero((nb, heads, seq, d), (0, 1), 3, cuda, scale=(0.5, 2.0)).float()
    q[..., :nb] = 0
    k[..., :nb] = 0
    big = 7.5 * math.sqrt(d)                 # logit 4 * big / sqrt(d) = 30
    for b in range(nb):
        q[b, :, :, b] = 4.0
        if b + 1 < nb and tail:
            k[b + 1, :, :tail, b] = big
            v[b + 1, :, :tail] += 16.0
    q, k, v = q.half(), k.half(), v.half()
    out = guarded((nb * seq, heads * d), pitch=heads * d + 64, device=cuda)
    ops.attention(_q_layout(q, dp), _q_layout(k, dp), _vt_layout(v, dp), out.view, nb=nb, heads=heads, sq=seq, skv=seq,
                  d_real=d, dp=dp, k_bstride=seq, vt_bstride=seq)
    out.assert_untouched(f"self-attn out seq={seq} d={d}/{dp}")
    ref = _attn64(q, k, v, d)
    what = f"self-attn nb={nb} seq={seq} d={d}/{dp} (tail reads {tail} keys of the next item)"
    if tail:
        # item b sees item b+1's first `extra` keys as well (the last item's tail is out of bounds: zero keys, masked)
        def leak(extra):
            kk = torch.cat([k, torch.cat([k[1:, :, :extra], torch.zeros_like(k[:1, :, :extra])])], dim=2)
            vv = torch.cat([v, torch.cat([v[1:, :, :extra], torch.zeros_like(v[:1, :, :extra])])], dim=2)
            return _attn64(q, kk, vv, d)
        assert_discriminates(out.view, ref, leak(tail), *ATTN_TOL, what, "tail tile not masked")
        assert_discriminates(out.view, ref, leak(1), *ATTN_TOL, what, "kv mask one column too wide")
    s = q.double() @ k.double().transpose(-1, -2) / math.sqrt(d)
    wrong_v = (torch.softmax(s, dim=-1) @ v[:1].double()).permute(0, 2, 1, 3).reshape(nb * seq, -1)
    assert_discriminates(out.view, ref, wrong_v, *ATTN_TOL, what, "batch item 0's values for every item")


# the mid-block token counts of the smallest engines (64 x 64: 1, 128 x 128: 4, 128 x 192: 6), at stream batch 3: fewer
# tokens than one 8-column V^T group, and a batch that is not a power of two
PADDED_VT_SEQS = [36, 196, 1, 4, 6]


def _padded_vt_batch(seq):
    return 4 if seq >= 8 else 3


@pytest.mark.parametrize("seq", PADDED_VT_SEQS)
@pytest.mark.parametrize("d,dp", [(40, 64), (80, 128), (160, 192)])
def test_self_attention_padded_vt_batch_stride(cuda, seq, d, dp):
    """The transformer program for token counts that are not a multiple of 8 with several images (SD-1.5 at 192x192: 36 and 9
    tokens; at 448x448: 196 and 49): K rows of image b start at b * seq, but V^T columns at b * seqp, seqp = seq rounded up to
    8, because each image's V^T is its own GEMM into a column range whose origin the TMA unit needs 16-byte aligned.  The V^T
    pad columns [b * seqp + seq, (b + 1) * seqp) hold poison (64) that only the skv mask keeps out of P.V, and the batch-tail
    poison of test_self_attention_batch_tail_poisoned makes the keys item b's tail tile reads from item b+1 dominate its
    softmax if unmasked.  Catches: V^T addressed with k_bstride, K addressed with vt_bstride, the pad columns or the tail
    keys leaking in."""
    ops = _ops()
    from tests import launch_ref as R
    nb, heads = _padded_vt_batch(seq), 2
    seqp = -(-seq // 8) * 8
    bkv = _bkv(dp)
    tail = -(-seq // bkv) * bkv - seq
    q = _rand((nb, heads, seq, d), cuda, 1)
    k = _rand((nb, heads, seq, d), cuda, 2)
    v = hetero((nb, heads, seq, d), (0, 1), 3, cuda, scale=(0.5, 2.0)).float()
    q[..., :nb] = 0
    k[..., :nb] = 0
    big = 7.5 * math.sqrt(d)
    for b in range(nb):
        q[b, :, :, b] = 4.0
        if b + 1 < nb:
            k[b + 1, :, :min(tail, seq), b] = big
            v[b + 1, :, :min(tail, seq)] += 16.0
    q, k, v = q.half(), k.half(), v.half()
    vt = torch.zeros(heads, dp, nb, seqp, dtype=torch.float16, device=cuda)
    vt[:, :, :, seq:] = 64.0                             # pad columns of every image
    vt[:, :d, :, :seq] = v.permute(1, 3, 0, 2)
    vt = vt.reshape(heads * dp, nb * seqp)
    qb, kb = _q_layout(q, dp), _q_layout(k, dp)
    out = guarded((nb * seq, heads * d), pitch=heads * d + 64, device=cuda)
    ops.attention(qb, kb, vt, out.view, nb=nb, heads=heads, sq=seq, skv=seq, d_real=d, dp=dp, k_bstride=seq, vt_bstride=seqp)
    out.assert_untouched(f"self-attn out seq={seq} d={d}/{dp}")
    a = {"nb": nb, "heads": heads, "sq": seq, "skv": seq, "d_real": d, "dp": dp, "k_bstride": seq, "vt_bstride": seqp}
    ref = _attn64(q, k, v, d)
    assert torch.allclose(R.attention_ref(a, qb, kb, vt), ref, rtol=1e-9, atol=1e-9)   # the layout above is what `a` describes
    what = f"self-attn nb={nb} seq={seq} (V^T stride {seqp}) d={d}/{dp}"
    assert_discriminates(out.view, ref, R.attention_ref(dict(a, vt_bstride=seq), qb, kb, vt), *ATTN_TOL, what,
                         "V^T addressed with the K batch stride")
    if seq > 1:   # one key per image: the output does not depend on which key it is
        assert_discriminates(out.view, ref, R.attention_ref(dict(a, k_bstride=seqp), qb,
                                                            torch.cat([kb, kb.new_zeros((nb * seqp, kb.shape[1]))]), vt),
                             *ATTN_TOL, what, "K addressed with the V^T batch stride")
    assert_discriminates(out.view, ref, R.attention_ref(dict(a, skv=seqp), qb, torch.cat([kb, kb.new_zeros((8, kb.shape[1]))]), vt),
                         *ATTN_TOL, what, "V^T pad columns (and the keys past seq) not masked")


@pytest.mark.parametrize("nb", [1, 4])
@pytest.mark.parametrize("d,dp,heads", [(40, 64, 8), (64, 64, 5), (80, 128, 8), (160, 192, 8)])
@pytest.mark.parametrize("rows", [128, 77])
def test_cross_attention_prompt_poisoned(cuda, nb, d, dp, heads, rows):
    """attn2 against the 77-token prompt K / V^T cache shared by every batch item (k_bstride = vt_bstride = 0), V^T with row
    pitch 128.  rows = 128: K and V^T handed over with 128 rows / columns, of which 77..127 are poison (a logit of ~+30 for every
    query, values of 64) that only the skv = 77 mask keeps out.  rows = 77: the engine's k_rows = vt_cols = 77, with the same
    poison sitting in memory just past the tensor-map bounds.  dp = 192 runs KV blocks of 64: the second has 13 valid
    columns.  Catches: a mask one column too wide, a KV tail not masked, reading past k_rows / vt_cols."""
    ops = _ops()
    skv, sq = 77, 576
    q = _rand((nb, heads, sq, d), cuda, 1) * 1.5
    q[..., 0] = 4.0
    k = _rand((1, heads, 128, d), cuda, 2)
    k[..., 0] = 0.0
    k[:, :, skv:, 0] = 7.5 * math.sqrt(d)
    v = hetero((1, heads, 128, d), (1,), 3, cuda, scale=(0.5, 2.0)).float()
    v[:, :, skv:] = 64.0
    q, k, v = q.half(), k.half(), v.half()
    kbuf = _q_layout(k, dp)                       # [128, heads*dp]
    vtbuf = _vt_layout(v, dp, pitch=128)          # [heads*dp, 128]
    out = guarded((nb * sq, heads * d), pitch=heads * d + 32, device=cuda)
    ops.attention(_q_layout(q, dp), kbuf[:rows], vtbuf[:, :rows], out.view, nb=nb, heads=heads, sq=sq, skv=skv, d_real=d, dp=dp,
                  k_bstride=0, vt_bstride=0)
    out.assert_untouched(f"cross-attn out d={d}/{dp}")
    ref = _attn64(q, k[:, :, :skv], v[:, :, :skv], d)
    what = f"cross-attn nb={nb} heads={heads} d={d}/{dp} rows={rows}"
    assert_discriminates(out.view, ref, _attn64(q, k[:, :, :skv + 1], v[:, :, :skv + 1], d), *ATTN_TOL, what,
                         "kv mask one column too wide")
    nread = -(-skv // _bkv(dp)) * _bkv(dp)
    assert_discriminates(out.view, ref, _attn64(q, k[:, :, :nread], v[:, :, :nread], d), *ATTN_TOL, what, "KV tail not masked")


def _online_no_alpha(q, k, v, d, bkv):
    """The flash-attention recurrence with the O rescale by alpha = exp(m_old - m_new) left out (l is still rescaled): what a
    kernel computes if it forgets to rescale its accumulator when the running maximum rises."""
    s = q.double() @ k.double().transpose(-1, -2) / math.sqrt(d)
    m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=torch.float64, device=s.device)
    l = torch.zeros_like(m)
    o = torch.zeros(s.shape[:-1] + (d,), dtype=torch.float64, device=s.device)
    for j in range(0, s.shape[-1], bkv):
        sj = s[..., j:j + bkv]
        m_new = torch.maximum(m, sj.amax(-1, keepdim=True))
        p = torch.exp(sj - m_new)
        l = l * torch.exp(m - m_new) + p.sum(-1, keepdim=True)
        o = o + p @ v.double()[..., j:j + bkv, :]
        m = m_new
    o = o / l
    return o.permute(0, 2, 1, 3).reshape(q.shape[0] * q.shape[2], -1)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("d,dp", [(64, 64), (80, 128), (160, 192)])
def test_attention_peaked_softmax(cuda, where, d, dp):
    """Logits with std ~9 plus a +70 bonus on one key, placed in the first, a middle or the last KV block: P is close to one-hot,
    so the alpha rescale of the running accumulator and the fp16 rounding of P carry the whole result.  Catches: O not
    rescaled when the running maximum rises, the KV block holding the maximum lost (ring stage / phase error)."""
    ops = _ops()
    nb, heads, seq = 1, 2, 576
    bkv = _bkv(dp)
    t = {"first": 5, "middle": (seq // bkv // 2) * bkv + 7, "last": seq - 3}[where]
    q = _rand((nb, heads, seq, d), cuda, 1) * 9.0
    k = _rand((nb, heads, seq, d), cuda, 2)
    v = _rand((nb, heads, seq, d), cuda, 3)
    q[..., 0] = 8.0
    k[..., 0] = 0.0
    k[..., t, 0] = 70.0 * math.sqrt(d) / 8.0
    q, k, v = q.half(), k.half(), v.half()
    out = guarded((nb * seq, heads * d), device=cuda)
    ops.attention(_q_layout(q, dp), _q_layout(k, dp), _vt_layout(v, dp), out.view, nb=nb, heads=heads, sq=seq, skv=seq,
                  d_real=d, dp=dp, k_bstride=seq, vt_bstride=seq)
    out.assert_untouched("peaked attention out")
    ref = _attn64(q, k, v, d)
    what = f"peaked attention d={d}/{dp} max at key {t} ({where} block)"
    j0 = t // bkv * bkv
    keep = torch.ones(seq, dtype=torch.bool, device=cuda)
    keep[j0:j0 + bkv] = False
    assert_discriminates(out.view, ref, _attn64(q, k[:, :, keep], v[:, :, keep], d), *ATTN_TOL, what,
                         "KV block holding the maximum lost")
    if where != "first":
        assert_discriminates(out.view, ref, _online_no_alpha(q, k, v, d, bkv), *ATTN_TOL, what, "O not rescaled by alpha")


@pytest.mark.parametrize("nb,h,w,ca,cb,silu,eps", [
    (1, 64, 64, 320, 0, True, 1e-5), (2, 32, 32, 640, 0, False, 1e-6), (1, 16, 16, 1280, 1280, True, 1e-5),
    (1, 32, 32, 1280, 640, True, 1e-5),   # 1920 channels: groups of 60 straddle the concat boundary
    (4, 8, 8, 1280, 0, True, 1e-5), (1, 24, 24, 640, 320, True, 1e-5),
    (1, 64, 64, 640, 320, True, 1e-5),    # cluster of 8 CTAs per group
    (1, 8, 8, 1280, 1280, True, 1e-5),    # one-CTA cluster
    (1, 96, 96, 640, 320, True, 1e-5),    # too large for a cluster and for the register cache: statistics + apply launches
])
def test_groupnorm(cuda, nb, h, w, ca, cb, silu, eps):
    ops = _ops()
    xa = (_rand((nb, h, w, ca), cuda, 1) * 1.5 + 0.3).half()
    xb = (_rand((nb, h, w, cb), cuda, 2) * 0.7 - 0.2).half() if cb else None
    c = ca + cb
    gamma = (1 + 0.1 * _rand((c,), cuda, 3)).float()
    beta = (0.1 * _rand((c,), cuda, 4)).float()
    y = torch.empty((nb, h, w, c), dtype=torch.float16, device=cuda)
    ops.groupnorm(xa, xb, gamma, beta, y, eps=eps, silu=silu)
    x = xa if xb is None else torch.cat([xa, xb], dim=3)
    ref = F.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, eps)
    if silu:
        ref = F.silu(ref)
    assert_close(y, ref.permute(0, 2, 3, 1), 3e-3, 2e-3, f"groupnorm {ca}+{cb}")


def _gn_stats(x, groups=32):
    """float64 (mean, biased variance) per (batch item, group) of an NHWC tensor."""
    nb, h, w, c = x.shape
    xg = x.double().reshape(nb, h * w, groups, c // groups)
    return xg.mean(dim=(1, 3)), xg.var(dim=(1, 3), unbiased=False)


def _gn_apply(x, mean, var, gamma, beta, eps, silu, chan_group=None, groups=32):
    """GroupNorm(+SiLU) of NHWC x with the given per-(batch item, group) statistics, in float64; chan_group maps channel ->
    group (default c // cpg)."""
    c = x.shape[3]
    if chan_group is None:
        chan_group = torch.arange(c, device=x.device) // (c // groups)
    m = mean[:, chan_group][:, None, None, :]
    r = (var[:, chan_group] + eps).rsqrt()[:, None, None, :]
    y = (x.double() - m) * r * gamma.double() + beta.double()
    return F.silu(y) if silu else y


def _gn_case(cuda, nb, h, w, ca, cb, eps, seed=1):
    """hetero NHWC input (own offset / scale per batch item and channel), split at the concat boundary; group 1 of the last batch
    item is shrunk to std ~2e-3 so its variance is comparable with eps (a swapped eps moves that group's output by O(1))."""
    c = ca + cb
    x = hetero((nb, h, w, c), (0, 3), seed, cuda)
    cpg = c // 32
    x[nb - 1, :, :, cpg:2 * cpg] = (_rand((h, w, cpg), cuda, seed + 7) * 2e-3).half()
    gamma = (1 + 0.2 * _rand((c,), cuda, 3)).float()
    beta = (0.2 * _rand((c,), cuda, 4)).float()
    xa = x[..., :ca].contiguous()
    xb = x[..., ca:].contiguous() if cb else None
    return x, xa, xb, gamma, beta


def _gn_expected_path(ca, cb, hw):
    cl, th, ppc = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    from ai_rtc_agent_b200.host import capi
    assert capi.lib().b2sd_groupnorm_plan_dry(ca, cb, 32, hw, ctypes.byref(cl), ctypes.byref(th), ctypes.byref(ppc)) == 0
    return cl.value


# (path, cluster size or None, nb, h, w, ca, cb, eps).  The fused / stats+apply split of the non-cluster shapes is the
# planner's (elementwise.cu groupnorm_launch): fused when a CTA's chunk fits the GN_CACHE = 12 register iterations
# (ceil(ppc / rpi)) and the whole grid (128 chunks x nb) is co-resident.  (1,96,96,640): vc 80, rpi 6, ppc 72 -> 12 iterations,
# 128 chunks; 640+320 at 96x96: rpi 4 -> 18 iterations; 640+320 at 72x72: ppc 41, rpi 4 -> 11 iterations, 127 chunks.
GN_PATH_CASES = [
    ("cluster", 1, 1, 16, 16, 1280, 0, 1e-5), ("cluster", 1, 4, 16, 16, 1280, 0, 1e-6),
    ("cluster", 2, 1, 32, 32, 640, 0, 1e-6), ("cluster", 2, 4, 32, 32, 640, 0, 1e-5),
    ("cluster", 4, 1, 64, 64, 320, 0, 1e-5), ("cluster", 4, 4, 64, 64, 320, 0, 1e-5),
    ("cluster", 8, 1, 64, 64, 640, 320, 1e-5), ("cluster", 8, 4, 64, 64, 640, 320, 1e-6),   # groups of 30 straddle the concat
    ("cluster", 4, 2, 32, 32, 1280, 640, 1e-5),                                              # groups of 60 straddle the concat
    ("cluster", 1, 4, 1, 1, 1280, 0, 1e-5),                                                  # 64 x 64 engine: 1-pixel images
    ("fused", None, 1, 96, 96, 640, 0, 1e-5), ("fused", None, 1, 96, 96, 640, 0, 1e-6),
    ("fused", None, 1, 72, 72, 640, 320, 1e-5),                                              # fused, straddling groups
    ("stats+apply", None, 1, 96, 96, 640, 320, 1e-5),                                        # straddling groups
    ("stats+apply", None, 4, 96, 96, 640, 0, 1e-6),   # 4 x 128 chunks: more CTAs than are co-resident
]
GN_OCCUPANCY_DEPENDENT = {("fused", 1, 96, 96, 640, 0), ("fused", 1, 72, 72, 640, 320), ("stats+apply", 4, 96, 96, 640, 0)}


@pytest.mark.parametrize("path,cl,nb,h,w,ca,cb,eps", GN_PATH_CASES)
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_paths_discriminate(cuda, path, cl, nb, h, w, ca, cb, eps, silu):
    """Every GroupNorm kernel (cluster of 1/2/4/8 CTAs, cooperative fused, statistics + apply) against a float64 reference on
    inputs whose batch items and groups all have different statistics.  Catches: another batch item's statistics, a
    neighbouring group's statistics, a channel put into the neighbouring group, eps 1e-5 and 1e-6 confused."""
    ops = _ops()
    assert _gn_expected_path(ca, cb, h * w) == (cl or 0), "planner no longer picks this cluster size; re-derive the case"
    x, xa, xb, gamma, beta = _gn_case(cuda, nb, h, w, ca, cb, eps)
    c = ca + cb
    y = torch.full((nb, h, w, c), float("nan"), dtype=torch.float16, device=cuda)
    _, ran = ops.groupnorm(xa, xb, gamma, beta, y, eps=eps, silu=silu, return_path=True)
    print(f"groupnorm nb={nb} {h}x{w} {ca}+{cb}: path={ran} (wanted {path})")
    mean, var = _gn_stats(x)
    ref = _gn_apply(x, mean, var, gamma, beta, eps, silu)
    what = f"groupnorm[{ran}] nb={nb} {h}x{w} {ca}+{cb} eps={eps}"
    tol = (3e-3, 2e-3)
    cpg = c // 32
    shifted = ((torch.arange(c, device=cuda) + 1) // cpg).clamp(max=31)
    assert_discriminates(y, ref, _gn_apply(x, mean.roll(1, 1), var.roll(1, 1), gamma, beta, eps, silu), *tol, what,
                         "statistics of group g-1")
    assert_discriminates(y, ref, _gn_apply(x, mean, var, gamma, beta, eps, silu, chan_group=shifted), *tol, what,
                         "group boundary shifted by one channel")
    assert_discriminates(y, ref, _gn_apply(x, mean, var, gamma, beta, 1e-6 if eps == 1e-5 else 1e-5, silu), *tol, what,
                         "eps 1e-5 and 1e-6 swapped")
    if nb > 1:
        assert_discriminates(y, ref, _gn_apply(x, mean[:1].expand_as(mean), var[:1].expand_as(var), gamma, beta, eps, silu),
                             *tol, what, "batch item 0's statistics for every item")
    if ran != path:
        assert (path, nb, h, w, ca, cb) in GN_OCCUPANCY_DEPENDENT, f"{what}: ran the {ran} path, the planner's choice is {path}"
        pytest.skip(f"{what}: this device's occupancy selected the {ran} path, not {path} (the output was verified)")


@pytest.mark.parametrize("nb,h,w,ca,cb,path", [
    (1, 32, 32, 640, 0, "cluster"), (2, 64, 64, 640, 320, "cluster"), (1, 16, 16, 1280, 0, "cluster"),
    (1, 96, 96, 640, 0, "fused"), (1, 96, 96, 640, 320, "stats+apply"),
])
def test_groupnorm_offset_heavy(cuda, nb, h, w, ca, cb, path):
    """Groups whose mean is 30-100 standard deviations away from zero (within fp16 range).  Every GroupNorm kernel sums
    x - pilot and (x - pilot)^2 in fp32, the pilot being the group's first channel at the image's first pixel, so the
    variance keeps fp32 precision however far the mean is from zero, as long as the pilot lies within a few standard
    deviations of the mean; test_precision_gpu.test_floor_groupnorm holds every path to the fp16 floor for |mean|/std up to
    100 on such data, and test_precision_audit_gpu measures the pilot's distance on real activations (at most 3.3 std).  The case's error, in units of the tolerance, is printed."""
    ops = _ops()
    c = ca + cb
    g = torch.Generator().manual_seed(11)
    sign = torch.randint(0, 2, (nb, 1, 1, 32, 1), generator=g).double() * 2 - 1
    mags = torch.stack([torch.linspace(30, 100, 32, dtype=torch.float64)[torch.randperm(32, generator=g)] for _ in range(nb)])
    gmean = sign * mags.reshape(nb, 1, 1, 32, 1)
    coff = 0.5 * (torch.rand((nb, 1, 1, 32, c // 32), generator=g, dtype=torch.float64) * 2 - 1)
    x = (gmean + coff + torch.randn((nb, h, w, 32, c // 32), generator=g, dtype=torch.float64)).reshape(nb, h, w, c)
    x = x.half().to(cuda)
    gamma = (1 + 0.2 * _rand((c,), cuda, 3)).float()
    beta = (0.2 * _rand((c,), cuda, 4)).float()
    y = torch.full((nb, h, w, c), float("nan"), dtype=torch.float16, device=cuda)
    _, ran = ops.groupnorm(x[..., :ca].contiguous(), x[..., ca:].contiguous() if cb else None, gamma, beta, y, eps=1e-5,
                           silu=True, return_path=True)
    mean, var = _gn_stats(x)
    ratio = (mean.abs() / var.sqrt()).min().item(), (mean.abs() / var.sqrt()).max().item()
    ref = _gn_apply(x, mean, var, gamma, beta, 1e-5, True)
    err = ((y.double() - ref).abs() / (3e-3 + 2e-3 * ref.abs())).max().item()
    print(f"groupnorm offset-heavy nb={nb} {h}x{w} {ca}+{cb}: path={ran} |mean|/std in [{ratio[0]:.0f}, {ratio[1]:.0f}], "
          f"max error = {err:.3f} x tolerance")
    assert ratio[0] >= 25 and ratio[1] >= 90
    assert_discriminates(y, ref, _gn_apply(x, mean.roll(1, 1), var.roll(1, 1), gamma, beta, 1e-5, True), 3e-3, 2e-3,
                         f"offset-heavy groupnorm[{ran}]", "statistics of group g-1")
    if ran != path:
        pytest.skip(f"offset-heavy {h}x{w} {ca}+{cb}: ran the {ran} path, not {path} (the output was verified)")


@pytest.mark.parametrize("rows,c", [(4096, 320), (1024, 640), (77, 1280), (5, 64)])
def test_layernorm(cuda, rows, c):
    """Every row has its own offset and scale: catches a kernel that normalises a row with a neighbouring row's statistics."""
    ops = _ops()
    x = hetero((rows, c), (0,), 1, cuda)
    gamma = (1 + 0.1 * _rand((c,), cuda, 2)).float()
    beta = (0.1 * _rand((c,), cuda, 3)).float()
    y = torch.empty_like(x)
    ops.layernorm(x, gamma, beta, y)
    xd = x.double()
    ref = F.layer_norm(xd, (c,), gamma.double(), beta.double(), 1e-5)
    mean, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    wrong = (xd - mean.roll(1, 0)) * (var.roll(1, 0) + 1e-5).rsqrt() * gamma.double() + beta.double()
    assert_discriminates(y, ref, wrong, 3e-3, 2e-3, f"layernorm {rows}x{c}", "statistics of the neighbouring row")


@pytest.mark.parametrize("rows,c", [(1024, 320), (256, 1280)])
def test_layernorm_offset_heavy(cuda, rows, c):
    """Rows with |mean|/std of 30..100: layernorm_kernel sums x - x[0] and (x - x[0])^2 in fp32, so the variance keeps fp32
    precision however far the mean is from zero while x[0] lies within a few standard deviations of the mean;
    test_precision_gpu.test_floor_layernorm holds it to the fp16 floor for |mean|/std up to 100 on such rows.
    The error, in units of the tolerance, is printed."""
    ops = _ops()
    x = offset_heavy_rows(rows, c, cuda)
    gamma = (1 + 0.1 * _rand((c,), cuda, 2)).float()
    beta = (0.1 * _rand((c,), cuda, 3)).float()
    y = torch.empty_like(x)
    ops.layernorm(x, gamma, beta, y)
    xd = x.double()
    ref = F.layer_norm(xd, (c,), gamma.double(), beta.double(), 1e-5)
    err = ((y.double() - ref).abs() / (3e-3 + 2e-3 * ref.abs())).max().item()
    print(f"layernorm offset-heavy {rows}x{c}: max error = {err:.3f} x tolerance")
    mean, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    wrong = (xd - mean.roll(1, 0)) * (var.roll(1, 0) + 1e-5).rsqrt() * gamma.double() + beta.double()
    assert_discriminates(y, ref, wrong, 3e-3, 2e-3, f"offset-heavy layernorm {rows}x{c}", "statistics of the neighbouring row")


def test_upsample2x(cuda):
    ops = _ops()
    x = _rand((2, 8, 12, 64), cuda, 1).half()
    y = torch.empty((2, 16, 24, 64), dtype=torch.float16, device=cuda)
    ops.upsample2x(x, y)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(y.float(), ref)


def test_smallconv_unet_conv_in(cuda):
    ops = _ops()
    x = _rand((2, 16, 16, 4), cuda, 1).half()
    w = _rand((320, 4, 3, 3), cuda, 2, 1 / 6.0).half()
    b = _rand((320,), cuda, 3).float()
    y = torch.empty((2, 16, 16, 320), dtype=torch.float16, device=cuda)
    ops.smallconv(x, w, b, y)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1).permute(0, 2, 3, 1)
    assert_close(y, ref, 2e-3, 2e-3, "conv_in 4->320")


def test_smallconv_taesd_encoder_head_u8(cuda):
    """lib/pipeline.py:61-63 (u8 NHWC -> f32/255 -> NCHW) + VaeImageProcessor 2x-1 + EncoderTiny (x+1)/2 + conv."""
    ops = _ops()
    g = torch.Generator().manual_seed(0)
    frame = torch.randint(0, 256, (1, 64, 48, 3), dtype=torch.uint8, generator=g).to(cuda)
    w = _rand((64, 3, 3, 3), cuda, 2, 1 / 5.0).half()
    b = _rand((64,), cuda, 3).float()
    y = torch.empty((1, 64, 48, 64), dtype=torch.float16, device=cuda)
    ops.smallconv(frame, w, b, y, flags=1)
    x = frame.float() / 255.0
    x = ((2 * x - 1) + 1) / 2
    ref = F.conv2d(x.permute(0, 3, 1, 2), w.float(), b, padding=1).permute(0, 2, 3, 1)
    assert_close(y, ref, 2e-3, 2e-3, "taesd encoder head (u8 in)")


def test_smallconv_resize_nearest(cuda):
    """VaeImageProcessor.preprocess resizes (nearest) when the frame is not HxW (SURVEY a-4)."""
    ops = _ops()
    g = torch.Generator().manual_seed(1)
    frame = torch.randint(0, 256, (1, 30, 40, 3), dtype=torch.uint8, generator=g).to(cuda)
    w = _rand((64, 3, 3, 3), cuda, 2, 1 / 5.0).half()
    y = torch.empty((1, 64, 64, 64), dtype=torch.float16, device=cuda)
    ops.smallconv(frame, w, None, y, flags=1)
    x = F.interpolate((frame.float() / 255.0).permute(0, 3, 1, 2), size=(64, 64))
    ref = F.conv2d(x, w.float(), None, padding=1).permute(0, 2, 3, 1)
    assert_close(y, ref, 2e-3, 2e-3, "encoder head with nearest resize")


# camera frames into engine sizes; the last pair has an exact 5:4 ratio, where every nearest rule agrees
_RESIZE_PAIRS = [((600, 800), (576, 768)), ((720, 1280), (448, 768)), ((1080, 1920), (832, 896)), ((300, 400), (128, 192)),
                 ((150, 200), (576, 768)), ((480, 640), (384, 512))]
_EXACT_RATIO = ((480, 640), (384, 512))


def _pair_id(p):
    return "x".join(map(str, p))


def _nearest_index_map(src, dst, device):
    """long [2, h, w]: the (row, column) of the source pixel that F.interpolate(size=dst, mode="nearest") reads for each
    output pixel, found by resizing a tensor of source coordinates on `device`."""
    yy, xx = torch.meshgrid(torch.arange(src[0], dtype=torch.float32), torch.arange(src[1], dtype=torch.float32), indexing="ij")
    return F.interpolate(torch.stack([yy, xx])[None].to(device), size=dst, mode="nearest")[0].long().cpu()


def _integer_rule_map(src, dst):
    """The exact-integer rule floor(dst * in / out), for comparison: it differs from torch's wherever out has an odd factor."""
    ys = torch.arange(dst[0]) * src[0] // dst[0]
    xs = torch.arange(dst[1]) * src[1] // dst[1]
    return torch.stack(torch.meshgrid(ys, xs, indexing="ij"))


def _coordinate_frame(h, w):
    """u8 [1, h, w, 3] whose pixel (y, x) encodes its own coordinates: R = x & 255, G = y & 255, B = (x >> 8) | (y >> 8) << 4."""
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    return torch.stack([xx & 255, yy & 255, (xx >> 8) | ((yy >> 8) << 4)], -1).to(torch.uint8)[None]


@pytest.mark.parametrize("entry", ["u8", "f32", "f16"])
@pytest.mark.parametrize("src,dst", _RESIZE_PAIRS, ids=[f"{_pair_id(s)}-{_pair_id(d)}" for s, d in _RESIZE_PAIRS])
def test_smallconv_resize_index_map(cuda, src, dst, entry):
    """Every output pixel of the frame resize reads the source pixel torch's nearest rule picks (VaeImageProcessor.resize ->
    F.interpolate(size=...)): min(floor(dst * fp32(in / out)), in - 1).  The frame encodes each pixel's coordinates and the
    conv copies them through (centre-tap identity weights), so the decoded output is the index map itself.  Catches the
    exact-integer rule floor(dst * in / out): 800 -> 768 differs from torch on 7 rows / columns, 720 -> 448 on row 308."""
    ops = _ops()
    frame = _coordinate_frame(*src)
    if entry == "u8":
        x, flags = frame.to(cuda), 1
    else:   # the (3, H, W) float entries; the wrapper reads (nb, in_h, in_w, cin) from the shape, the data stays NCHW
        dt, flags = (torch.float32, 8) if entry == "f32" else (torch.float16, 16)
        x = (frame.permute(0, 3, 1, 2).double() / 255.0).to(dt).contiguous().to(cuda).permute(0, 2, 3, 1)
    w = torch.zeros((16, 3, 3, 3), dtype=torch.float16, device=cuda)
    w[[0, 1, 2], [0, 1, 2], 1, 1] = 1.0
    y = torch.full((1, *dst, 16), float("nan"), dtype=torch.float16, device=cuda)
    ops.smallconv(x, w, None, y, flags=flags)
    code = (y[0, ..., :3].double() * 255.0).round().long().cpu()
    got = torch.stack([code[..., 1] | (code[..., 2] >> 4) << 8, code[..., 0] | (code[..., 2] & 15) << 8])
    ref = _nearest_index_map(src, dst, "cpu")
    assert torch.equal(ref, _nearest_index_map(src, dst, cuda)), "torch's CPU and CUDA nearest rules disagree"
    integer = _integer_rule_map(src, dst)
    assert torch.equal(integer, ref) == ((src, dst) == _EXACT_RATIO), "the pair cannot tell the integer rule from torch's"
    bad_rows = (got[0] != ref[0]).any(1).nonzero().flatten().tolist()
    bad_cols = (got[1] != ref[1]).any(0).nonzero().flatten().tolist()
    assert torch.equal(got, ref), (f"{entry} {src} -> {dst}: source rows differ at output rows {bad_rows[:16]}, source columns "
                                   f"at output columns {bad_cols[:16]}")


@pytest.mark.parametrize("head", ["silu", "offset"])
def test_smallconv_ext_heads_resize(cuda, head):
    """The epilogue instantiations read the frame through the same resize: the ControlNet conditioning embedding's conv_in (u8,
    SiLU) and HED's first conv (u8 minus per-channel offsets, ReLU), on a 400x300 noise frame into a 192x128 engine, against a
    float64 conv of the frame resized by torch.  Catches the exact-integer resize rule (3 source columns differ)."""
    ops = _ops()
    from oracle import weights as ow
    src, dst = (300, 400), (128, 192)
    frame = ow.make_frame(*src, seed=31, smooth=False)
    g = torch.Generator().manual_seed(32)

    def resized(m):   # float64 NCHW [1, 3, h, w] of the frame read through the index map m
        return frame[0][m[0], m[1]].permute(2, 0, 1)[None].double().to(cuda)
    if head == "silu":
        wt = (torch.randn((16, 3, 3, 3), generator=g) * 0.8).half().to(cuda)
        bias = (torch.randn(16, generator=g) * 0.5).float().to(cuda)
        out = torch.full((1, *dst, 16), float("nan"), dtype=torch.float16, device=cuda)
        ops.smallconv_ex(frame.to(cuda), wt, bias, out, flags=1 | 32)
        tol = (2e-3, 4e-3)

        def f(m):
            x = (resized(m) / 255.0).half().double()
            return F.silu(F.conv2d(x, wt.double(), bias.double(), padding=1)).permute(0, 2, 3, 1)
    else:
        off = torch.tensor([117.0, 104.5, 96.25], device=cuda)
        wt = (torch.randn((64, 3, 3, 3), generator=g) * 0.2).half().to(cuda)
        bias = (torch.randn(64, generator=g) * 0.5).float().to(cuda)
        out = torch.full((1, *dst, 64), float("nan"), dtype=torch.float16, device=cuda)
        ops.smallconv_ex(frame.to(cuda), wt, bias, out, flags=1 | 4 | 64, in_off=off)
        tol = (5e-2, 4e-3)

        def f(m):
            x = (resized(m) - off.double().view(1, 3, 1, 1)).half().double()
            return F.relu(F.conv2d(x, wt.double(), bias.double(), padding=1)).permute(0, 2, 3, 1)
    ref, wrong = f(_nearest_index_map(src, dst, "cpu")), f(_integer_rule_map(src, dst))
    assert_discriminates(out, ref, wrong, *tol, f"smallconv {head} head, {src} -> {dst}", bug="exact-integer resize rule")


def test_smallconv_taesd_decoder_head(cuda):
    ops = _ops()
    z = (_rand((1, 16, 16, 4), cuda, 1) * 2).half()
    w = _rand((64, 4, 3, 3), cuda, 2, 1 / 6.0).half()
    b = _rand((64,), cuda, 3).float()
    y = torch.empty((1, 16, 16, 64), dtype=torch.float16, device=cuda)
    ops.smallconv(z, w, b, y, flags=2 | 4)
    x = (torch.tanh(z.float() / 3) * 3).half().float()
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2), w.float(), b, padding=1)).permute(0, 2, 3, 1)
    assert_close(y, ref, 2e-3, 2e-3, "taesd decoder head")


@pytest.mark.parametrize("T", [1, 4])
def test_lcm_step_matches_streamdiffusion(cuda, T):
    """scheduler_step_batch + buffer update vs the oracle restatement (oracle/stream.py)."""
    ops = _ops()
    from oracle import stream as ostream
    hw = (8, 8)
    t_list = [18, 26, 35, 45][:T] if T > 1 else [32]
    so = ostream.StreamOracle({}, None, {}, t_list, 64, 64)
    so.prepare(torch.zeros(1, 77, 8), guidance_scale=0.0)
    x = _rand((T, 4, *hw), "cpu", 1).half().float()
    eps = _rand((T, 4, *hw), "cpu", 2).half().float()
    so.init_noise = so.init_noise.half().float()
    x0 = so.scheduler_step_batch(eps, x)
    coef = torch.stack([so.alpha_prod_t_sqrt.flatten(), so.beta_prod_t_sqrt.flatten(), so.c_skip.flatten(),
                        so.c_out.flatten()]).float().contiguous().to(cuda)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().half().to(cuda)
    xd, ed, nd = nhwc(x), nhwc(eps), nhwc(so.init_noise)
    outd = torch.empty((1, *hw, 4), dtype=torch.float16, device=cuda)
    ops.lcm_step(xd, ed, nd, coef, outd)
    assert_close(outd[0].permute(2, 0, 1), x0[-1], 2e-3, 2e-3, "x0 of the last slot")
    if T > 1:
        buf = so.alpha_prod_t_sqrt[1:] * x0[:-1] + so.beta_prod_t_sqrt[1:] * so.init_noise[1:]
        assert_close(xd[1:].permute(0, 3, 1, 2), buf, 2e-3, 2e-3, "x_t_latent_buffer")


def test_post_u8_truncation_semantics(cuda):
    """fp16 chain of DecoderTiny tail, postprocess_image and lib/pipeline.py:72-74: bit exact vs torch half ops."""
    ops = _ops()
    y = (_rand((1, 32, 32, 3), cuda, 1) * 0.4 + 0.5).half()
    y[0, 0, 0, 0] = 1.7   # clamps
    y[0, 0, 1, 0] = -0.3
    out = torch.empty((1, 3, 32, 32), dtype=torch.uint8, device=cuda)
    ops.post_u8(y, out)
    img = y.permute(0, 3, 1, 2).mul(2).sub(1)           # fp16
    den = (img / 2 + 0.5).clamp(0, 1)                   # fp16
    ref = (den * 255.0).clamp(0, 255).to(torch.uint8)   # truncation
    assert torch.equal(out, ref), f"mismatch {(out != ref).sum().item()} px"


# ---- codec boundary (SURVEY 8f-1): NV12 <-> RGB colour conversion next to NVDEC / NVENC -----------------------------------
def _csc_ref(flags):
    kr, kb = (0.299, 0.114) if flags & 1 else (0.2126, 0.0722)
    yo, ys, cs = (0.0, 1.0, 1.0) if flags & 2 else (16.0, 219.0 / 255.0, 224.0 / 255.0)
    return kr, 1.0 - kr - kb, kb, yo, ys, cs


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
@pytest.mark.parametrize("h,w", [(64, 96), (512, 512), (30, 50)])
def test_nv12_rgb_colour_conversion(cuda, flags, h, w):
    """Both directions against the textbook BT.709 / BT.601 matrices (limited and full range), 2x2 chroma averaging."""
    from ai_rtc_agent_b200.host import codec
    g = torch.Generator().manual_seed(7)
    rgb = torch.randint(0, 256, (1, 3, h, w), dtype=torch.uint8, generator=g)
    kr, kg, kb, yo, ys, cs = _csc_ref(flags)
    r, gg, b = (rgb[0, i].double() for i in range(3))
    yl = kr * r + kg * gg + kb * b
    y_ref = (yo + ys * yl).round().clamp(0, 255)
    cb = (b - yl) / (2 * (1 - kb))
    cr = (r - yl) / (2 * (1 - kr))
    pool = lambda t: torch.nn.functional.avg_pool2d(t[None, None], 2, ceil_mode=True, count_include_pad=False)[0, 0]
    cb_ref = (128 + cs * pool(cb)).round().clamp(0, 255)
    cr_ref = (128 + cs * pool(cr)).round().clamp(0, 255)
    y, uv = codec.rgb_to_nv12(rgb.to(cuda), flags)
    assert (y.cpu().double() - y_ref).abs().max() <= 1
    assert (uv.cpu()[:, 0::2].double()[:, :cb_ref.shape[1]] - cb_ref).abs().max() <= 1
    assert (uv.cpu()[:, 1::2].double()[:, :cr_ref.shape[1]] - cr_ref).abs().max() <= 1
    # decode direction: exact formula on the encoder's planes
    back = codec.nv12_to_rgb(y, uv, flags).cpu()[0].double()      # (H,W,3)
    yy = (y.cpu().double() - yo) / ys
    up = lambda t: t.repeat_interleave(2, 0).repeat_interleave(2, 1)[:h, :w]
    cbd = up((uv.cpu()[:, 0::2].double() - 128) / cs)
    crd = up((uv.cpu()[:, 1::2].double() - 128) / cs)
    rr = yy + 2 * (1 - kr) * crd
    bb = yy + 2 * (1 - kb) * cbd
    gr = (yy - kr * rr - kb * bb) / kg
    ref = torch.stack([rr, gr, bb], dim=-1).round().clamp(0, 255)
    assert (back - ref).abs().max() <= 1
    # a smooth image survives the round trip closely (chroma sub-sampling aside)
    xs = torch.linspace(0, 255, w)[None, :].expand(h, w)
    smooth = torch.stack([xs, xs.flip(1), torch.full_like(xs, 128.0)]).round().to(torch.uint8)[None]
    ys_, uvs = codec.rgb_to_nv12(smooth.to(cuda), flags)
    rt = codec.nv12_to_rgb(ys_, uvs, flags).cpu()[0].permute(2, 0, 1).double()
    assert (rt - smooth[0].double()).abs().max() <= 6     # 2x2 chroma averaging of a 5-levels-per-pixel ramp + two roundings


def test_codec_sessions_report_unavailable(cuda):
    from ai_rtc_agent_b200.host import codec
    libs = codec.codec_libraries()
    assert set(libs) == {"nvdec", "nvenc"}
    with pytest.raises(codec.CodecUnavailable):
        codec.open_decoder()
    with pytest.raises(codec.CodecUnavailable):
        codec.open_encoder()
