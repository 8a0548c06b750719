"""The launch audit's descriptor-driven references (tests/launch_ref.py) against independent torch.nn computations, on small
synthetic descriptors.  CPU only: the audit trusts these references, so they are checked where no kernel is involved."""
import math

import torch
import torch.nn.functional as F

from tests import launch_ref as R


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64) * scale


def _view(x):
    n, h, w, c = x.shape
    return {"ptr": 0, "n": n, "h": h, "w": w, "c": c, "ld": c}


def _desc(srcs, ntaps, w, nb, ho, wo, n_valid, **kw):
    d = {"src": [_view(x) for x in srcs], "ntap": list(ntaps), "nseg": len(srcs), "w_rows": w.shape[0], "w_ld": w.shape[1],
         "stride": 1, "nb": nb, "ho": ho, "wo": wo, "bn": 64, "splits": 1, "colbias_bstride": 0, "acc_scale": 1.0,
         "res_scale": 1.0, "flags": 0, "n_valid": n_valid, "swap": 0, "ln_c": 0, "ln_eps": 1e-5, "out2": 0, "ld2": 0, "col2": 0}
    d.update(kw)
    return d


def _pack(w_oihw):
    """OIHW conv weight -> packed [n][tap][c] rows"""
    n, c, kh, kw = w_oihw.shape
    return w_oihw.permute(0, 2, 3, 1).reshape(n, kh * kw * c)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _rows(y_nchw):
    return y_nchw.permute(0, 2, 3, 1).reshape(-1, y_nchw.shape[1])


def test_three_segment_conv_with_shortcut():
    """conv3x3 over the concat [x1 | x2] plus a 1x1 shortcut over x3 as a third K segment, per-image bias, acc/res scales,
    residual and ReLU: the UNet's up-block resnet conv2 shape."""
    nb, h, w, n = 2, 5, 7, 48
    x1, x2, x3 = _rand((nb, h, w, 64), 1), _rand((nb, h, w, 128), 2), _rand((nb, h, w, 64), 3)
    wa, ws = _rand((n, 192, 3, 3), 4, 0.05), _rand((n, 64, 1, 1), 5, 0.1)
    wp = torch.cat([_pack(wa[:, :64]), _pack(wa[:, 64:]), _pack(ws)], dim=1)
    bias = _rand((nb * 64,), 6)
    res = _rand((nb * h * w, n), 7)
    d = _desc([x1, x2, x3], [9, 9, 1], wp, nb, h, w, n, colbias_bstride=64, acc_scale=0.7, res_scale=1.3, flags=R.IG_RELU)
    got = R.contraction_ref(d, {"src": [x1, x2, x3], "w": wp, "colbias": bias, "res": res})
    ref = F.conv2d(_nchw(torch.cat([x1, x2], dim=3)), wa, padding=1) + F.conv2d(_nchw(x3), ws)
    ref = ref + bias.reshape(nb, 64)[:, :n, None, None]
    ref = F.relu(0.7 * _rows(ref) + 1.3 * res)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    wrong = R.contraction_ref(d, {"src": [x1, x2, x3], "w": wp, "colbias": bias, "res": res}, bias0=True)
    assert (wrong[h * w:] - ref[h * w:]).abs().max() > 0.1 and torch.equal(wrong[:h * w], got[:h * w])


def test_stride2_and_tap_origin_zero():
    """stride-2 3x3 with zero padding on both sides (UNet downsamplers) and with the AutoencoderKL's F.pad(x, (0,1,0,1))."""
    nb, h, w, c, n = 1, 9, 12, 64, 32
    x = _rand((nb, h, w, c), 8)
    wt = _rand((n, c, 3, 3), 9, 0.05)
    for pad0 in (False, True):
        ho, wo = ((h - 2) // 2 + 1, (w - 2) // 2 + 1) if pad0 else ((h + 1) // 2, (w + 1) // 2)
        d = _desc([x], [9], _pack(wt), nb, ho, wo, n, stride=2, flags=R.IG_PAD0 if pad0 else 0)
        got = R.contraction_ref(d, {"src": [x], "w": _pack(wt)})
        xin = F.pad(_nchw(x), (0, 1, 0, 1)) if pad0 else _nchw(x)
        ref = _rows(F.conv2d(xin, wt, stride=2, padding=0 if pad0 else 1))
        assert ref.shape == got.shape
        torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def test_geglu_interleave_bn128():
    """GEGLU over weight rows interleaved per 128-wide N tile as [64 value rows | 64 gate rows], with the bias interleaved
    alike: out = (x Wv^T + bv) * gelu_erf(x Wg^T + bg), as diffusers' GEGLU computes."""
    m, c, inner = 40, 64, 256
    x = _rand((1, 1, m, c), 10)
    wv, wg = _rand((inner, c), 11, 0.2), _rand((inner, c), 12, 0.2)
    bv, bg = _rand((inner,), 13), _rand((inner,), 14)
    perm = []
    for t in range(inner // 64):
        perm += list(range(t * 64, t * 64 + 64)) + list(range(inner + t * 64, inner + t * 64 + 64))
    wp = torch.cat([wv, wg])[perm]
    bp = torch.cat([bv, bg])[perm]
    d = _desc([x], [1], wp, 1, 1, m, inner, bn=128, flags=R.IG_GEGLU)
    got = R.contraction_ref(d, {"src": [x], "w": wp, "colbias": bp})
    xx = x.reshape(m, c)
    ref = F.linear(xx, wv, bv) * F.gelu(F.linear(xx, wg, bg))
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def _fixed_point_stats(x):
    s1 = torch.round(x.sum(1) * R.STAT_SCALE)
    s2 = torch.round((x * x).sum(1) * R.STAT_SCALE)
    return torch.stack([s1, s2], dim=1).to(torch.int64)


def test_layernorm_fold_equals_layernorm_then_linear():
    """The folded LayerNorm: weights W diag(gamma), colsum = row sums of those, bias' = W beta + b, statistics from the
    producer's fixed-point sums -> F.layer_norm followed by F.linear."""
    m, c, n = 24, 128, 96
    x = _rand((m, c), 15) * 2 + _rand((m, 1), 16) * 3
    gamma, beta = 1 + 0.3 * _rand((c,), 17), 0.5 * _rand((c,), 18)
    W, b = _rand((n, c), 19, 0.1), _rand((n,), 20)
    wf = W * gamma[None]
    d = _desc([x.reshape(1, 1, m, c)], [1], wf, 1, 1, m, n, ln_c=c, ln_eps=1e-5)
    snap = {"src": [x.reshape(1, 1, m, c)], "w": wf, "colbias": W @ beta + b, "colsum": wf.sum(1),
            "rowstat_in": _fixed_point_stats(x)}
    got = R.contraction_ref(d, snap)
    ref = F.linear(F.layer_norm(x, (c,), gamma, beta, 1e-5), W, b)
    torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6)
    wrong = R.contraction_ref(d, snap, stats_shift=True)
    assert (wrong - ref).abs().max() > 1.0


def test_out2_split_is_the_transposed_v_block():
    """Fused [q | k | v] projection: columns >= col2 go to out2 transposed (V^T, token index contiguous)."""
    m, c, cp = 20, 64, 64
    x = _rand((1, 1, m, c), 21)
    w = _rand((3 * cp, c), 22, 0.1)
    d = _desc([x], [1], w, 1, 1, m, 3 * cp, out2=1, col2=2 * cp, ld2=24)
    main, vt = R.split_out2(d, R.contraction_ref(d, {"src": [x], "w": w}))
    xx = x.reshape(m, c)
    torch.testing.assert_close(main, xx @ w[:2 * cp].T, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(vt, (xx @ w[2 * cp:].T).T, rtol=1e-12, atol=1e-12)


def test_attention_unequal_batch_strides_and_padded_heads():
    """Self-attention of the unfolded transformer program: K rows at b * HW, V^T columns at b * HWp (HWp = HW rounded up to 8),
    heads of 40 zero-padded to 64, softmax scale 40^-0.5."""
    nb, heads, hw, d, dp = 3, 2, 36, 40, 64
    hwp = 40
    q, k, v = _rand((nb, heads, hw, d), 23), _rand((nb, heads, hw, d), 24), _rand((nb, heads, hw, d), 25)
    qb = torch.zeros(nb * hw, heads * dp, dtype=torch.float64)
    kb = torch.zeros(nb * hw, heads * dp, dtype=torch.float64)
    vt = torch.full((heads * dp, nb * hwp), 1e3, dtype=torch.float64)   # pad columns: poison the skv bound keeps out
    for h in range(heads):
        qb[:, h * dp:h * dp + d] = q[:, h].reshape(nb * hw, d)
        kb[:, h * dp:h * dp + d] = k[:, h].reshape(nb * hw, d)
        vt[h * dp:(h + 1) * dp] = 0
        for b in range(nb):
            vt[h * dp:h * dp + d, b * hwp:b * hwp + hw] = v[b, h].T
    a = {"nb": nb, "heads": heads, "sq": hw, "skv": hw, "d_real": d, "dp": dp, "k_bstride": hw, "vt_bstride": hwp}
    got = R.attention_ref(a, qb, kb, vt, qchunk=16)
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(nb * hw, heads * d)
    torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-10)
    for wrong in (R.attention_ref(a, qb, kb, vt, kv_item0=True), R.attention_ref(a, qb, kb, vt, dp_scale=True),
                  R.attention_ref(a, qb, kb, vt, drop_last_block=32)):
        assert (wrong - ref).abs().max() > 0.05


def test_groupnorm_groups_straddle_the_concat():
    """GroupNorm(+SiLU) over [xa | xb] with a group that takes channels from both sources (ca = 36, 8 channels per group)."""
    nb, hw, ca, cb, G = 2, 10, 36, 92, 16
    xa, xb = _rand((nb * hw, ca), 26) + 2, _rand((nb * hw, cb), 27) * 3
    gamma, beta = 1 + 0.2 * _rand((ca + cb,), 28), _rand((ca + cb,), 29)
    g = {"nb": nb, "hw": hw, "groups": G, "eps": 1e-6, "silu": 1}
    got = R.groupnorm_ref(g, xa, xb, gamma, beta)
    x = torch.cat([xa, xb], dim=1).reshape(nb, hw, ca + cb).permute(0, 2, 1)
    ref = F.silu(F.group_norm(x, G, gamma, beta, 1e-6)).permute(0, 2, 1).reshape(nb * hw, ca + cb)
    torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-10)
    assert (R.groupnorm_ref(g, xa, xb, gamma, beta, shift_groups=True) - ref).abs().max() > 0.1


def test_layernorm_reference():
    rows, c = 12, 96
    x = _rand((rows, c), 30) + _rand((rows, 1), 31) * 4
    gamma, beta = 1 + 0.2 * _rand((c,), 32), _rand((c,), 33)
    got = R.layernorm_ref({"eps": 1e-5}, x, gamma, beta)
    torch.testing.assert_close(got, F.layer_norm(x, (c,), gamma, beta, 1e-5), rtol=1e-10, atol=1e-10)
    assert (R.layernorm_ref({"eps": 1e-5}, x, gamma, beta, shift_rows=True) - got).abs().max() > 0.5


def test_tolerance_units():
    ref = torch.tensor([1.0, -1.0, 0.0, 2.0], dtype=torch.float64)
    rms = math.sqrt(6 / 4)
    got = ref.clone()
    got[2] = 3e-3 * rms
    assert abs(R.tol_units(got, ref, 3e-3, 3e-3) - 1.0) < 1e-9
    got[0] = float("nan")
    assert R.tol_units(got, ref, 3e-3, 3e-3) == float("inf")


# ---- the elementwise kernels and the prepare-time launches ------------------------------------------------------------------
def _sc_args(nb, h, w, cin, cout, in_h, in_w, flags, res_bstride=0):
    return {"nb": nb, "h": h, "w": w, "cin": cin, "cout": cout, "in_h": in_h, "in_w": in_w, "flags": flags,
            "res_bstride": res_bstride}


def _wt(w_oihw):
    """OIHW -> smallconv's prepared fp32 [cin*9][cout], k = tap*cin + c"""
    o, c = w_oihw.shape[:2]
    return w_oihw.permute(2, 3, 1, 0).reshape(9 * c, o)


def test_smallconv_u8_head_with_resize():
    """u8 NHWC frame / 255 (rounded to fp16), resized 720x20 -> 448x12 with torch's nearest rule, 3x3 conv + bias + ReLU ->
    F.interpolate(size=...) + F.conv2d.  720 -> 448 is a pair where torch's rule and the exact-integer rule differ."""
    g = torch.Generator().manual_seed(40)
    x = torch.randint(0, 256, (1, 720, 20, 3), generator=g, dtype=torch.uint8)
    w, b = _rand((64, 3, 3, 3), 41, 0.3), _rand((64,), 42)
    a = _sc_args(1, 448, 12, 3, 64, 720, 20, R.SC_IN_U8 | R.SC_OUT_RELU)
    got = R.smallconv_ref(a, x, _wt(w), b)
    v = (x.float() * (1.0 / 255.0)).half().float().permute(0, 3, 1, 2)   # fp32: torch's rule for float64 scales in float64
    ref = _rows(F.relu(F.conv2d(F.interpolate(v, size=(448, 12), mode="nearest").double(), w, b, padding=1)))
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    assert not torch.equal(R.nearest_index(720, 448), R.nearest_index(720, 448, exact_integer=True))
    assert (R.smallconv_ref(a, x, _wt(w), b, exact_integer=True) - ref).abs().max() > 0.1
    assert (R.smallconv_ref(a, x, _wt(w), b, mirrored=True) - ref).abs().max() > 0.1


def test_smallconv_offset_input_pads_in_the_shifted_domain():
    """HED's first conv / the AutoencoderKL head: u8 - in_off[c], zero padding applied after the shift; SiLU epilogue."""
    g = torch.Generator().manual_seed(43)
    x = torch.randint(0, 256, (1, 9, 11, 3), generator=g, dtype=torch.uint8)
    off = torch.tensor([122.7, 116.6, 104.0])
    w, b = _rand((16, 3, 3, 3), 44, 0.02), _rand((16,), 45)
    a = _sc_args(1, 9, 11, 3, 16, 9, 11, R.SC_IN_U8 | R.SC_IN_OFFSET | R.SC_OUT_SILU)
    got = R.smallconv_ref(a, x, _wt(w), b, in_off=off)
    v = (x.float() - off).half().double().permute(0, 3, 1, 2)
    ref = _rows(F.silu(F.conv2d(v, w, b, padding=1)))
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    wrong = R.smallconv_ref(a, x, _wt(w), b, in_off=off, offset_after_pad=True).reshape(9, 11, 16)
    assert (wrong - ref.reshape(9, 11, 16))[0].abs().max() > 0.1                                # the border moves
    torch.testing.assert_close(wrong[1:-1, 1:-1], ref.reshape(9, 11, 16)[1:-1, 1:-1], rtol=1e-12, atol=1e-12)


def test_smallconv_fp16_tanh_input_and_per_item_residual():
    """fp16 latent through tanh(x/3)*3 (DecoderTiny), per-item residual (item n at n * res_bstride), batch 2."""
    nb, h, w = 2, 6, 5
    x = (_rand((nb, h, w, 4), 46) * 4).half()
    wc, b = _rand((32, 4, 3, 3), 47, 0.2), _rand((32,), 48)
    res = _rand((nb, h * w, 32), 49).half()
    a = _sc_args(nb, h, w, 4, 32, h, w, R.SC_IN_TANH3, res_bstride=h * w * 32)
    got = R.smallconv_ref(a, x, _wt(wc), b, res=res)
    v = (torch.tanh(x.float() / 3) * 3).half().double().permute(0, 3, 1, 2)
    ref = _rows(F.conv2d(v, wc, b, padding=1)) + res.double().reshape(nb * h * w, 32)
    torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6)   # fp32 tanh vs the fp32 x/3 product: rare fp16 ties
    assert (R.smallconv_ref(a, x, _wt(wc), b, res=res, res_item0=True) - ref)[h * w:].abs().max() > 0.1
    assert (R.smallconv_ref(a, x, _wt(wc), b, res=res, no_res=True) - ref).abs().max() > 0.1


def _frac_differ(a, b):
    return (a != b).double().mean().item()


def test_upsample2x_and_maxpool2x2():
    x = _rand((2, 5, 7, 16), 50).half()
    ref = F.interpolate(x.permute(0, 3, 1, 2).double(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    got = R.upsample2x_ref(x)
    assert torch.equal(got.double(), ref)
    assert _frac_differ(R.upsample2x_ref(x, shifted=True), got) >= 0.01
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).double(), 2).permute(0, 2, 3, 1)
    got = R.maxpool2x2_ref(x[:, :4, :6])
    assert torch.equal(got.double(), F.max_pool2d(x[:, :4, :6].permute(0, 3, 1, 2).double(), 2).permute(0, 2, 3, 1))
    assert ref.shape[1] == 2 and got.shape[1:3] == (2, 3)
    for wrong in (R.maxpool2x2_ref(x[:, :4, :6], average=True), R.maxpool2x2_ref(x[:, :4, :6], shifted=True)):
        assert _frac_differ(wrong, got) >= 0.01


def test_hed_project_reference():
    x, w, b = _rand((40, 64), 51).half(), _rand((64,), 52), _rand((1,), 53)
    got = R.hed_project_ref(x, w, b)
    ref = F.conv2d(x.double().T.reshape(1, 64, 40, 1), w.reshape(1, 64, 1, 1), b).reshape(40)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    for wrong in (R.hed_project_ref(x, w, b, no_bias=True), R.hed_project_ref(x, w, b, swap_pairs=True)):
        assert (wrong - ref).abs().max() > 0.1


def test_hed_fuse_matches_the_oracle_post_processing(monkeypatch):
    """Five side outputs at h / 2^k -> oracle/hed.py's detect tail (F.interpolate bilinear, align_corners=False, mean,
    sigmoid, * 255, clamp, u8 cast); the oracle's own code, fed these maps."""
    from oracle import hed as ohed
    h, w = 48, 80
    maps = [_rand((h >> k, w >> k), 54 + k, 2.0) for k in range(5)]
    monkeypatch.setattr(ohed, "side_outputs", lambda sd, x: [m[None, None] for m in maps])
    ref = ohed.detect(None, torch.zeros(1, 3, h, w, dtype=torch.float64))[0, 0]
    got = R.hed_fuse_ref(maps, h, w)
    assert torch.equal(got, ref)
    assert R.hed_fuse_mismatch(got, maps, h, w) == (0, True)
    for wrong in (R.hed_fuse_ref(maps, h, w, align_corners=True), R.hed_fuse_ref(maps, h, w, rounding=True)):
        assert _frac_differ(wrong, got) >= 0.01


def test_lcm_step_matches_the_oracle_scheduler_and_buffer_update():
    """oracle/stream.py scheduler_step_batch + predict_x0_batch's buffer update (T = 4, with and without the noise term)."""
    from types import SimpleNamespace

    from oracle import stream as ostream
    T, h, w = 4, 3, 5
    x, eps, noise = (_rand((T, 4, h, w), s) for s in (60, 61, 62))
    coef = torch.cat([0.5 + 0.5 * torch.rand(T, dtype=torch.float64), 0.2 + 0.7 * torch.rand(T, dtype=torch.float64),
                      0.3 * torch.rand(T, dtype=torch.float64), 0.5 + torch.rand(T, dtype=torch.float64)])
    c = coef.reshape(4, T)
    for dan in (1, 0):
        ns = SimpleNamespace(denoising_steps_num=T, x_t_latent_buffer=x[1:].clone(), init_noise=noise,
                             stock_noise=noise.clone(), do_add_noise=bool(dan), static_buffers=False, last={},
                             alpha_prod_t_sqrt=c[0].view(T, 1, 1, 1), beta_prod_t_sqrt=c[1].view(T, 1, 1, 1),
                             c_skip=c[2].view(T, 1, 1, 1), c_out=c[3].view(T, 1, 1, 1))
        ns.unet_step = lambda xx, ns=ns: (ostream.StreamOracle.scheduler_step_batch(ns, eps, xx), eps)
        out = ostream.StreamOracle.predict_x0_batch(ns, x[:1])

        def flat(t):
            return t.permute(0, 2, 3, 1).reshape(t.shape[0], h * w, 4)
        a = {"T": T, "do_add_noise": dan}
        got_out, got_x = R.lcm_step_ref(a, flat(x), flat(eps), flat(noise), coef)
        torch.testing.assert_close(got_out, flat(out)[0], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(got_x[1:], flat(ns.x_t_latent_buffer), rtol=1e-12, atol=1e-12)
        assert torch.equal(got_x[0], flat(x)[0])
        w_out, _ = R.lcm_step_ref(a, flat(x), flat(eps), flat(noise), coef, swap_cskip_cout=True)
        _, w_x = R.lcm_step_ref(a, flat(x), flat(eps), flat(noise), coef, own_x0=True)
        assert (w_out - got_out).abs().max() > 0.1 and (w_x - got_x).abs().max() > 0.1


def test_post_u8_matches_torch_half_ops():
    nb, h, w = 2, 16, 24
    y = (torch.rand(nb * h * w, 3, generator=torch.Generator().manual_seed(63), dtype=torch.float64) * 1.4 - 0.2).half()
    y[:6, 0] = torch.tensor([-0.5, 0.0, 0.5, 1.0, 1.5, 0.25], dtype=torch.float16)
    a = {"nb": nb, "h": h, "w": w}
    got = R.post_u8_ref(a, y)
    v = y.reshape(nb, h, w, 3).permute(0, 3, 1, 2)
    v = v * 2 - 1
    v = v / 2 + 0.5
    v = v.clamp(0, 1) * 255
    ref = v.clamp(0, 255).to(torch.uint8)
    assert v.dtype == torch.float16 and torch.equal(got, ref)
    for wrong in (R.post_u8_ref(a, y, rounding=True), R.post_u8_ref(a, y, bgr=True)):
        assert _frac_differ(wrong, got) >= 0.01


def test_timestep_embedding_and_time_mlp_match_the_oracle():
    """timestep_embedding vs oracle.unet.timestep_embedding; the time MLP (linear_1, SiLU, linear_2) as two small_linear
    launches vs oracle.unet.time_embed; a resnet's time bias conv1.bias + time_emb_proj(silu(emb)) vs F.linear."""
    from oracle import unet as ounet
    t = torch.tensor([999.0, 261.0, 35.0, 1.0])
    c0 = 64
    emb = R.timestep_embedding_ref(t, c0)
    torch.testing.assert_close(emb, ounet.timestep_embedding(t, c0).double(), rtol=0, atol=R.TEMB_ATOL)
    for wrong in (R.timestep_embedding_ref(t, c0, sin_first=True), R.timestep_embedding_ref(t, c0, half_minus_one=True)):
        assert (wrong - emb).abs().max() > 0.1
    td = 4 * c0
    sd = {"time_embedding.linear_1.weight": _rand((td, c0), 64, 0.2).half().double(),
          "time_embedding.linear_1.bias": _rand((td,), 65), "time_embedding.linear_2.weight": _rand((td, td), 66, 0.1).half().double(),
          "time_embedding.linear_2.bias": _rand((td,), 67)}
    l1 = {"k": c0, "silu_in": 0}
    l2 = {"k": td, "silu_in": 1}
    hid = R.small_linear_ref(l1, emb, sd["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.bias"])
    out = R.small_linear_ref(l2, hid, sd["time_embedding.linear_2.weight"], sd["time_embedding.linear_2.bias"])
    torch.testing.assert_close(out, ounet.time_embed(sd, ounet.tiny_config(True), t), rtol=1e-4, atol=1e-4)
    wp, bp = _rand((128, td), 68, 0.1).half(), _rand((128,), 69)
    bias = R.small_linear_ref(l2, out, wp, bp)
    torch.testing.assert_close(bias, F.linear(F.silu(out), wp.double(), bp), rtol=1e-12, atol=1e-12)
    for kw in ({"no_silu": True}, {"no_bias": True}, {"slot0": True}):
        assert (R.small_linear_ref(l2, out, wp, bp, **kw) - bias).abs().max() > 0.1
