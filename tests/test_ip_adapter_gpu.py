"""IP-Adapter on the GPU: the decoupled cross-attention kernel (b2sd_op_attention_ip) against a float64 reference, and the
engine's image prompts (global and per state) against the fp32 oracle and against plain engines.

Op level: out = softmax(Q K^T / sqrt(d)) V + softmax(Q Kip^T / sqrt(d)) Vip, the image softmax over the first n_ip of a
64-key block whose other keys are poison; every case prints by how much the reference rejects each named wrong variant."""
import math

import pytest
import torch

from tests.util import assert_discriminates, guarded, hetero

pytestmark = pytest.mark.gpu

ATTN_TOL = (2e-3, 4e-3)   # as the text-only attention's parity tests: fp16 operands, P rounded to fp16 before P.V


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


def _q_layout(x, dp):
    """[nb,heads,s,d] -> [nb*s, heads*dp], each head zero-padded to dp"""
    nb, heads, s, d = x.shape
    xp = torch.zeros(nb, s, heads, dp, dtype=torch.float16, device=x.device)
    xp[..., :d] = x.permute(0, 2, 1, 3)
    return xp.reshape(nb * s, heads * dp)


def _vt_layout(v, dp, cols):
    """[1,heads,s,d] -> V^T [heads*dp, cols]"""
    _, heads, s, d = v.shape
    vt = torch.zeros(heads, dp, cols, dtype=torch.float16, device=v.device)
    vt[:, :d, :s] = v[0].permute(0, 2, 1)
    return vt.reshape(heads * dp, cols)


def _softmax_v(q, k, v, d):
    """float64 softmax(q k^T / sqrt(d)) v as [nb, heads, sq, d]"""
    s = q.double() @ k.double().transpose(-1, -2) / math.sqrt(d)
    return torch.softmax(s, dim=-1) @ v.double()


def _flat(o):
    return o.permute(0, 2, 1, 3).reshape(o.shape[0] * o.shape[2], -1)


# (d, dp, heads): SD-1.5's head dims 40 / 80 / 160 padded to 64 / 128 / 192, and SD-2.1's 64
HEADS = [(40, 64, 8), (64, 64, 5), (80, 128, 8), (160, 192, 8)]


@pytest.mark.parametrize("d,dp,heads", HEADS)
@pytest.mark.parametrize("n_ip", [1, 4, 16, 64])
@pytest.mark.parametrize("nb,sq", [(1, 576), (3, 100)])   # 576: a 24x24 latent level; 100: query tail in the one q tile
def test_attention_ip_against_float64(cuda, d, dp, heads, n_ip, nb, sq):
    """Text keys: the 77-token prompt cache shared by the batch.  Image keys: n_ip of a 64-key block shared by the batch, keys
    past n_ip poisoned in K (a logit of ~+30) and zero in V^T.  The image values are scaled by 0.7 (a folded IP scale)."""
    ops = _ops()
    skv = 77
    q = _rand((nb, heads, sq, d), cuda, 1) * 1.5
    q[..., 0] = 4.0
    q = q.half()
    k = _rand((1, heads, skv, d), cuda, 2)
    k[..., 0] = 0.0
    k = k.half()
    v = hetero((1, heads, skv, d), (1,), 3, cuda, scale=(0.5, 2.0))
    ki = _rand((1, heads, 64, d), cuda, 4, scale=1.3)
    ki[..., 0] = 0.0
    ki[:, :, n_ip:, 0] = 7.5 * math.sqrt(d)   # a logit of ~+30 for every query if the padding keys were read
    ki = ki.half()
    vi = (hetero((1, heads, 64, d), (1,), 5, cuda, scale=(0.5, 2.0)).float() * 0.7).half()
    vi[:, :, n_ip:] = 0
    kbuf = _q_layout(k, dp)
    vtbuf = _vt_layout(v, dp, 128)
    kip = _q_layout(ki, dp)
    vtip = _vt_layout(vi, dp, 64).contiguous()
    n_dev = torch.tensor([n_ip], dtype=torch.int32, device=cuda)
    out = guarded((nb * sq, heads * d), pitch=heads * d + 32, device=cuda)
    a = dict(nb=nb, heads=heads, sq=sq, skv=skv, d_real=d, dp=dp, k_bstride=0, vt_bstride=0)
    ops.attention_ip(_q_layout(q, dp), kbuf, vtbuf[:, :skv], out.view, kip, vtip, n_dev, **a)
    torch.cuda.synchronize()
    out.assert_untouched(f"attention_ip out d={d}/{dp}")
    txt = _softmax_v(q, k, v, d)
    img = _softmax_v(q, ki[:, :, :n_ip], vi[:, :, :n_ip], d)
    ref = _flat(txt + img)
    what = f"attention_ip nb={nb} sq={sq} heads={heads} d={d}/{dp} n_ip={n_ip}"
    kk, vv = torch.cat([k, ki[:, :, :n_ip]], 2), torch.cat([v, vi[:, :, :n_ip]], 2)
    wrong = {
        "image segment dropped": _flat(txt),
        "one softmax over text and image keys": _flat(_softmax_v(q, kk, vv, d)),
        "scale applied twice": _flat(txt + 0.7 * img),
    }
    if n_ip < 64:   # a full block has no padding keys
        wrong["padding keys not masked"] = _flat(txt + _softmax_v(q, ki, vi, d))
    margins = {}
    for bug, w in wrong.items():
        assert_discriminates(out.view, ref, w, *ATTN_TOL, what, bug)
        margins[bug] = ((w - ref).abs() / (ATTN_TOL[0] + ATTN_TOL[1] * ref.abs())).max().item()
    print(what + ": rejection margins " + ", ".join(f"{b}: {m:.0f}x" for b, m in margins.items()))


@pytest.mark.parametrize("d,dp,heads", HEADS)
def test_attention_ip_zero_tokens_is_bit_identical(cuda, d, dp, heads):
    """n_ip = 0 (an adapter engine without an image prompt) skips the segment: bit for bit the text-only kernel, however
    the image block's memory looks"""
    ops = _ops()
    nb, sq, skv = 2, 300, 77
    q = _q_layout((_rand((nb, heads, sq, d), cuda, 11) * 1.5).half(), dp)
    k = _q_layout(_rand((1, heads, skv, d), cuda, 12).half(), dp)
    vt = _vt_layout(_rand((1, heads, skv, d), cuda, 13).half(), dp, 128)[:, :skv]
    kip = torch.full((64, heads * dp), 30.0, dtype=torch.float16, device=cuda)
    vtip = torch.full((heads * dp, 64), 64.0, dtype=torch.float16, device=cuda)
    a = dict(nb=nb, heads=heads, sq=sq, skv=skv, d_real=d, dp=dp, k_bstride=0, vt_bstride=0)
    plain = torch.empty((nb * sq, heads * d), dtype=torch.float16, device=cuda)
    got = torch.empty_like(plain)
    ops.attention(q, k, vt, plain, **a)
    ops.attention_ip(q, k, vt, got, kip, vtip, torch.zeros(1, dtype=torch.int32, device=cuda), **a)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), plain.view(torch.int16)), f"n_ip = 0 differs from the text-only kernel (d={d}/{dp})"


def test_attention_ip_refuses_half_a_segment(cuda):
    import ctypes as C
    from ai_rtc_agent_b200.host import capi
    q = torch.zeros((128, 64), dtype=torch.float16, device=cuda)
    k = torch.zeros((77, 64), dtype=torch.float16, device=cuda)
    vt = torch.zeros((64, 128), dtype=torch.float16, device=cuda)[:, :77]
    kip = torch.zeros((64, 64), dtype=torch.float16, device=cuda)
    vtip = torch.zeros((64, 64), dtype=torch.float16, device=cuda)
    out = torch.empty((128, 64), dtype=torch.float16, device=cuda)
    d = capi.AttnDesc()
    d.q, d.ldq, d.k, d.ldk, d.k_rows, d.vt, d.ldvt, d.vt_cols = q.data_ptr(), 64, k.data_ptr(), 64, 77, vt.data_ptr(), 128, 77
    d.out, d.ldo, d.nb, d.heads, d.sq, d.skv, d.d_real, d.dp = out.data_ptr(), 64, 1, 1, 128, 77, 64, 64
    rc = capi.lib().b2sd_op_attention_ip(C.byref(d), kip.data_ptr(), vtip.data_ptr(), None, capi.current_stream_ptr())
    assert rc != 0 and b"n_ip" in capi.lib().b2sd_last_error()


# ---- engine ------------------------------------------------------------------------------------------------------------------------
T4 = [18, 26, 35, 45]


def _u8_check(got, ref, what):
    """the u8 tolerance of the engine's oracle parity: |d| <= 2 on >= 99.9 % of the values, max |d| <= 8"""
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"


def _adapter(arch):
    from ai_rtc_agent_b200.host import image_prompt as I
    return I.adapter_from_state_dict(I.synthetic_adapter_state_dict(arch), arch)


def _image(seed, hw=48):
    import numpy as np
    return np.random.default_rng(seed).integers(0, 256, (hw, hw, 3), dtype=np.uint8)


def _tiny(turbo, tl, adapter=True, cn=False, hed=False, hw=128, **kw):
    """(engine, oracle weights) of a tiny model: with an adapter, its to_k_ip / to_v_ip sit in the oracle's UNet weights"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    usd, vsd = ow.make_unet_weights(cfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    ad = _adapter(arch) if adapter else None
    cn16 = ocn.make_weights(cfg) if cn else None
    hed16 = {k: v.half().float() for k, v in A.synthetic_hed().items()} if hed else None
    sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, width=hw, height=hw, controlnet_sd=cn16, hed_sd=hed16, ip_adapter=ad,
                         **kw)
    sd.prepare("p", guidance_scale=0.0)
    return sd, dict(cfg=cfg, usd={**usd, **(ad.unet if ad else {})}, vsd=vsd, emb=emb, cn=cn16, hed=hed16, tl=tl, hw=hw)


def _oracle(sd, w):
    from oracle import controlnet as ocn
    from oracle import stream as ostream
    from oracle import weights as ow
    if w["cn"] is not None:
        orc = ocn.ControlNetStreamOracle(ow.to_float(w["usd"]), w["cfg"], ow.to_float(w["vsd"]), ow.to_float(w["cn"]), w["tl"],
                                         w["hw"], w["hw"], hed_sd=w["hed"])
    else:
        orc = ostream.StreamOracle(ow.to_float(w["usd"]), w["cfg"], ow.to_float(w["vsd"]), w["tl"], w["hw"], w["hw"])
    orc.prepare(w["emb"].float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    return orc


@pytest.mark.parametrize("control", [False, True], ids=["plain", "controlnet-hed"])
@pytest.mark.parametrize("turbo,tl", [(False, T4), (True, [32])], ids=["sd15-T4", "turbo-T1"])
def test_engine_image_prompt_matches_oracle(cuda, turbo, tl, control):
    """8 frames against the fp32 oracle with the same image tokens: frames 0-3 with image A at scale 1, frames 4-7 with image
    B at scale 0.6, both changes enqueued between queued frames (no synchronisation), and no graph recaptured"""
    from oracle import ip_adapter as OI
    from oracle import pipeline as opipe
    from oracle import weights as ow
    sd, w = _tiny(turbo, tl, cn=control, hed=control)
    orc = _oracle(sd, w)
    launches = sd.launches_per_step
    tok = [sd.image_tokens(_image(1)), sd.image_tokens(_image(2))]
    plan = [(tok[0], 1.0)] * 4 + [(tok[1], 0.6)] * 4
    frames = [ow.make_frame(128, 128, seed=40 + i) for i in range(8)]
    outs = []
    for i, (t, s) in enumerate(plan):
        if i in (0, 4):
            sd.set_image_tokens(t, s)
        outs.append(sd.step_u8(frames[i].to(cuda)))
    torch.cuda.synchronize()
    for i, (t, s) in enumerate(plan):
        with OI.image_prompt(t.float(), s):
            ref = opipe.frame_to_u8(orc, frames[i])
        _u8_check(outs[i], ref, f"frame {i}")
    assert sd.launches_per_step == launches
    plain = _oracle(sd, w)   # the image prompt changes the frames well beyond the tolerance
    d = (outs[0].cpu().int() - opipe.frame_to_u8(plain, frames[0]).int()).abs()
    assert d.max().item() > 8, "the image prompt must change the frame"


@pytest.mark.parametrize("turbo,tl", [(False, T4), (True, [32])], ids=["sd15-T4", "turbo-T1"])
def test_adapter_engine_without_image_prompt_is_bit_identical(cuda, turbo, tl):
    """An adapter engine with no image prompt bound (never, or set and cleared again) gives a plain engine's frames"""
    from oracle import weights as ow
    plain, _ = _tiny(turbo, tl, adapter=False)
    ip, _ = _tiny(turbo, tl)
    frames = [ow.make_frame(128, 128, seed=60 + i).to(cuda) for i in range(6)]
    for i, f in enumerate(frames):
        if i == 3:
            ip.set_image_tokens(ip.image_tokens(_image(3)), 0.8)
            ip.set_image_tokens(None)
        a, b = plain.step_u8(f), ip.step_u8(f)
        assert torch.equal(a, b), f"frame {i}"


def test_image_prompt_switches_keep_device_memory(cuda):
    """Twenty image-prompt switches, global and per state, leave cudaMemGetInfo unchanged"""
    from oracle import weights as ow
    sd, _ = _tiny(False, T4)
    st = sd.new_state()
    tok = [sd.image_tokens(_image(k)) for k in range(4)]
    f = ow.make_frame(128, 128, seed=7).to(cuda)

    def cycle(k):
        sd.set_image_tokens(tok[k % 4], 0.5 + 0.1 * (k % 3))
        st.set_image_tokens(tok[(k + 1) % 4], 0.9)
        sd.step_u8(f)
        sd.step_u8(f, state=st)
    for k in range(4):
        cycle(k)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(20):
        cycle(k)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


# ---- per viewer --------------------------------------------------------------------------------------------------------------------
def _pipe(model_id, tl, lanes, monkeypatch):
    from ai_rtc_agent_b200.host import weights as W
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    turbo = "turbo" in model_id
    cfg = ounet.tiny_config(turbo)
    W.register_preloaded(model_id, A.TINY_TURBO if turbo else A.TINY_SD15, ow.make_unet_weights(cfg), ow.make_taesd_weights())
    try:
        return StreamDiffusionPipeline(model_id, t_index_list=tl, width=128, height=128, lanes=lanes, live_lora=True,
                                       per_peer_streams=True, ip_adapter="synthetic")
    finally:
        W._PRELOADED.pop(model_id, None)


def _lora(tmp_path, turbo):
    from safetensors.torch import save_file
    from oracle import unet as ounet
    from oracle import weights as ow
    usd = ow.make_unet_weights(ounet.tiny_config(turbo))
    g = torch.Generator().manual_seed(5)
    sd = {}
    for m in ("down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k", "mid_block.attentions.0.transformer_blocks.0.attn2.to_q",
              "up_blocks.1.resnets.0.conv2"):
        w = usd[m + ".weight"]
        rows, cols = w.shape[0], w[0].numel()
        down = torch.randn(4, cols, generator=g) / cols ** 0.5
        up = torch.randn(rows, 4, generator=g) * (0.3 * float(w.float().std()) / 2)
        if w.dim() == 4:
            down, up = down.reshape(4, *w.shape[1:]), up.reshape(rows, 4, 1, 1)
        sd[f"unet.{m}.lora_A.weight"], sd[f"unet.{m}.lora_B.weight"] = down.half(), up.half()
    path = str(tmp_path / f"style{int(turbo)}.safetensors")
    save_file(sd, path)
    return {path: 1.0}


@pytest.fixture
def env(monkeypatch):
    monkeypatch.setenv("NVENC", "1")
    monkeypatch.setenv("B200SD_SYNTHETIC_WEIGHTS", "1")
    for v in ("B200SD_LANES", "B200SD_MAX_STYLES", "B200SD_POLICY_FRAMES", "B200SD_IP_ADAPTER"):
        monkeypatch.delenv(v, raising=False)
    return monkeypatch


@pytest.mark.parametrize("model_id,tl,lanes", [("tiny-turbo", [32], 8), ("tiny-sd15", T4, 2)], ids=["T1-8lanes", "T4-2lanes"])
def test_viewers_equal_single_viewer_pipelines(cuda, tmp_path, env, model_id, tl, lanes):
    """Four interleaved viewers -- no image prompt, image A, image B, image A with a style LoRA -- each
    bit for bit a pipeline alone whose global image prompt (and style) is the viewer's"""
    from oracle import weights as ow
    style = _lora(tmp_path, "turbo" in model_id)
    img = {"A": _image(11), "B": _image(12)}
    setups = [(None, None), ("A", None), ("B", None), ("A", style)]
    n = 5
    p = _pipe(model_id, tl, lanes, env)
    launches = p.model.stream.launches_per_step
    views = [p.open_stream() for _ in setups]
    for v, (im, lo) in zip(views, setups):
        if lo is not None:
            v.update_lora(lo)
        if im is not None:
            v.update_image_prompt(img[im], 0.8)
    frame = lambda k, i: ow.make_frame(128, 128, seed=500 + 10 * k + i).cuda()  # noqa: E731
    tickets = {k: [] for k in range(len(views))}
    for i in range(n):
        for k, v in enumerate(views):
            tickets[k].append(v.enqueue(frame(k, i)))
    got = {k: [t.result().cpu() for t in ts] for k, ts in tickets.items()}
    assert p.model.stream.launches_per_step == launches and all(e.launches_per_step == launches for e in p._engines)
    for k, (im, lo) in enumerate(setups):
        q = _pipe(model_id, tl, lanes, env)
        if lo is not None:
            q.update_lora(lo)
        if im is not None:
            q.update_image_prompt(img[im], 0.8)
        with q.open_stream() as v:
            want = [t.result().cpu() for t in [v.enqueue(frame(k, i)) for i in range(n)]]
        for i in range(n):
            assert torch.equal(got[k][i], want[i]), f"viewer {k} ({im}, style {lo is not None}): frame {i}"
        del q


def test_global_lora_recomputes_a_viewers_image_prompt(cuda, tmp_path, env):
    """A global LoRA switch after viewers set image prompts: a viewer with only an image prompt and one with its own prompt
    too must each see, bit for bit, a pipeline alone with that LoRA and that global image prompt (the text K / V^T of the
    first come from the new global block, not from the block in force when its image prompt was set)."""
    from oracle import weights as ow
    style = _lora(tmp_path, True)
    img = _image(21)
    frame = lambda k, i: ow.make_frame(128, 128, seed=700 + 10 * k + i).cuda()  # noqa: E731
    p = _pipe("tiny-turbo", [32], 2, env)
    a, b = p.open_stream(), p.open_stream()
    a.update_image_prompt(img, 0.8)
    b.update_prompt("b's own prompt")
    b.update_image_prompt(img, 0.8)
    for k, v in enumerate((a, b)):
        v.enqueue(frame(k, 9)).result()
    p.update_lora(style)
    got = [[t.result().cpu() for t in [v.enqueue(frame(k, i)) for i in range(3)]] for k, v in enumerate((a, b))]
    for k, own in enumerate((None, "b's own prompt")):
        q = _pipe("tiny-turbo", [32], 2, env)
        q.update_lora(style)
        q.update_image_prompt(img, 0.8)
        with q.open_stream() as v:
            if own is not None:
                v.update_prompt(own)
            want = [t.result().cpu() for t in [v.enqueue(frame(k, i)) for i in range(3)]]
        for i in range(3):
            assert torch.equal(got[k][i], want[i]), f"viewer {k}: frame {i} after the LoRA switch"
        del q


# ---- launch audit of a full-size adapter engine ------------------------------------------------------------------------------------
def _image_term(a, q, kip, vtip, n, qchunk=4096):
    """float64 softmax(Q Kip^T / sqrt(d_real)) Vip over image keys [0, n), shared by every image: [nb*sq, heads*d_real]"""
    heads, dr, dp = a["heads"], a["d_real"], a["dp"]
    rows = a["nb"] * a["sq"]
    out = torch.empty(rows, heads * dr, dtype=torch.float64, device=q.device)
    for h in range(heads):
        K = kip[:n, h * dp:(h + 1) * dp].double()
        V = vtip[h * dp:h * dp + dr, :n].double().T
        for r0 in range(0, rows, qchunk):
            Q = q[r0:r0 + qchunk, h * dp:(h + 1) * dp].double()
            out[r0:r0 + qchunk, h * dr:(h + 1) * dr] = torch.softmax((Q @ K.T) * dr ** -0.5, dim=-1) @ V
    return out


def _ip_auditor():
    """The launch auditor, with a float64 reference for the attention launches that carry an image segment"""
    from tests import launch_ref as R
    from tests import test_launch_audit_gpu as LA

    class IpAuditor(LA.Auditor):
        ip_launches = 0

        def _before_attn(self, rec):
            s = super()._before_attn(rec)
            if rec.attn_n_ip:
                a = R.as_dict(rec.attn)
                w = a["heads"] * a["dp"]
                s["ip"] = (LA._snap(rec.attn_k_ip, 64, w, a["ldk"]), LA._snap(rec.attn_vt_ip, w, 64, 64),
                           int(torch.as_tensor(LA._Dev(int(rec.attn_n_ip), (1,), (4,), "<i4"), device="cuda").item()))
            return s

        def _after_attn(self, rec, kind, label, s):
            if "ip" not in s:
                return super()._after_attn(rec, kind, label, s)
            a = R.as_dict(rec.attn)
            kip, vtip, n = s["ip"]
            assert 1 <= n <= 64, f"{label}: {n} image tokens bound"
            atol, rtol = R.TOL["attention"]
            txt = R.attention_ref(a, s["q"], s["k"], s["vt"])
            img = _image_term(a, s["q"], kip, vtip, n)
            ref = txt + img
            got = LA._dev(a["out"], a["nb"] * a["sq"], a["heads"] * a["d_real"], a["ldo"])
            units = R.tol_units(got, ref, atol, rtol)
            skv = a["skv"]
            one = dict(a, skv=skv + n, k_rows=skv + n, vt_cols=skv + n)
            wrongs = {"image segment dropped": R.tol_units(txt, ref, atol, rtol),
                      "one softmax over text and image keys": R.tol_units(
                          R.attention_ref(one, s["q"], torch.cat([s["k"][:skv], kip[:n]]),
                                          torch.cat([s["vt"][:, :skv], vtip[:, :n]], dim=1)), ref, atol, rtol)}
            if n < 64:
                wrongs["padding keys not masked"] = R.tol_units(txt + _image_term(a, s["q"], kip, vtip, 64), ref, atol, rtol)
            if s["spare"] is not None:
                now = LA._dev(a["out"], a["nb"] * a["sq"] - 1, a["ldo"], a["ldo"])[:, a["heads"] * a["d_real"]:].view(torch.int16)
                assert torch.equal(now, s["spare"]), f"{label}: stray write into the spare output columns"
            self.ip_launches += 1
            self._record("attention", label, units, wrongs)

    return IpAuditor()


def test_full_size_sd15_launch_audit_with_an_image_prompt(cuda):
    """Full-size SD-1.5 at 512x512, T = 4, with an image prompt bound: every launch of a frame checked by the launch auditor
    against float64 (the 16 UNet cross-attentions with their image segment), and the audited frame equal to a graph step of
    an identical lane"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import unet as ounet
    from oracle import weights as ow
    from tests import test_launch_audit_gpu as LA
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    LA._release_device_memory()
    sd = lane = None
    try:
        emb = ow.make_prompt_embeds(ounet.SD15.cross_attention_dim)
        sd = StreamDiffusion(A.SD15, ow.make_unet_weights(ounet.SD15), ow.make_taesd_weights(), T4, lambda p: emb, width=512,
                             height=512, ip_adapter=_adapter(A.SD15))
        sd.prepare("p", guidance_scale=0.0)
        sd.set_image_tokens(sd.image_tokens(_image(31, 224)), 0.8)
        lane = sd.add_lane()
        lane.set_concurrency(1)
        lane._prepare_like(sd)
        frames = [ow.make_frame(512, 512, seed=300 + i).cuda() for i in range(2)]
        sd.step_u8(frames[0])
        lane.step_u8(frames[0])
        aud = _ip_auditor()
        got = sd.audit_step(frames[1], aud).clone()
        want = lane.step_u8(frames[1])
        torch.cuda.synchronize()
        print("\n" + aud.table("sd15-T4-512 with an image prompt") + f"\n  image-segment launches: {aud.ip_launches}")
        assert not aud.other, f"launches without a record: {dict(aud.other)}"
        for cls in aud.launches:
            assert aud.checked[cls] == aud.launches[cls], cls
        assert aud.calls == sum(aud.checked.values()) == sd.launches_per_step
        assert aud.ip_launches == 16, aud.ip_launches
        assert torch.equal(got, want), "the audited frame differs from a graph step of an identical lane"
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        if sd is not None:
            sd.lanes.clear()
        sd = lane = None
        LA._release_device_memory()


def test_refuses_a_non_finite_scale_and_too_many_tokens(cuda):
    from ai_rtc_agent_b200.host import capi
    sd, _ = _tiny(True, [32])
    st = sd.new_state()
    tok = sd.image_tokens(_image(41))
    for bad in (float("inf"), float("-inf"), float("nan")):
        with pytest.raises(capi.B2Error, match="scale finite"):
            sd.set_image_tokens(tok, bad)
        with pytest.raises(capi.B2Error, match="scale finite"):
            st.set_image_tokens(tok, bad)
    with pytest.raises(capi.B2Error, match="n_tok must be 1..4"):
        sd.set_image_tokens(torch.cat([tok, tok], 1), 1.0)
