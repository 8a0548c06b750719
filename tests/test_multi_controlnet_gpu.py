"""Several ControlNets on the H100 (diffusers' MultiControlNetModel): each net on its own control image, with its own per-slot
scales, the nets' residuals summed into the UNet's skips.  The engine against the fp32 multi-net restatement
(tests/multi_controlnet_ref.py) on identical seeded weights, and the bit-exact properties: a net at scale 0 or masked on every
slot adds exactly nothing, a list of one net is the single net, lanes, CUDA graphs, per-viewer settings and packed blobs.

Tolerances as in tests/test_controlnet_gpu.py: activations max|d| <= 2e-2 * max|ref| and cosine >= 0.999; u8 frames |d| <= 2
LSB on >= 99.9 % of the pixels, max |d| <= 8."""
import pytest
import torch
import torch.nn.functional as F

from tests.multi_controlnet_ref import MultiControlNetStreamOracle

pytestmark = pytest.mark.gpu

T4 = [18, 26, 35, 45]


def _hed16():
    from ai_rtc_agent_b200.host import arch as A
    return {k: v.half().float() for k, v in A.synthetic_hed().items()}


def _models(turbo, full=False):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    if full:
        cfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
    else:
        cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    return cfg, arch, ow.make_unet_weights(cfg), ow.make_taesd_weights(), ow.make_prompt_embeds(cfg.cross_attention_dim)


def _nets(cfg, n):
    """n seeded ControlNets that differ from each other"""
    from oracle import controlnet as ocn
    return [ocn.make_weights(cfg, seed=5678 + 31 * i) for i in range(n)]


def _engine(models, tl, hw, cns, procs, hed=None, graph=True, concurrency=1, blob=None, live_lora=False):
    """cns: None (no ControlNet), one state dict (procs: its processor) or a list of them (procs: one per net)"""
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    cfg, arch, usd, vsd, emb = models
    height, width = (hw, hw) if isinstance(hw, int) else hw
    multi = isinstance(cns, list)
    kw = dict(width=width, height=height, use_cuda_graph=graph, live_lora=live_lora)
    if multi:
        kw["control_processors"] = procs
    if blob is not None:
        sd = StreamDiffusion(arch, {}, {}, tl, lambda p: emb, packed_blob=blob, hed_sd={} if hed is not None else None,
                             controlnet_sd=[{}] * len(cns) if multi else ({} if cns is not None else None), **kw)
    else:
        sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, controlnet_sd=cns, hed_sd=hed, **kw)
    if concurrency > 1:
        sd.set_concurrency(concurrency)
    sd.prepare("p", guidance_scale=0.0)
    return sd


def _cmp(got_nhwc, ref_nchw):
    got = got_nhwc.float().permute(0, 3, 1, 2)
    ref = ref_nchw.float().cpu()
    err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
    cos = F.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
    return err, cos


def _u8_check(got, ref, what):
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"


def _frames(h, w, seed, n):
    from oracle import weights as ow
    return [ow.make_frame(h, w, seed=seed + i).cuda() for i in range(n)]


# ---- bit-exact reductions -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("turbo,tl,hw", [(False, T4, 128), (True, [32], (64, 192)), (False, [18, 35], (192, 128))])
def test_a_silent_net_adds_exactly_nothing(cuda, turbo, tl, hw):
    """[A, B] with B at scale 0, or with B's window masking every slot, equals A alone; [A, B] with A at 0 equals B alone; [A]
    equals A.  A reads the frame, B the HED edge map."""
    models = _models(turbo)
    a, b = _nets(models[0], 2)
    hed = _hed16()
    h, w = (hw, hw) if isinstance(hw, int) else hw
    a_alone = _engine(models, tl, hw, a, None)
    b_alone = _engine(models, tl, hw, b, "hed", hed=hed)
    one = _engine(models, tl, hw, [a], [None])
    b_zero = _engine(models, tl, hw, [a, b], [None, "hed"], hed=hed)
    b_masked = _engine(models, tl, hw, [a, b], [None, "hed"], hed=hed)
    a_zero = _engine(models, tl, hw, [a, b], [None, "hed"], hed=hed)
    both = _engine(models, tl, hw, [a, b], [None, "hed"], hed=hed)
    b_zero.set_control_scale([1.0, 0.0])
    b_masked.set_control_scale(1.0, [0.0, 0.98], [1.0, 1.0])   # (t + 1) / 50 <= 0.98 for every slot: none kept
    a_zero.set_control_scale([0.0, 1.0])
    assert one.launches_per_step == a_alone.launches_per_step
    for i, f in enumerate(_frames(h, w, 10, 3)):
        ra, rb = a_alone.step_u8(f).cpu(), b_alone.step_u8(f).cpu()
        assert torch.equal(one.step_u8(f).cpu(), ra), f"[A] vs A, frame {i}"
        assert torch.equal(b_zero.step_u8(f).cpu(), ra), f"[A, B] with B at 0 vs A, frame {i}"
        assert torch.equal(b_masked.step_u8(f).cpu(), ra), f"[A, B] with B masked vs A, frame {i}"
        assert torch.equal(a_zero.step_u8(f).cpu(), rb), f"[A, B] with A at 0 vs B, frame {i}"
        assert not torch.equal(both.step_u8(f).cpu(), ra)


@pytest.mark.parametrize("turbo,tl", [(False, T4), (True, [32])])
def test_fullsize_silent_net_adds_exactly_nothing_512(cuda, turbo, tl):
    """Full-size synthetic SD-1.5 T=4 and SD-Turbo T=1 at 512x512: frame + HED nets with the HED net at scale 0 equal the frame
    net alone, and with the frame net at 0 the HED net alone, bit for bit."""
    models = _models(turbo, full=True)
    a, b = _nets(models[0], 2)
    hed = _hed16()
    pair = _engine(models, tl, 512, [a, b], [None, "hed"], hed=hed)
    a_alone = _engine(models, tl, 512, a, None)
    b_alone = _engine(models, tl, 512, b, "hed", hed=hed)
    frames = _frames(512, 512, 20, 2)
    pair.set_control_scale([1.0, 0.0])
    for i, f in enumerate(frames):
        assert torch.equal(pair.step_u8(f).cpu(), a_alone.step_u8(f).cpu()), f"B at 0, frame {i}"
    pair2 = _engine(models, tl, 512, [a, b], [None, "hed"], hed=hed)
    pair2.set_control_scale([0.0, 1.0])
    for i, f in enumerate(frames):
        assert torch.equal(pair2.step_u8(f).cpu(), b_alone.step_u8(f).cpu()), f"A at 0, frame {i}"


# ---- against the multi-net restatement ----------------------------------------------------------------------------------------
def _check_against_oracle(sd, orc, frames, settings, n_nets, taps_on=(0,)):
    """Step sd and the oracle on frames, applying settings[i] before frame i; the u8 frames on every frame, every net's taps on
    the frames in taps_on"""
    from ai_rtc_agent_b200.host.stream import control_vector
    from oracle import pipeline as opipe
    tl = sd.t_list
    T = len(tl)
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    orc.to("cuda")
    try:
        _steps(sd, orc, frames, settings, n_nets, taps_on, tl, T)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def _steps(sd, orc, frames, settings, n_nets, taps_on, tl, T):
    from ai_rtc_agent_b200.host.stream import control_vector
    from oracle import pipeline as opipe
    for i, f in enumerate(frames):
        if i in settings:
            sd.set_control_scale(*settings[i])
            v = control_vector(sd.control, tl, 50)
            orc.scales = [v[k * T:(k + 1) * T] for k in range(n_nets)]
        out = sd.step_u8(f)
        with torch.no_grad():
            ref = opipe.frame_to_u8(orc, f)
        _u8_check(out, ref, f"frame {i}")
        if i not in taps_on:
            continue
        un, nets = orc.last["unet_taps"], orc.last["nets"]
        rows = []
        for n in range(n_nets):   # net n's chain: skip + r_0 + ... + r_n
            later = nets[n + 1:]
            for k in range(12):
                rows.append((f"cn{n}.res.{k}", un[f"res.{k}"] - sum((x["res"][k] for x in later), torch.zeros(()))))
            rows.append((f"cn{n}.mid", un["cn_mid"] - sum((x["mid"] for x in later), torch.zeros(()))))
            rows.append((f"cn{n}_cond", nets[n]["cn_taps"]["cond"]))
        rows.append(("eps", orc.last["eps"]))
        res = [(name, *_cmp(sd.get_tensor(name), r)) for name, r in rows]
        table = "\n".join(f"{n:12s} relerr={e:.2e} cos={c:.6f}" for n, e, c in res)
        for n, e, c in res:
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: tap {n} out of tolerance\n{table}"


@pytest.mark.parametrize("turbo,tl,hw", [(False, T4, 128), (True, [32], 64), (False, T4, (192, 128)), (True, [32], (128, 320)),
                                         (True, [32], 1024)])
def test_frame_and_hed_nets_match_the_oracle(cuda, turbo, tl, hw):
    """A frame net and a HED net at different scales and windows, changed between frames: the per-net residual chains, each
    net's conditioning embedding and the frames against the fp32 restatement (diffusers' summation order)."""
    from oracle import weights as ow
    models = _models(turbo)
    cfg, arch, usd, vsd, emb = models
    nets = _nets(cfg, 2)
    hed = _hed16()
    h, w = (hw, hw) if isinstance(hw, int) else hw
    sd = _engine(models, tl, hw, nets, [None, "hed"], hed=hed)
    orc = MultiControlNetStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), [ow.to_float(n) for n in nets], [None, "hed"],
                                      tl, w, h, hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    n = 3 if h * w >= 1024 * 1024 else 5
    settings = {0: (1.0, 0.0, 1.0), 1: ([0.6, 1.3], 0.0, 1.0), 2: ([1.0, -0.5], [0.0, 0.5], [0.6, 1.0]),
                3: (0.8, [0.3, 0.0], 0.9), 4: ([0.0, 1.1], 0.0, 1.0)}
    _check_against_oracle(sd, orc, _frames(h, w, 30, n), settings, 2, taps_on=(0, 2))


def test_fullsize_frame_and_hed_nets_match_the_oracle_512(cuda):
    """Full-size synthetic SD-1.5 T=4 at 512x512, a frame net and a HED net both contributing, at different scales and windows
    changed between frames: the u8 frames, each net's residual chain (cn<i>.res.K, cn<i>.mid) and conditioning embedding
    against the fp32 restatement run by torch on the GPU, at the shapes whose tile and split policies the tiny models do not
    reach"""
    from oracle import weights as ow
    models = _models(False, full=True)
    cfg, arch, usd, vsd, emb = models
    nets = _nets(cfg, 2)
    hed = _hed16()
    sd = _engine(models, T4, 512, nets, [None, "hed"], hed=hed)
    orc = MultiControlNetStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), [ow.to_float(n) for n in nets], [None, "hed"],
                                      T4, 512, 512, hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    settings = {0: ([0.8, 1.1], [0.0, 0.2], 1.0), 2: ([1.2, 0.6], 0.0, [0.7, 1.0])}
    _check_against_oracle(sd, orc, _frames(512, 512, 40, 3), settings, 2, taps_on=(0, 2))


@pytest.mark.parametrize("procs", [["hed", None, "hed"], [None, "hed", None, "hed"]])
def test_three_and_four_nets_share_one_hed(cuda, procs):
    """Three and four nets at tiny size against the restatement; the frame program runs HED exactly once (one fuse launch and
    one HED input head), however many nets read the edge map."""
    from ai_rtc_agent_b200.host import capi
    from oracle import weights as ow
    models = _models(False)
    cfg, arch, usd, vsd, emb = models
    nets = _nets(cfg, len(procs))
    hed = _hed16()
    sd = _engine(models, T4, 128, nets, procs, hed=hed)
    orc = MultiControlNetStreamOracle(ow.to_float(usd), cfg, ow.to_float(vsd), [ow.to_float(n) for n in nets], procs, T4, 128,
                                      128, hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    scales = [0.5 + 0.25 * k for k in range(len(procs))]
    _check_against_oracle(sd, orc, _frames(128, 128, 50, 3), {0: (scales, 0.0, 1.0), 1: (scales, [0.0] * len(procs),
                                                                                                    [0.7] * len(procs))},
                          len(procs), taps_on=(0,))
    seen = []
    sd.audit_step(_frames(128, 128, 60, 1)[0], lambda i, after, rec: seen.append((rec.kind, rec.label)) if not after else None)
    assert sum(k == capi.LAUNCH_HED_FUSE for k, _ in seen) == 1, "HED's fuse launch"
    assert [lbl for _, lbl in seen].count(b"smallconv hed head") == 1, "HED's input head"
    assert sum(1 for _, lbl in seen if lbl.startswith(b"smallconv controlnet") and lbl.endswith(b" head")) == procs.count(None)
    assert len(seen) == sd.launches_per_step


# ---- lanes, graphs, updates between queued frames ------------------------------------------------------------------------------
def test_lanes_and_graphs_are_bit_identical(cuda):
    """Throughput lanes (T=1), a T=4 state stepped alternately on two lanes (stage-pipelined) and a CUDA-graph engine against
    an eager one, each equal to frames submitted one at a time, with two nets at their own scales."""
    hed = _hed16()
    m1 = _models(True)
    nets = _nets(m1[0], 2)
    par = _engine(m1, [32], 128, nets, [None, "hed"], hed=hed, concurrency=4)
    lanes = [par.add_lane() for _ in range(3)]
    par.set_control_scale([0.7, 1.2])
    frames = _frames(128, 128, 70, 4)
    outs = [eng.step_u8(f) for eng, f in zip([par] + lanes, frames)]
    torch.cuda.synchronize()
    for i, f in enumerate(frames):
        assert torch.equal(outs[i].cpu(), par.step_u8(f).cpu()), f"throughput lane {i}"
    m4 = _models(False)
    nets4 = _nets(m4[0], 2)
    single = _engine(m4, T4, 128, nets4, ["hed", None], hed=hed, concurrency=2)
    owner = _engine(m4, T4, 128, nets4, ["hed", None], hed=hed, concurrency=2)
    eager = _engine(m4, T4, 128, nets4, ["hed", None], hed=hed, concurrency=2, graph=False)
    for e in (single, owner, eager):
        e.set_control_scale([0.9, 0.4], [0.0, 0.3], 1.0)
    lane = owner.add_lane()
    state = owner.new_state()
    for i, f in enumerate(_frames(128, 128, 80, 6)):
        a = single.step_u8(f).cpu()
        b = (owner if i % 2 == 0 else lane).step_u8(f, state=state).cpu()
        assert torch.equal(a, b), f"stage-pipelined frame {i}"
        assert torch.equal(a, eager.step_u8(f).cpu()), f"graph vs eager frame {i}"


def test_updates_between_queued_frames(cuda):
    """Updates enqueued between queued frames split them exactly there: frames enqueued before an update use the old settings
    and frames after it the new ones, as on an engine that waits for every frame; no graph is recaptured and
    launches_per_step does not change."""
    m = _models(False)
    nets = _nets(m[0], 2)
    hed = _hed16()
    settings = [([1.0, 1.0], 0.0, 1.0), ([0.3, 1.4], 0.0, 1.0), (1.0, [0.5, 0.0], [1.0, 0.6])]
    frames = _frames(128, 128, 90, 6)
    ref = _engine(m, T4, 128, nets, [None, "hed"], hed=hed)
    sd = _engine(m, T4, 128, nets, [None, "hed"], hed=hed)
    launches = sd.launches_per_step
    want, outs = [], []
    for i, f in enumerate(frames):
        if i % 2 == 0:
            ref.set_control_scale(*settings[i // 2])
            sd.set_control_scale(*settings[i // 2])
        want.append(ref.step_u8(f).cpu())   # waits for the frame
        outs.append(sd.step_u8(f))          # queued without waiting
    torch.cuda.synchronize()
    for i, o in enumerate(outs):
        assert torch.equal(o.cpu(), want[i]), f"frame {i}"
    assert not torch.equal(want[2], _engine(m, T4, 128, nets, [None, "hed"], hed=hed).step_u8(frames[0]).cpu())
    assert sd.launches_per_step == launches


def test_viewers_with_their_own_per_net_settings(cuda):
    """Three viewers round-robin on shared lanes with different per-net settings, one on a LoRA style (the base weights on a
    store of its own): each equals an engine whose global settings are that viewer's, bit for bit.  A global t_index_list
    update re-masks them; a global update replaces them."""
    m = _models(False)
    nets = _nets(m[0], 2)
    hed = _hed16()
    own = [None, ([0.5, 1.5], 0.0, 1.0), (1.0, [0.0, 0.5], [0.7, 1.0])]
    new_t = [5, 25, 30, 49]

    def single(control, t):
        e = _engine(m, T4, 128, nets, [None, "hed"], hed=hed, concurrency=2, live_lora=True)
        if t != T4:
            e.t_list, e.sub_timesteps = list(t), [e.timesteps[i] for i in t]
            e.sync_timesteps()
        if control is not None:
            e.set_control_scale(*control)
        return e
    root = _engine(m, T4, 128, nets, [None, "hed"], hed=hed, concurrency=2, live_lora=True)
    pool = [root, root.add_lane()]
    style = root.add_style()
    states = [root.new_state() for _ in range(3)]
    states[1].set_control_scale(*own[1])
    states[2].set_control_scale(*own[2], engine=style)

    def run(refs, seed):
        for i in range(3):
            for k, st in enumerate(states):
                f = _frames(128, 128, seed + 10 * i + k, 1)[0]
                eng = style if k == 2 else pool[(i * 3 + k) % 2]
                assert torch.equal(eng.step_u8(f, state=st).cpu(), refs[k].step_u8(f).cpu()), f"viewer {k} frame {i}"
    run([single(c, T4) for c in own], 200)
    root.t_list, root.sub_timesteps = list(new_t), [root.timesteps[i] for i in new_t]
    root.sync_timesteps()
    assert [st.own_control for st in states] == [None, ((0.5, 1.5), (0.0, 0.0), (1.0, 1.0)), ((1.0, 1.0), (0.0, 0.5), (0.7, 1.0))]
    states[2].set_control_scale(*states[2].own_control, engine=style)
    for st in states:
        st.reset()
    run([single(c, new_t) for c in own], 300)
    root.set_control_scale([0.2, 0.9])
    for st in states:
        st.reset()
        assert st.own_control is None
    run([single(([0.2, 0.9], 0.0, 1.0), new_t) for _ in own], 400)


# ---- packed blobs -------------------------------------------------------------------------------------------------------------
def test_two_net_packed_blob_round_trip(cuda, tmp_path):
    """A two-net engine's blob loads into a two-net engine with the same processors and gives its frames bit for bit; an engine
    with other processors or another net count refuses it; a single-net engine's blob still loads as before."""
    from ai_rtc_agent_b200.host import capi
    m = _models(False)
    nets = _nets(m[0], 2)
    hed = _hed16()
    a = _engine(m, [18, 35], 128, nets, [None, "hed"], hed=hed)
    a.set_control_scale([0.8, 1.1])
    path = str(tmp_path / "two.b2pack")
    a.export_packed(path)
    b = _engine(m, [18, 35], 128, nets, [None, "hed"], hed=hed, blob=path)
    b.set_control_scale([0.8, 1.1])
    for i, f in enumerate(_frames(128, 128, 110, 3)):
        assert torch.equal(a.step_u8(f).cpu(), b.step_u8(f).cpu()), f"frame {i}"
    with pytest.raises(capi.B2Error):
        _engine(m, [18, 35], 128, nets, ["hed", None], hed=hed, blob=path)
    with pytest.raises(capi.B2Error):
        _engine(m, [18, 35], 128, nets[0], None, blob=path)


def test_version_4_blob_still_loads(cuda, tmp_path):
    """A blob written in format 4 (b2sd_config up to ip_tokens) loads into a single-net engine and gives its frames"""
    import struct
    from ai_rtc_agent_b200.host import capi
    m = _models(False)
    net = _nets(m[0], 1)[0]
    a = _engine(m, [18, 35], 128, net, None)
    path = tmp_path / "v5.b2pack"
    a.export_packed(str(path))
    raw = path.read_bytes()
    assert raw[:8] == b"B2SDPACK" and struct.unpack("<I", raw[8:12])[0] == 5
    cfg_size = __import__("ctypes").sizeof(capi.EngineConfig)
    more = 4 * (capi.MAX_CONTROLNETS - 1)
    v4 = raw[:8] + struct.pack("<I", 4) + raw[12:12 + cfg_size - more] + raw[12 + cfg_size:]
    (tmp_path / "v4.b2pack").write_bytes(v4)
    b = _engine(m, [18, 35], 128, net, None, blob=str(tmp_path / "v4.b2pack"))
    for i, f in enumerate(_frames(128, 128, 120, 2)):
        assert torch.equal(a.step_u8(f).cpu(), b.step_u8(f).cpu()), f"frame {i}"
