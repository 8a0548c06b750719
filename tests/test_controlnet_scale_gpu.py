"""ControlNet conditioning scale on the H100: the per-item accumulator scale of the zero-conv contractions against float64 under
every plan the engine's policies pick, and the engine against the scaled fp32 restatement (tests/controlnet_scale_ref.py),
with its bit-exactness properties (scale 1 = no scale, scale 0 = no ControlNet) and live updates on lanes and states."""
import math

import pytest
import torch

from tests.controlnet_scale_ref import ScaledControlNetOracle
from tests.util import assert_discriminates, guarded, hetero

pytestmark = pytest.mark.gpu

SCALES = [0.0, 1.0, -0.5, 0.37]


def _ops():
    from ai_rtc_agent_b200.host import ops
    return ops


def _plans(ops, x, wp, out, nb, **kw):
    """(name, igemm kwargs) of every plan to run: the latency and throughput policies' choices for this contraction, and
    single CTAs at each N tile dividing it, split-K 2 / 4 and CTA pairs"""
    c = out.shape[3]
    plans = []
    for pol in (1, 2):
        p = ops.igemm_engine_plan([(x, 1)], wp, out, autotile=pol, allow_swap=False, **kw)
        assert p.swap == 0
        plans.append((f"policy{pol}", dict(bn=p.bn, splits=p.splits, pair=p.mode == 1)))
    for bn in (64, 128, 160, 256):
        if c % bn == 0:
            plans.append((f"bn{bn}", dict(bn=bn, splits=1)))
    plans += [("splitk2", dict(bn=64 if c % 128 else 128, splits=2)), ("splitk4", dict(bn=64 if c % 128 else 128, splits=4)),
              ("pair", dict(bn=64 if c % 128 else 128, splits=1, pair=True)),
              ("pair-splitk2", dict(bn=64 if c % 128 else 128, splits=2, pair=True))]
    return plans


@pytest.mark.parametrize("size", [128, 512, 1024])
@pytest.mark.parametrize("level", [0, 1, 2, 3])
def test_igemm_per_item_scale_on_the_zero_conv_shapes(cuda, size, level):
    """out = s[b] * (acc + bias) + res on the zero convs' 1x1 shapes (C = 320 / 640 / 1280 / 1280 at latent / 2^level), batch
    1..4 with per-item scales 0, 1, -0.5, 0.37, under every plan.  Rejected answers: the scale also on the residual, item 0's
    scale for every item, the scale before the bias, the scale applied twice (per split-K slice and after the reduction).  An
    all-ones vector gives the NULL pointer's result bit for bit."""
    ops = _ops()
    c = [320, 640, 1280, 1280][level]
    hw = size // 8 >> level
    w = (torch.randn((c, c, 1, 1), generator=torch.Generator().manual_seed(level), dtype=torch.float64) / math.sqrt(c))
    wh = w.half().to(cuda)
    wp = ops.pack_conv_weight(wh)
    bias = (torch.randn((1, c), generator=torch.Generator().manual_seed(9), dtype=torch.float64) * 2).float().to(cuda)
    split = {}
    caught = {}   # plan -> the wrong answers it was told apart from (a bug is harmless under some scales, e.g. 0 and 1)
    for nb in (1, 2, 3, 4):
        x = hetero((nb, hw, hw, c), (0, 3), 10 + nb, cuda, offset=1.0)
        res = hetero((nb, hw, hw, c), (0, 3), 20 + nb, cuda)
        s = torch.tensor([SCALES[(b + level) % 4] for b in range(nb)], dtype=torch.float32, device=cuda)
        sd = s.double().view(-1, 1, 1, 1)
        acc = torch.einsum("nhwc,oc->nhwo", x.double(), wh.double()[:, :, 0, 0])
        pre = acc + bias.double()[0]
        ref = sd * pre + res.double()
        wrong = {"scale on the residual too": sd * (pre + res.double()),
                 "item 0's scale for every item": sd[:1] * pre + res.double(),
                 "scale before the bias": sd * acc + bias.double()[0] + res.double(),
                 "scale applied per K slice and again": sd * sd * acc + sd * bias.double()[0] + res.double()}
        ones = torch.ones(nb, dtype=torch.float32, device=cuda)
        for name, kw in _plans(ops, x, wp, torch.empty((nb, hw, hw, c), dtype=torch.float16, device=cuda), nb,
                               colbias=bias, res=res, acc_scale_b=s):
            if kw.get("pair") and (nb * hw * hw) // 128 < 2:
                continue   # a CTA pair needs two M tiles
            g = guarded((nb * hw * hw, c), pitch=c + 8, device=cuda)
            out = g.view.view(nb, hw, hw, c)
            ops.igemm([(x, 1)], wp, out, colbias=bias, res=res, acc_scale_b=s, **kw)
            what = f"{size}px level {level} nb {nb} {name} {kw}"
            for bug, wr in wrong.items():
                if torch.equal(wr, ref) or (bug.startswith("scale applied per K") and kw.get("splits", 1) == 1):
                    continue
                assert_discriminates(out, ref, wr, 2e-3, 4e-3, what, bug=bug)
                caught.setdefault(name, set()).add(bug)
            split[name] = split.get(name, False) or kw.get("splits", 1) > 1
            g.assert_untouched(what)
            a = torch.empty_like(out)
            b = torch.empty_like(out)
            ops.igemm([(x, 1)], wp, a, colbias=bias, res=res, acc_scale_b=ones, **kw)
            ops.igemm([(x, 1)], wp, b, colbias=bias, res=res, **kw)
            assert torch.equal(a, b), f"{what}: all-ones scale differs from none"
    for name, bugs in caught.items():
        want = set(wrong) if split[name] else set(wrong) - {"scale applied per K slice and again"}
        assert bugs == want, f"{name}: only {sorted(bugs)} were told apart"


def test_igemm_per_item_scale_refuses_what_it_does_not_cover(cuda):
    from ai_rtc_agent_b200.host import capi
    ops = _ops()
    x = hetero((1, 16, 16, 64), (3,), 1, cuda)
    wp = ops.pack_conv_weight(torch.randn((64, 64, 1, 1), device=cuda).half())
    out = torch.empty((1, 16, 16, 64), dtype=torch.float16, device=cuda)
    s = torch.ones(1, dtype=torch.float32, device=cuda)
    for kw in (dict(swap=True, bn=64), dict(bn=48), dict(silu=True, bn=64)):
        with pytest.raises(capi.B2Error):
            ops.igemm([(x, 1)], wp, out, acc_scale_b=s, **kw)
    # the halo-tile kernel has no per-item scale: a 64 -> 64 3x3 convolution it runs refuses one instead of ignoring it
    w3 = ops.pack_conv_weight(torch.randn((64, 64, 3, 3), device=cuda).half() * 0.05)
    ops.igemm([(x, 9)], w3, out, tconv=True)
    with pytest.raises(capi.B2Error):
        ops.igemm([(x, 9)], w3, out, tconv=True, acc_scale_b=s)


# ---- the engine ---------------------------------------------------------------------------------------------------------------
def _engine(turbo, t_index_list, cn16, hed=None, hw=128):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    usd, vsd = ow.make_unet_weights(cfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    sd = StreamDiffusion(arch, usd, vsd, t_index_list, lambda p: emb, width=hw, height=hw, controlnet_sd=cn16, hed_sd=hed)
    sd.prepare("p", guidance_scale=0.0)
    return sd, cfg, usd, vsd, emb


def _u8_check(got, ref, what):
    d = (got.cpu().int() - ref.cpu().int()).abs()
    frac = (d <= 2).float().mean().item()
    assert frac >= 0.999 and d.max().item() <= 8, f"{what}: frac(|d|<=2)={frac:.5f} max={d.max().item()}"


def _hed16():
    from ai_rtc_agent_b200.host import arch as A
    return {k: v.half().float() for k, v in A.synthetic_hed().items()}


@pytest.mark.parametrize("processor", [None, "hed"])
@pytest.mark.parametrize("turbo,t_index_list", [(False, [18, 26, 35, 45]), (True, [32])])
def test_engine_matches_the_scaled_oracle(cuda, turbo, t_index_list, processor):
    """Several settings, switched between frames, against the fp32 restatement; each update is enqueued between frames and
    splits them exactly there, with launches_per_step unchanged"""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import weights as ow
    from ai_rtc_agent_b200.host.stream import control_scales
    from oracle import unet as ounet
    cn16 = ocn.make_weights(ounet.tiny_config(turbo))
    hed = _hed16() if processor == "hed" else None
    sd, cfg, usd, vsd, emb = _engine(turbo, t_index_list, cn16, hed)
    orc = ScaledControlNetOracle(ow.to_float(usd), cfg, ow.to_float(vsd), ow.to_float(cn16), t_index_list, 128, 128, hed_sd=hed)
    orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    launches = sd.launches_per_step
    i = 0
    for control in [(1.0, 0.0, 1.0), (0.6, 0.0, 1.0), (1.0, 0.5, 1.0), (-0.5, 0.0, 0.6), (1.3, 0.3, 0.8)]:
        sd.set_control_scale(*control)
        orc.scales = control_scales(control, t_index_list, 50)
        for _ in range(2):
            frame = ow.make_frame(128, 128, seed=60 + i)
            _u8_check(sd.step_u8(frame.to(cuda)), opipe.frame_to_u8(orc, frame), f"{control} frame {i}")
            i += 1
    assert sd.launches_per_step == launches


def test_defaults_and_zero_scale_are_bit_identical(cuda):
    """Default settings set explicitly equal never set; scale 0, or a window that masks every slot, equals the same UNet
    without a ControlNet, bit for bit.  Twenty updates leave the device memory as it was."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    tl = [18, 26, 35, 45]
    cn16 = ocn.make_weights(ounet.tiny_config(False))
    plain, *_ = _engine(False, tl, None)
    never, *_ = _engine(False, tl, cn16)
    explicit, *_ = _engine(False, tl, cn16)
    zero, *_ = _engine(False, tl, cn16)
    masked, *_ = _engine(False, tl, cn16)
    explicit.set_control_scale(1.0, 0.0, 1.0)
    zero.set_control_scale(0.0)
    masked.set_control_scale(0.8, 0.95, 1.0)   # 45 / 50 < 0.95: every slot is outside the window
    for i in range(4):
        f = ow.make_frame(128, 128, seed=40 + i).to(cuda)
        p, n, e, z, m = (x.step_u8(f).cpu() for x in (plain, never, explicit, zero, masked))
        assert torch.equal(n, e), f"frame {i}: explicit defaults"
        assert torch.equal(z, p) and torch.equal(m, p), f"frame {i}: scale 0 / masked window"
        assert not torch.equal(n, p)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(20):
        explicit.set_control_scale(0.05 * k, 0.0, 1.0)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


@pytest.mark.parametrize("turbo,lanes", [(False, 2), (True, 8)])
def test_viewers_with_their_own_settings(cuda, turbo, lanes):
    """Four interleaved states on the lanes: global settings, own scale, own window with own t_index_list, own scale on a
    style.  Each one's frames equal a single engine whose global settings are that viewer's, bit for bit.  A global
    t_index_list update re-masks the own settings; a global ControlNet update replaces them."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    tl = [32] if turbo else [18, 26, 35, 45]
    own_t = [20] if turbo else [10, 20, 30, 40]
    new_t = [40] if turbo else [5, 25, 30, 49]
    cfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    cn16 = ocn.make_weights(cfg)
    usd, vsd = ow.make_unet_weights(cfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)

    def engine():
        sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, width=128, height=128, controlnet_sd=cn16, live_lora=True)
        sd.set_concurrency(lanes)
        sd.prepare("p", guidance_scale=0.0)
        return sd

    def single(control, t):
        e = engine()
        if t != tl:
            e.t_list, e.sub_timesteps = list(t), [e.timesteps[i] for i in t]
            e.sync_timesteps()
        e.set_control_scale(*control)
        return e
    # the references of the three phases below: a dedicated engine per viewer and phase
    phases = [[((1.0, 0.0, 1.0), tl), ((0.6, 0.0, 1.0), tl), ((1.0, 0.5, 1.0), own_t), ((-0.5, 0.0, 1.0), tl)],
              [((1.0, 0.0, 1.0), new_t), ((0.6, 0.0, 1.0), new_t), ((1.0, 0.5, 1.0), new_t), ((-0.5, 0.0, 1.0), new_t)],
              [((0.8, 0.0, 0.9), new_t)] * 4]
    refs = [[single(c, t) for c, t in wants] for wants in phases]
    root = engine()
    pool = [root] + [root.add_lane() for _ in range(lanes - 1)]
    style = root.add_style()   # the base weights, on a store of its own
    states = [root.new_state() for _ in range(4)]
    states[1].set_control_scale(0.6)
    states[2].set_t_index_list(own_t)
    states[2].set_control_scale(1.0, 0.5, 1.0)
    states[3].set_control_scale(-0.5, engine=style)

    def run(phase, n=3):
        for i in range(n):
            for k, st in enumerate(states):
                f = ow.make_frame(128, 128, seed=100 * phase + 10 * i + k).to(cuda)
                eng = style if k == 3 else pool[(i * 4 + k) % lanes]
                got = eng.step_u8(f, state=st).cpu()
                assert torch.equal(got, refs[phase][k].step_u8(f).cpu()), f"phase {phase} viewer {k} frame {i}"
    run(0)
    # a global t_index_list update re-masks the own settings (and drops viewer 2's own list)
    root.t_list, root.sub_timesteps = list(new_t), [root.timesteps[i] for i in new_t]
    root.sync_timesteps()
    assert [st.own_control for st in states] == [None, (0.6, 0.0, 1.0), (1.0, 0.5, 1.0), (-0.5, 0.0, 1.0)]
    states[3].set_control_scale(*states[3].own_control, engine=style)   # a style's states are refreshed on a style engine
    for st in states:
        st.reset()
    run(1)
    # a global ControlNet update replaces them
    root.set_control_scale(0.8, 0.0, 0.9)
    for st in states:
        st.reset()
        assert st.own_control is None
    run(2)
