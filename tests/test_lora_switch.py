"""Live LoRA switching, host side (no GPU): the shared key resolver, the factors handed to the engine, the errors that must be
raised before the engine is called, and how the live mode is chosen."""
import inspect
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_host import _write_tiny_checkpoint  # noqa: E402

TQ = "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q"


def _fuse_lora_before(unet_sd, lora_sd, scale=1.0, strict=True):
    """fuse_lora as it was before its key resolution was shared with the live path (the yardstick of its results)"""
    pairs = {}
    for k, v in lora_sd.items():
        base = None
        for down_tag, up_tag in ((".lora_A.weight", ".lora_B.weight"), (".lora.down.weight", ".lora.up.weight"),
                                 (".lora_down.weight", ".lora_up.weight")):
            if k.endswith(down_tag):
                base, role = k[: -len(down_tag)], "down"
            elif k.endswith(up_tag):
                base, role = k[: -len(up_tag)], "up"
            else:
                continue
            break
        if base is None:
            if k.endswith(".alpha"):
                pairs.setdefault(k[: -len(".alpha")], {})["alpha"] = v
            continue
        pairs.setdefault(base, {})[role] = v
    index = {k[: -len(".weight")].replace(".", "_"): k for k in unet_sd if k.endswith(".weight")}
    fused, unmatched = 0, []
    for base, d in pairs.items():
        if "up" not in d or "down" not in d:
            continue
        name = base
        for prefix in ("unet.", "lora_unet_", "base_model.model."):
            if name.startswith(prefix):
                name = name[len(prefix):]
        name = name.replace(".processor", "").replace("to_out_lora", "to_out.0").replace("_lora", "")
        key = name + ".weight" if (name + ".weight") in unet_sd else index.get(name.replace(".", "_"))
        if key is None:
            if not base.startswith(("lora_te_", "text_encoder.", "lora_te1_", "lora_te2_")):
                unmatched.append(base)
            continue
        up, down = d["up"].float(), d["down"].float()
        rank = down.shape[0]
        alpha = float(d["alpha"]) if "alpha" in d else float(rank)
        delta = (up.flatten(1) @ down.flatten(1)) * (scale * alpha / rank)
        w = unet_sd[key]
        unet_sd[key] = (w.float() + delta.reshape(w.shape)).to(w.dtype)
        fused += 1
    if strict and (fused == 0 or unmatched):
        raise KeyError(f"LoRA fusing matched {fused} of {fused + len(unmatched)} UNet modules; unmatched (first 5): {unmatched[:5]}")
    return fused


def _style_loras():
    """One LoRA dict per key style the resolver handles, on a tiny SD-1.5 UNet"""
    g = torch.Generator().manual_seed(3)
    r = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    peft = {f"unet.{TQ}.lora_A.weight": r(4, 64).half(), f"unet.{TQ}.lora_B.weight": r(64, 4).half()}
    # `lora.down` / `lora.up`, with the processor / to_out_lora / _lora rewrites of attention-processor names
    diffusers = {"unet.mid_block.attentions.0.transformer_blocks.0.attn1.processor.to_out_lora.lora.down.weight": r(2, 256),
                 "unet.mid_block.attentions.0.transformer_blocks.0.attn1.processor.to_out_lora.lora.up.weight": r(256, 2),
                 "unet.up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k_lora.lora.down.weight": r(3, 64),
                 "unet.up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k_lora.lora.up.weight": r(256, 3)}
    kohya = "lora_unet_" + "up_blocks.3.resnets.0.conv1".replace(".", "_")
    kt = "lora_unet_" + "down_blocks.1.resnets.0.time_emb_proj".replace(".", "_")
    locon = {kohya + ".lora_down.weight": r(2, 192, 3, 3).half(), kohya + ".lora_up.weight": r(64, 2, 1, 1).half(),
             kohya + ".alpha": torch.tensor(1.0), kt + ".lora_down.weight": r(4, 256), kt + ".lora_up.weight": r(128, 4),
             kt + ".alpha": torch.tensor(8.0), "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": r(2, 8),
             "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_up.weight": r(8, 2)}
    base_model = {f"base_model.model.{TQ}.lora_A.weight": r(8, 64), f"base_model.model.{TQ}.lora_B.weight": r(64, 8)}
    return [peft, diffusers, locon, base_model]


def test_shared_resolver_keeps_fuse_lora_results(tmp_path):
    from ai_rtc_agent_b200.host.weights import fuse_lora
    from oracle import unet as ounet
    from oracle import weights as ow
    unet = ow.make_unet_weights(ounet.tiny_config(False), seed=5)
    _, _, _, _, _, _, lcm, style = _write_tiny_checkpoint(str(tmp_path))
    cases = [(lcm, 1.0), (style, 0.5)] + [(lora, s) for lora, s in zip(_style_loras(), (0.7, 1.3, 0.25, 2.0))]
    got, want = dict(unet), dict(unet)
    for lora, scale in cases:
        assert fuse_lora(got, lora, scale) == _fuse_lora_before(want, lora, scale)
    assert all(torch.equal(got[k], want[k]) for k in unet)
    assert sum(not torch.equal(got[k], unet[k]) for k in unet) == 6


def test_factors_are_what_fusing_means(tmp_path):
    """lora_factors: one (key, up, down, scale * alpha / rank) per pair, files in dict order; fusing them on the host in that
    order gives fuse_lora's weights bit for bit"""
    from safetensors.torch import save_file
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.weights import fuse_lora, lora_factors
    from oracle import unet as ounet
    from oracle import weights as ow
    unet = ow.make_unet_weights(ounet.tiny_config(False), seed=5)
    shapes = A.unet_param_shapes(A.TINY_SD15)
    paths = {}
    for i, (lora, scale) in enumerate(zip(_style_loras(), (0.7, 1.3, 0.25, 2.0))):
        p = str(tmp_path / f"l{i}.safetensors")
        save_file({k: v.contiguous() for k, v in lora.items()}, p)
        paths[p] = scale
    factors = lora_factors(shapes, paths)
    assert [f[0] for f in factors] == [TQ + ".weight", "mid_block.attentions.0.transformer_blocks.0.attn1.to_out.0.weight",
                                       "up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k.weight",
                                       "down_blocks.1.resnets.0.time_emb_proj.weight", "up_blocks.3.resnets.0.conv1.weight",
                                       TQ + ".weight"]   # within a file: the file's key order (sorted by safetensors)
    conv = factors[4]
    assert conv[1].shape == (64, 2) and conv[2].shape == (2, 192 * 9) and conv[3] == 0.25 * 1.0 / 2
    assert factors[3][3] == 0.25 * 8.0 / 4
    want = dict(unet)
    for p, s in paths.items():
        from ai_rtc_agent_b200.host.weights import load_lora_file
        fuse_lora(want, load_lora_file(p), s)
    got = dict(unet)
    for key, up, down, scale in factors:
        w = got[key]
        got[key] = (w.float() + ((up.float() @ down.float()) * scale).reshape(w.shape)).to(w.dtype)
    assert all(torch.equal(got[k], want[k]) for k in unet)
    assert lora_factors(shapes, None) == [] and lora_factors(shapes, {}) == []


class _RecordingLib:
    """Stands in for libb200sd.so: records every call"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            if name == "b2sd_apply_lora":
                n, arr = args[1], args[2]
                self.factors = [(arr[i].key.decode(), arr[i].rank, arr[i].dtype, arr[i].scale) for i in range(n)]
            return 0
        return call


def _fake_engine(shapes, monkeypatch):
    from ai_rtc_agent_b200.host import stream as S
    eng = S.StreamDiffusion.__new__(S.StreamDiffusion)
    eng.live_lora, eng._prepared, eng._unet_shapes = True, True, shapes
    eng._lib, eng.lanes, eng._states, eng._handle = _RecordingLib(), [], set(), None
    eng.device = torch.device("cpu")
    monkeypatch.setattr(S, "_on_device", lambda t, device: t)
    monkeypatch.setattr(S.StreamDiffusion, "_stream", lambda self: 0)
    return eng


def test_errors_are_raised_before_the_engine_is_called(tmp_path, monkeypatch):
    from safetensors.torch import save_file
    from ai_rtc_agent_b200.host import arch as A
    shapes = A.unet_param_shapes(A.TINY_SD15)
    eng = _fake_engine(shapes, monkeypatch)
    good = str(tmp_path / "good.safetensors")
    save_file({k: v.contiguous() for k, v in _style_loras()[0].items()}, good)
    # a pickle, and a file named like safetensors that is not one
    pkl = str(tmp_path / "style.pt")
    torch.save(_style_loras()[0], pkl)
    fake = str(tmp_path / "fake.safetensors")
    with open(fake, "wb") as f:
        f.write(b"\x80\x04not a safetensors header")
    # a pair whose shape does not fit its parameter, a LoRA on no UNet module, a text-encoder-only LoRA
    bad_shape = str(tmp_path / "shape.safetensors")
    save_file({f"unet.{TQ}.lora_A.weight": torch.zeros(4, 65), f"unet.{TQ}.lora_B.weight": torch.zeros(64, 4)}, bad_shape)
    nowhere = str(tmp_path / "nowhere.safetensors")
    save_file({"unet.some.module.lora_A.weight": torch.zeros(2, 8), "unet.some.module.lora_B.weight": torch.zeros(8, 2)}, nowhere)
    te_only = str(tmp_path / "te.safetensors")
    save_file({"lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": torch.zeros(2, 8),
               "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_up.weight": torch.zeros(8, 2)}, te_only)
    for bad, err in ((pkl, ValueError), (fake, ValueError), (bad_shape, ValueError), (nowhere, KeyError), (te_only, KeyError)):
        with pytest.raises(err):
            eng.apply_lora({good: 1.0, bad: 1.0})    # the good file first: nothing of it may reach the engine either
        assert eng._lib.calls == []
    eng.apply_lora({good: 0.5})
    assert [c[0] for c in eng._lib.calls] == ["b2sd_apply_lora", "b2sd_refresh_conditioning"]
    assert eng._lib.factors == [(TQ + ".weight", 4, 0, pytest.approx(0.5))]
    eng.apply_lora(None)
    assert eng._lib.calls[-2][0] == "b2sd_apply_lora" and eng._lib.factors == []


def test_fp32_factors_are_scaled_exactly():
    """fp32 factors reach the engine as fp32 scaled by powers of two (largest magnitude in [1, 2)) with the scale compensated;
    fp16 pairs as they are"""
    from ai_rtc_agent_b200.host.stream import _factor_operands
    g = torch.Generator().manual_seed(1)
    up, down = torch.randn(64, 4, generator=g) * 3e-4, torch.randn(4, 32, generator=g) * 40
    u, d, s = _factor_operands(up, down, 0.75)
    assert u.dtype == d.dtype == torch.float32
    assert 1 <= u.abs().max() < 2 and 1 <= d.abs().max() < 2
    assert torch.equal((u.double() @ d.double()) * s, (up.double() @ down.double()) * 0.75)
    uh, dh = up.half(), down.half()
    u, d, s = _factor_operands(uh, dh, 0.75)
    assert u is not None and torch.equal(u, uh) and torch.equal(d, dh) and s == 0.75


def test_live_mode_is_chosen_at_construction(monkeypatch):
    """StreamDiffusionPipeline(live_lora=...) and $B200SD_LIVE_LORA select the mode; the wrapper learns it without a
    constructor keyword (its signature stays the reference's); update_lora without the mode raises"""
    from ai_rtc_agent_b200.host import pipeline as P
    from ai_rtc_agent_b200.host import wrapper as Wm
    assert "live_lora" not in inspect.signature(Wm.StreamDiffusionWrapper.__init__).parameters
    seen = []

    class Stop(Exception):
        pass

    def fake_load(self, **kw):
        seen.append((self.live_lora, self._pending_lora))
        raise Stop
    monkeypatch.setattr(Wm.StreamDiffusionWrapper, "_load_model", fake_load)
    for env, arg, want in (("", None, False), ("1", None, True), ("0", True, True), ("1", False, False), ("off", None, False)):
        monkeypatch.setenv("B200SD_LIVE_LORA", env)
        with pytest.raises(Stop):
            P.StreamDiffusionPipeline("tiny-sd15", live_lora=arg)
        assert seen[-1] == (want, None)
        with pytest.raises(Stop):
            Wm.StreamDiffusionWrapper("tiny-sd15", [0], lora_dict={"a.safetensors": 1.0})
        assert seen[-1] == (env in ("1",), {"a.safetensors": 1.0} if env == "1" else None)
    monkeypatch.setenv("B200SD_LIVE_LORA", "maybe")
    with pytest.raises(ValueError):
        P.StreamDiffusionPipeline("tiny-sd15")
    w = Wm.StreamDiffusionWrapper.__new__(Wm.StreamDiffusionWrapper)
    w.live_lora = False
    with pytest.raises(RuntimeError, match="live LoRA mode"):
        w.update_lora({})
    p = P.StreamDiffusionPipeline.__new__(P.StreamDiffusionPipeline)
    p.model = w
    with pytest.raises(RuntimeError, match="live_lora=True"):
        p.update_lora(None)


def test_lora_factor_layout_matches_the_c_header(tmp_path):
    """sizeof / offsetof of b2sd_lora_factor against its ctypes mirror (gcc on the plain-C header)"""
    import ctypes
    import subprocess
    from ai_rtc_agent_b200.host import capi
    cls = capi.LoraFactor
    lines = ['printf("%zu\\n", sizeof(b2sd_lora_factor));'] + \
        [f'printf("%zu\\n", offsetof(b2sd_lora_factor, {f}));' for f, _ in cls._fields_]
    want = [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sd.h"\nint main(void){\n' + "\n".join(lines) +
                   "\nreturn 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == want
