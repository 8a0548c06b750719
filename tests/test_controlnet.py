"""ControlNet on the CPU: the oracle restatement, the parameter inventories, checkpoint loading, the packed-blob key and the
wrapper's processor validation.  (Engine parity on the H100: tests/test_controlnet_gpu.py.)"""
import json
import math
import os

import pytest
import torch


def _tiny(turbo):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    return ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)


def _inputs(cfg, B=2, hw=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, 4, hw // 8, hw // 8), generator=g)
    t = torch.tensor([999, 499][:B] + [259] * max(0, B - 2), dtype=torch.long)
    ctx = torch.randn((B, 77, cfg.cross_attention_dim), generator=g)
    control = torch.rand((1, 3, hw, hw), generator=g)
    return x, t, ctx, control


@pytest.mark.parametrize("turbo", [True, False])
def test_controlnet_body_is_the_unet_down_path(turbo):
    """A ControlNet holding the UNet's conv_in / time embedding / down / mid weights, with a zero conditioning-embedding
    conv_out, computes exactly the UNet's down.I.J and mid activations before its zero convs."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg, _ = _tiny(turbo)
    usd = ow.to_float(ow.make_unet_weights(cfg))
    cn = ow.to_float(ocn.make_weights(cfg))
    for k in cn:
        if k.startswith(("conv_in.", "time_embedding.", "down_blocks.", "mid_block.")):
            cn[k] = usd[k].clone()
    p = "controlnet_cond_embedding.conv_out."
    cn[p + "weight"].zero_()
    cn[p + "bias"].zero_()
    x, t, ctx, control = _inputs(cfg)
    ref, got = {}, {}
    ounet.unet_forward(usd, cfg, x, t, ctx, ref)
    ocn.controlnet_forward(cn, cfg, x, t, ctx, control, got)
    assert torch.count_nonzero(got["cond"]) == 0
    names = ["conv_in", "mid"] + [f"down.{i}.{j}" for i in range(4) for j in range(cfg.layers_per_block)]
    for n in names:
        assert torch.equal(got[n], ref[n]), n


@pytest.mark.parametrize("turbo", [True, False])
def test_unet_with_residuals_restates_the_unet(turbo):
    """The UNet forward with ControlNet residuals equals oracle/unet.py's bit for bit when the residuals are zero, and each
    residual moves the output (it reaches the up path)."""
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg, _ = _tiny(turbo)
    usd = ow.to_float(ow.make_unet_weights(cfg))
    x, t, ctx, _ = _inputs(cfg)
    taps = {}
    ounet.unet_forward(usd, cfg, x, t, ctx, taps)
    zeros = [torch.zeros_like(taps["conv_in"])]
    for i in range(4):
        zeros += [torch.zeros_like(taps[f"down.{i}.0"])] * cfg.layers_per_block
        if i != 3:
            zeros.append(torch.zeros_like(taps[f"down.{i}.0"][..., ::2, ::2]))
    assert len(zeros) == len(ocn.down_residual_channels(cfg)) == 12
    mid0 = torch.zeros_like(taps["mid"])
    base = ounet.unet_forward(usd, cfg, x, t, ctx)
    assert torch.equal(ocn.unet_forward(usd, cfg, x, t, ctx, zeros, mid0), base)
    for k in (0, 5, 11):
        res = list(zeros)
        res[k] = torch.ones_like(res[k])
        assert not torch.allclose(ocn.unet_forward(usd, cfg, x, t, ctx, res, mid0), base), f"residual {k} has no effect"
    assert not torch.allclose(ocn.unet_forward(usd, cfg, x, t, ctx, zeros, torch.ones_like(mid0)), base)


def test_zero_init_controlnet_leaves_the_stream_unchanged():
    """A freshly initialised ControlNet (zero convs = 0) changes nothing: the stream oracle's frames equal the plain one's."""
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import stream as ostream
    from oracle import weights as ow
    cfg, _ = _tiny(True)
    usd, vsd = ow.to_float(ow.make_unet_weights(cfg)), ow.to_float(ow.make_taesd_weights())
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim).float()
    a = ostream.StreamOracle(usd, cfg, vsd, [20, 40], 64, 64)
    b = ocn.ControlNetStreamOracle(usd, cfg, vsd, ow.to_float(ocn.make_weights(cfg, zero_init=True)), [20, 40], 64, 64)
    c = ocn.ControlNetStreamOracle(usd, cfg, vsd, ow.to_float(ocn.make_weights(cfg)), [20, 40], 64, 64)
    for o in (a, b, c):
        o.prepare(emb, guidance_scale=0.0, seed=3)
    for i in range(2):
        frame = ow.make_frame(64, 64, seed=i)
        fa, fb, fc = (opipe.frame_to_u8(o, frame) for o in (a, b, c))
        assert torch.equal(fa, fb)
        assert not torch.equal(fa, fc)   # non-zero zero convs (the synthetic default) do condition the output


@pytest.mark.parametrize("name", ["tiny-sd15", "tiny-turbo", "sd15", "sd-turbo"])
def test_controlnet_inventories_agree(name):
    """host/arch.py and oracle/controlnet.py list the same parameters with the same shapes (two independent restatements)."""
    from ai_rtc_agent_b200.host import arch as A
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    arch = {"tiny-sd15": A.TINY_SD15, "tiny-turbo": A.TINY_TURBO, "sd15": A.SD15, "sd-turbo": A.SD_TURBO}[name]
    cfg = {"tiny-sd15": ounet.tiny_config(False), "tiny-turbo": ounet.tiny_config(True), "sd15": ounet.SD15,
           "sd-turbo": ounet.SD_TURBO}[name]
    host, orc = A.controlnet_param_shapes(arch), ocn.param_shapes(cfg)
    assert sorted(host) == sorted(orc)
    for k in host:
        assert math.prod(host[k]) == math.prod(orc[k]), k
    n = sum(math.prod(v) for v in host.values())
    print(f"{name}: {len(host)} ControlNet tensors, {n} parameters")


def _write_controlnet_dir(path, arch, sd, config_over=None):
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    cfg = {"_class_name": "ControlNetModel", "block_out_channels": list(arch.block_out_channels),
           "cross_attention_dim": arch.cross_attention_dim, "layers_per_block": arch.layers_per_block,
           "conditioning_embedding_out_channels": [16, 32, 96, 256]}
    cfg.update(config_over or {})
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(path, "diffusion_pytorch_model.safetensors"))


def test_controlnet_checkpoint_directory_loads(tmp_path):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    arch = A.TINY_SD15
    sd = W.synthetic_controlnet(arch, seed=9)
    _write_controlnet_dir(tmp_path / "cn", arch, sd)
    got = W.load_controlnet(str(tmp_path / "cn"), arch)
    assert sorted(got) == sorted(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert W.resolve_controlnet(str(tmp_path / "cn"), arch, synthetic_ok=False).keys() == sd.keys()
    bad = dict(sd)
    bad["controlnet_down_blocks.4.weight"] = torch.zeros((64, 64, 1, 1), dtype=torch.float16)   # level 1 has 128 channels
    _write_controlnet_dir(tmp_path / "bad", arch, bad)
    with pytest.raises(ValueError, match="controlnet_down_blocks.4.weight"):
        W.load_controlnet(str(tmp_path / "bad"), arch)
    _write_controlnet_dir(tmp_path / "other", arch, sd, {"cross_attention_dim": 1024})
    with pytest.raises(ValueError, match="cross_attention_dim"):
        W.load_controlnet(str(tmp_path / "other"), arch)
    with pytest.raises(FileNotFoundError):
        W.resolve_controlnet(str(tmp_path / "missing"), arch, synthetic_ok=False)


def test_synthetic_controlnet_zero_init():
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    sd = W.synthetic_controlnet(A.TINY_TURBO)
    z = W.synthetic_controlnet(A.TINY_TURBO, zero_init=True)
    zero_keys = [k for k in z if k.startswith(("controlnet_down_blocks.", "controlnet_mid_block.",
                                               "controlnet_cond_embedding.conv_out."))]
    assert len(zero_keys) == 2 * 13 + 2
    for k in zero_keys:
        assert torch.count_nonzero(z[k]) == 0
        assert k.endswith(".bias") or torch.count_nonzero(sd[k]) > 0
    A.validate_state_dict(sd, A.controlnet_param_shapes(A.TINY_TURBO), "synthetic ControlNet")


def test_packed_blob_path_covers_the_controlnet(tmp_path):
    from ai_rtc_agent_b200.host import weights as W
    args = ("eng", "lykon/dreamshaper-8", "sd15", True, None, None, None, False)
    plain = W.packed_blob_path(*args)
    a = W.packed_blob_path(*args, controlnet="lllyasviel/sd-controlnet-hed")
    b = W.packed_blob_path(*args, controlnet="lllyasviel/sd-controlnet-canny")
    c = W.packed_blob_path(*args, controlnet="lllyasviel/sd-controlnet-hed", control_processor="hed")
    assert len({plain, a, b, c}) == 4
    assert W.packed_blob_path(*args, controlnet="lllyasviel/sd-controlnet-hed") == a
    from ai_rtc_agent_b200.host import arch as A
    d = tmp_path / "cn"
    _write_controlnet_dir(d, A.TINY_SD15, W.synthetic_controlnet(A.TINY_SD15))
    p1 = W.packed_blob_path(*args, controlnet=str(d))
    st = os.stat(d / "diffusion_pytorch_model.safetensors")
    os.utime(d / "diffusion_pytorch_model.safetensors", (st.st_atime, st.st_mtime + 10))
    assert W.packed_blob_path(*args, controlnet=str(d)) != p1   # replaced weights must not hit the old blob


@pytest.mark.parametrize("proc", ["canny", "depth", "openpose"])
def test_wrapper_rejects_other_control_preprocessors(proc):
    """Only "hed" (the reference's default) and None (the frame is the control image) are built; any other preprocessor id is
    refused by name instead of silently conditioning on the raw frame."""
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    with pytest.raises(NotImplementedError, match=repr(proc)):
        StreamDiffusionWrapper("tiny-turbo", [32], controlnet_id_or_path="some/controlnet", controlnet_processor_id=proc)


def _load_model_calls(monkeypatch, **kw):
    """Construct the wrapper with _load_model replaced by a recorder: what the argument validation lets through, and with
    which ControlNet settings."""
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    calls = []
    monkeypatch.setattr(StreamDiffusionWrapper, "_load_model", lambda self, **a: calls.append(a) or None)
    StreamDiffusionWrapper("tiny-turbo", [32], **kw)
    return calls


def test_wrapper_passes_hed_and_none_through(monkeypatch):
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path="some/controlnet")   # default processor: "hed"
    assert calls[0]["controlnet_id_or_path"] == "some/controlnet" and calls[0]["controlnet_processor_id"] == "hed"
    calls = _load_model_calls(monkeypatch, controlnet_id_or_path="some/controlnet", controlnet_processor_id=None)
    assert calls[0]["controlnet_processor_id"] is None
    # like the reference, the processor id alone (no ControlNet) is not validated
    calls = _load_model_calls(monkeypatch, controlnet_processor_id="canny")
    assert calls[0]["controlnet_id_or_path"] is None


def test_pack_cli_takes_the_controlnet_options():
    from ai_rtc_agent_b200 import pack
    a = pack.build_parser().parse_args(["--controlnet-id", "lllyasviel/sd-controlnet-hed"])
    assert a.controlnet_id == "lllyasviel/sd-controlnet-hed" and a.controlnet_processor_id == "hed"
    a = pack.build_parser().parse_args(["--controlnet-processor-id", "none"])
    assert a.controlnet_id is None and a.controlnet_processor_id is None


# ---- HED ----------------------------------------------------------------------------------------------------------------------
class _DoubleConvBlock(torch.nn.Module):
    """controlnet_aux's DoubleConvBlock, rebuilt with torch.nn (independent of oracle/hed.py's functional restatement)."""

    def __init__(self, cin, cout, n):
        super().__init__()
        self.convs = torch.nn.Sequential()
        self.convs.append(torch.nn.Conv2d(cin, cout, 3, padding=1))
        for _ in range(1, n):
            self.convs.append(torch.nn.Conv2d(cout, cout, 3, padding=1))
        self.projection = torch.nn.Conv2d(cout, 1, 1)

    def forward(self, x, down):
        h = torch.nn.functional.max_pool2d(x, kernel_size=(2, 2), stride=(2, 2)) if down else x
        for conv in self.convs:
            h = torch.nn.functional.relu(conv(h))
        return h, self.projection(h)


class _ControlNetHED(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.norm = torch.nn.Parameter(torch.zeros(1, 3, 1, 1))
        self.block1 = _DoubleConvBlock(3, 64, 2)
        self.block2 = _DoubleConvBlock(64, 128, 2)
        self.block3 = _DoubleConvBlock(128, 256, 3)
        self.block4 = _DoubleConvBlock(256, 512, 3)
        self.block5 = _DoubleConvBlock(512, 512, 3)

    def forward(self, x):
        h = x - self.norm
        outs = []
        for i, blk in enumerate((self.block1, self.block2, self.block3, self.block4, self.block5)):
            h, p = blk(h, i > 0)
            outs.append(p)
        return outs


def _resize_linear(img, hh, ww):
    """cv2.resize(img, (ww, hh), interpolation=INTER_LINEAR) for float images: half-pixel centres, edges clamped (numpy)."""
    import numpy as np
    h, w = img.shape

    def axis(n_out, n_in):
        s = np.maximum((np.arange(n_out) + 0.5) * (n_in / n_out) - 0.5, 0.0)
        i0 = np.minimum(np.floor(s).astype(int), n_in - 1)
        return i0, np.minimum(i0 + 1, n_in - 1), s - i0
    y0, y1, fy = axis(hh, h)
    x0, x1, fx = axis(ww, w)
    top = img[y0][:, x0] * (1 - fx) + img[y0][:, x1] * fx
    bot = img[y1][:, x0] * (1 - fx) + img[y1][:, x1] * fx
    return top * (1 - fy[:, None]) + bot * fy[:, None]


def test_hed_oracle_matches_an_independent_build():
    """oracle/hed.py equals ControlNetHED_Apache2 rebuilt with torch.nn (loaded strictly from the same state dict) followed by
    HEDdetector's numpy post-processing, on a 96x128 frame."""
    import numpy as np
    from ai_rtc_agent_b200.host import arch as A
    from oracle import hed as ohed
    from oracle import weights as ow
    sd = {k: v.half().float() for k, v in A.synthetic_hed().items()}
    net = _ControlNetHED()
    net.load_state_dict(sd, strict=True)
    frame = ow.make_frame(96, 128, seed=5)
    x255 = frame.permute(0, 3, 1, 2).float()
    with torch.no_grad():
        edges = [e[0, 0].numpy().astype(np.float32) for e in net(x255)]
        got_maps = ohed.side_outputs(sd, x255)
        got = ohed.detect(sd, x255)
    for e, g in zip(edges, got_maps):
        assert np.allclose(e, g[0, 0].numpy(), rtol=1e-4, atol=1e-4)
    fused = np.stack([_resize_linear(e, 96, 128) for e in edges], axis=2)
    ref = (1 / (1 + np.exp(-np.mean(fused, axis=2))) * 255.0).clip(0, 255).astype(np.uint8)
    d = np.abs(ref.astype(int) - got[0, 0].numpy().astype(int))
    assert d.max() <= 1 and (d == 0).mean() >= 0.999, (d.max(), (d == 0).mean())
    assert 10 < ref.std() and ref.min() < 100 < ref.max(), "synthetic HED weights should give a graded, unsaturated edge map"


def test_hed_checkpoint_loads(tmp_path):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    sd = A.synthetic_hed(seed=3)
    torch.save(sd, tmp_path / "ControlNetHED.pth")
    got = W.load_hed(str(tmp_path / "ControlNetHED.pth"))
    assert sorted(got) == sorted(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    bad = dict(sd)
    bad["block3.convs.1.weight"] = torch.zeros((256, 128, 3, 3))
    torch.save(bad, tmp_path / "bad.pth")
    with pytest.raises(ValueError, match="block3.convs.1.weight"):
        W.load_hed(str(tmp_path / "bad.pth"))
    n = sum(math.prod(v) for v in A.hed_param_shapes().values())
    print(f"HED: {len(A.hed_param_shapes())} tensors, {n} parameters")
