"""The model's own AutoencoderKL without a GPU: the fp32 oracle against an independent torch.nn build, the two parameter
inventories, checkpoint loading, and the wrapper / blob-path plumbing of use_tiny_vae=False."""
import json
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F


# ---- an independent torch.nn build of diffusers' AutoencoderKL (module names = state-dict keys) --------------------------------
class _Resnet(nn.Module):
    def __init__(self, ci, co):
        super().__init__()
        self.norm1, self.conv1 = nn.GroupNorm(32, ci, eps=1e-6), nn.Conv2d(ci, co, 3, padding=1)
        self.norm2, self.conv2 = nn.GroupNorm(32, co, eps=1e-6), nn.Conv2d(co, co, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(ci, co, 1) if ci != co else None

    def forward(self, x):
        h = self.conv2(F.silu(self.norm2(self.conv1(F.silu(self.norm1(x))))))
        return (x if self.conv_shortcut is None else self.conv_shortcut(x)) + h


class _Attn(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.group_norm = nn.GroupNorm(32, c, eps=1e-6)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c)])

    def forward(self, x):
        b, c, h, w = x.shape
        t = self.group_norm(x).flatten(2).transpose(1, 2)
        o = F.scaled_dot_product_attention(self.to_q(t)[:, None], self.to_k(t)[:, None], self.to_v(t)[:, None])[:, 0]
        return self.to_out[0](o).transpose(1, 2).reshape(b, c, h, w) + x


class _Mid(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(c, c), _Resnet(c, c)])
        self.attentions = nn.ModuleList([_Attn(c)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class _Down(nn.Module):
    def __init__(self, ci, co, n, down):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(ci if j == 0 else co, co) for j in range(n)])
        self.downsamplers = nn.ModuleList([nn.Module()]) if down else None
        if down:
            self.downsamplers[0].conv = nn.Conv2d(co, co, 3, stride=2)

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.downsamplers[0].conv(F.pad(x, (0, 1, 0, 1))) if self.downsamplers is not None else x


class _Up(nn.Module):
    def __init__(self, ci, co, n, up):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(ci if j == 0 else co, co) for j in range(n)])
        self.upsamplers = nn.ModuleList([nn.Module()]) if up else None
        if up:
            self.upsamplers[0].conv = nn.Conv2d(co, co, 3, padding=1)

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.upsamplers[0].conv(F.interpolate(x, scale_factor=2.0, mode="nearest")) if self.upsamplers is not None else x


class _KL(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.encoder, self.decoder = nn.Module(), nn.Module()
        e, d = self.encoder, self.decoder
        e.conv_in = nn.Conv2d(3, ch[0], 3, padding=1)
        e.down_blocks = nn.ModuleList([_Down(ch[max(i - 1, 0)], c, 2, i < 3) for i, c in enumerate(ch)])
        e.mid_block, e.conv_norm_out, e.conv_out = _Mid(ch[-1]), nn.GroupNorm(32, ch[-1], eps=1e-6), nn.Conv2d(ch[-1], 8, 3, padding=1)
        self.quant_conv, self.post_quant_conv = nn.Conv2d(8, 8, 1), nn.Conv2d(4, 4, 1)
        rev = list(reversed(ch))
        d.conv_in, d.mid_block = nn.Conv2d(4, ch[-1], 3, padding=1), _Mid(ch[-1])
        d.up_blocks = nn.ModuleList([_Up(rev[max(i - 1, 0)], c, 3, i < 3) for i, c in enumerate(rev)])
        d.conv_norm_out, d.conv_out = nn.GroupNorm(32, rev[-1], eps=1e-6), nn.Conv2d(rev[-1], 3, 3, padding=1)

    def encode_mean(self, x):
        e = self.encoder
        x = e.conv_in(x)
        for b in e.down_blocks:
            x = b(x)
        return self.quant_conv(e.conv_out(F.silu(e.conv_norm_out(e.mid_block(x)))))[:, :4]

    def decode(self, z):
        d = self.decoder
        x = d.mid_block(d.conv_in(self.post_quant_conv(z)))
        for b in d.up_blocks:
            x = b(x)
        return d.conv_out(F.silu(d.conv_norm_out(x)))


def test_oracle_matches_torch_nn_build():
    """oracle/autoencoder_kl.py against the nn.Module build loaded strictly from the same (synthetic, fp16-rounded) state dict."""
    from ai_rtc_agent_b200.host import arch as A
    from oracle import autoencoder_kl as oakl
    sd = {k: v.float() for k, v in A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL).items()}
    net = _KL(A.TINY_AUTOENCODER_KL.block_out_channels)
    net.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(0)
    img = torch.rand((1, 3, 64, 96), generator=g) * 2 - 1
    z = torch.randn((1, 4, 8, 12), generator=g)
    with torch.no_grad():
        for got, ref in ((oakl.encode_mean(sd, img, oakl.TINY), net.encode_mean(img)), (oakl.decode(sd, z, oakl.TINY), net.decode(z))):
            assert got.shape == ref.shape
            assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


@pytest.mark.parametrize("which", ["full", "tiny"])
def test_parameter_inventories_agree(which):
    from ai_rtc_agent_b200.host import arch as A
    from oracle import autoencoder_kl as oakl
    host = A.autoencoder_kl_param_shapes(A.AUTOENCODER_KL if which == "full" else A.TINY_AUTOENCODER_KL)
    orc = oakl.param_shapes(oakl.FULL if which == "full" else oakl.TINY)
    assert host == orc
    if which == "full":
        assert sum(torch.Size(s).numel() for s in host.values()) == 83653863   # diffusers AutoencoderKL of SD-1.5 / SD-2.1


def _write_checkpoint(tmp_path, sd, scaling_factor=None):
    from safetensors.torch import save_file
    repo = tmp_path / "model"
    (repo / "vae").mkdir(parents=True)
    save_file({k: v.contiguous() for k, v in sd.items()}, str(repo / "vae" / "diffusion_pytorch_model.safetensors"))
    if scaling_factor is not None:
        (repo / "vae" / "config.json").write_text(json.dumps({"scaling_factor": scaling_factor}))
    return str(repo)


@pytest.mark.parametrize("legacy", [False, True])
def test_checkpoint_directory_loads(tmp_path, legacy):
    """<model>/vae/diffusion_pytorch_model.safetensors with the current attention names, and with the legacy
    query / key / value / proj_attn names and [C, C, 1, 1] projections; scaling_factor from vae/config.json."""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    sd = A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL)
    disk = dict(sd)
    if legacy:
        names = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}
        disk = {}
        for k, v in sd.items():
            for new, old in names.items():
                if f".attentions.0.{new}." in k:
                    k = k.replace(f".attentions.0.{new}.", f".attentions.0.{old}.")
                    if v.dim() == 2:
                        v = v[:, :, None, None]
            disk[k] = v
    repo = _write_checkpoint(tmp_path, disk, scaling_factor=0.13025)
    got = W.load_autoencoder_kl(repo, A.TINY_AUTOENCODER_KL)
    assert got.keys() == sd.keys() and all(torch.equal(got[k], sd[k]) for k in sd)
    assert W.resolve_vae_scaling_factor(repo) == pytest.approx(0.13025)
    assert W.resolve_vae_scaling_factor(None) == pytest.approx(0.18215)


def test_wrong_shapes_are_refused_by_name(tmp_path):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import weights as W
    sd = A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL)
    sd["decoder.up_blocks.1.resnets.2.conv1.weight"] = sd["decoder.up_blocks.1.resnets.2.conv1.weight"][:, :64].contiguous()
    with pytest.raises(ValueError, match=r"decoder\.up_blocks\.1\.resnets\.2\.conv1\.weight"):
        W.load_autoencoder_kl(_write_checkpoint(tmp_path, sd), A.TINY_AUTOENCODER_KL)
    sd = A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL)
    del sd["post_quant_conv.bias"]
    with pytest.raises(ValueError, match=r"post_quant_conv\.bias"):
        W.load_autoencoder_kl(_write_checkpoint(tmp_path / "b", sd), A.TINY_AUTOENCODER_KL)


def test_wrapper_passes_use_tiny_vae_through(monkeypatch):
    """use_tiny_vae=False reaches the engine with the model's AutoencoderKL weights (seeded synthetic here); vae_id is ignored."""
    import ai_rtc_agent_b200.host.wrapper as Wm
    from ai_rtc_agent_b200.host import arch as A
    seen = {}

    class FakeStream:
        def __init__(self, arch, unet_sd, vae_sd, t_index_list, encoder, **kw):
            seen.update(kw, vae_keys=set(vae_sd))

    monkeypatch.setattr(Wm, "StreamDiffusion", FakeStream)
    monkeypatch.setattr(Wm, "make_prompt_encoder", lambda *a, **k: (lambda p: None))
    monkeypatch.setenv("B200SD_PACK_CACHE", "0")
    Wm.StreamDiffusionWrapper("tiny-turbo", [32], use_tiny_vae=False, vae_id="madebyollin/taesd", engine_dir=None)
    assert seen["use_tiny_vae"] is False and seen["vae_scaling_factor"] == pytest.approx(0.18215)
    assert seen["vae_keys"] == set(A.autoencoder_kl_param_shapes(A.TINY_AUTOENCODER_KL))
    seen.clear()
    Wm.StreamDiffusionWrapper("tiny-turbo", [32], engine_dir=None)
    assert seen["use_tiny_vae"] is True and seen["vae_keys"] == set(A.taesd_param_shapes())
    with pytest.raises(NotImplementedError, match="safety checker"):   # other refused keywords stay refused
        Wm.StreamDiffusionWrapper("tiny-turbo", [32], use_tiny_vae=False, use_safety_checker=True, engine_dir=None)


def test_blob_path_unchanged_for_taesd_and_distinct_for_kl(tmp_path):
    from ai_rtc_agent_b200.host import weights as W
    kw = dict(engine_dir=str(tmp_path), model_id_or_path="stabilityai/sd-turbo", arch_name="sd-turbo", use_lcm_lora=False,
              lcm_lora_id=None, lora_dict=None, vae_id=None, synthetic=True)
    taesd = W.packed_blob_path(**kw)
    # the name every TAESD blob had before the full VAE existed (same recipe, same hash)
    assert os.path.basename(taesd) == "b2sd-sd-turbo-2ed6eee74f1a6f91.b2pack"
    assert W.packed_blob_path(**kw, full_vae=False) == taesd
    kl = W.packed_blob_path(**kw, full_vae=True)
    assert kl != taesd and os.path.dirname(kl) == os.path.dirname(taesd)


def test_pack_cli_has_full_vae_flag():
    import importlib
    pack = importlib.import_module("ai_rtc_agent_b200.pack")
    assert pack.build_parser().parse_args(["--full-vae"]).full_vae is True
    assert pack.build_parser().parse_args([]).full_vae is False


def test_kl_stream_oracle_uses_the_autoencoder_kl():
    """oracle/stream_kl.py: x_t = alpha0 * scaling_factor * mean + beta0 * noise, and the image is the AutoencoderKL's decode of
    x0 / scaling_factor; with a ControlNet the same VAE path runs after the control image is set."""
    from ai_rtc_agent_b200.host import arch as A
    from oracle import autoencoder_kl as oakl
    from oracle import controlnet as ocn
    from oracle import pipeline as opipe
    from oracle import stream_kl as oskl
    from oracle import unet as ounet
    from oracle import weights as ow
    cfg = ounet.tiny_config(True)
    usd = ow.to_float(ow.make_unet_weights(cfg))
    vsd = ow.to_float(A.synthetic_autoencoder_kl(A.TINY_AUTOENCODER_KL))
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim).float()
    frame = ow.make_frame(64, 64, seed=3)
    img = 2.0 * opipe.preprocess(frame).unsqueeze(0) - 1.0
    for cls, extra in ((oskl.KLStreamOracle, ()), (oskl.KLControlNetStreamOracle, (ow.to_float(ocn.make_weights(cfg)),))):
        orc = cls(usd, cfg, vsd, *extra, [32], 64, 64, vae_kl=oakl.TINY)
        orc.prepare(emb, guidance_scale=0.0)
        opipe.frame_to_u8(orc, frame)
        z = oakl.encode_mean(vsd, img, oakl.TINY) * oakl.SCALING_FACTOR
        x_t = orc.alpha_prod_t_sqrt[0] * z + orc.beta_prod_t_sqrt[0] * orc.init_noise[0]
        assert torch.allclose(orc.last["x_t"], x_t, atol=1e-5), cls.__name__
        dec = oakl.decode(vsd, orc.last["x0"] / oakl.SCALING_FACTOR, oakl.TINY)
        assert torch.allclose(orc.last["image"], dec, atol=1e-5), cls.__name__
