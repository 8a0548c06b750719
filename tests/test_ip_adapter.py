"""IP-Adapter without a GPU: the adapter loader and its checks, the ip_adapter.{i} -> UNet module mapping, the fp32 oracle
against an independent torch.nn build, the packed-blob recipe, and the host routing of image prompts over a recording fake of
the C library."""
import ctypes
import os
import pickle
import types
import weakref

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ai_rtc_agent_b200.host import arch as A
from ai_rtc_agent_b200.host import image_prompt as I


def _save(sd, path):
    from safetensors.torch import save_file
    save_file({k: v.contiguous() for k, v in sd.items()}, str(path))
    return str(path)


# ---- loader ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", [A.TINY_SD15, A.SD15, A.SD_TURBO], ids=lambda a: a.name)
def test_loader_accepts_synthetic_adapter(tmp_path, arch):
    sd = I.synthetic_adapter_state_dict(arch, embed_dim=64 if arch is A.TINY_SD15 else 1024)
    ad = I.load_adapter(_save(sd, tmp_path / "ip-adapter_sd15.safetensors"), arch)
    assert ad.n_tok == I.IP_TOKENS and len(ad.unet) == 2 * len(I.cross_attention_modules(arch)) == 32
    assert I.load_adapter(str(tmp_path), arch).path.endswith("ip-adapter_sd15.safetensors"), "a directory holding one file"
    for k, v in ad.unet.items():
        assert k.endswith(("attn2.to_k_ip.weight", "attn2.to_v_ip.weight")) and v.dtype == torch.float16
    tok = ad.tokens(torch.randn(ad.embed_dim))
    assert tok.shape == (1, I.IP_TOKENS, arch.cross_attention_dim) and tok.dtype == torch.float16


def test_loader_refuses_a_pickle(tmp_path):
    sd = I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=64)
    with open(tmp_path / "ip-adapter_sd15.bin", "wb") as f:
        pickle.dump({"image_proj": sd}, f)
    with pytest.raises(ValueError, match="only .safetensors"):
        I.load_adapter(str(tmp_path / "ip-adapter_sd15.bin"), A.TINY_SD15)
    os.replace(tmp_path / "ip-adapter_sd15.bin", tmp_path / "ip-adapter_sd15.safetensors")   # a pickle under the right name
    with pytest.raises(ValueError, match="not a safetensors file"):
        I.load_adapter(str(tmp_path / "ip-adapter_sd15.safetensors"), A.TINY_SD15)


def _refusal(tmp_path, mutate, arch=A.TINY_SD15):
    sd = I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=64)
    mutate(sd)
    with pytest.raises(ValueError) as e:
        I.load_adapter(_save(sd, tmp_path / "a.safetensors"), arch)
    return str(e.value)


def test_loader_names_a_missing_to_v_ip(tmp_path):
    msg = _refusal(tmp_path, lambda sd: sd.pop("ip_adapter.7.to_v_ip.weight"))
    assert "missing 'ip_adapter.7.to_v_ip.weight'" in msg


def test_loader_names_a_wrong_shape(tmp_path):
    def mutate(sd):
        sd["ip_adapter.31.to_k_ip.weight"] = torch.zeros(3, 64, dtype=torch.float16)
    msg = _refusal(tmp_path, mutate)
    assert "'ip_adapter.31.to_k_ip.weight' has shape (3, 64)" in msg


def test_loader_names_a_wrong_cross_attention_dim(tmp_path):
    sd = I.synthetic_adapter_state_dict(A.SD15)                      # D = 768
    with pytest.raises(ValueError, match=r"'image_proj.norm.weight'.*cross_attention_dim is 768, the UNet's 1024"):
        I.load_adapter(_save(sd, tmp_path / "a.safetensors"), A.SD_TURBO)


def test_loader_names_a_wrong_number_of_cross_attentions(tmp_path):
    def mutate(sd):
        for w in ("to_k_ip", "to_v_ip"):
            sd.pop(f"ip_adapter.31.{w}.weight")
    assert "weights for 15 cross-attentions, the UNet (tiny-sd15) has 16" in _refusal(tmp_path, mutate)


# ---- mapping ------------------------------------------------------------------------------------------------------------------
def test_mapping_pinned_sd15_and_sd21_layouts():
    for arch in (A.SD15, A.SD_TURBO):
        m = I.adapter_key_map(arch)
        assert len(m) == 32 and sorted({int(k.split(".")[1]) for k in m}) == list(range(1, 32, 2))
        t = ".transformer_blocks.0.attn2.to_k_ip.weight"
        assert m["ip_adapter.1.to_k_ip.weight"] == "down_blocks.0.attentions.0" + t
        assert m["ip_adapter.3.to_k_ip.weight"] == "down_blocks.0.attentions.1" + t
        assert m["ip_adapter.11.to_k_ip.weight"] == "down_blocks.2.attentions.1" + t
        assert m["ip_adapter.13.to_k_ip.weight"] == "up_blocks.1.attentions.0" + t
        assert m["ip_adapter.29.to_v_ip.weight"] == "up_blocks.3.attentions.2.transformer_blocks.0.attn2.to_v_ip.weight"
        assert m["ip_adapter.31.to_k_ip.weight"] == "mid_block.attentions.0" + t, "the mid block is last"
        shapes = A.unet_param_shapes(arch)
        for unet_key in m.values():
            assert unet_key.replace("_ip.", ".") in shapes, "every target sits beside the UNet's own to_k / to_v"
    sh = I.adapter_shapes(A.SD15)
    assert sh["image_proj.proj.weight"] == (4 * 768, 1024) and sh["ip_adapter.1.to_k_ip.weight"] == (320, 768)
    assert sh["ip_adapter.31.to_v_ip.weight"] == (1280, 768)
    assert I.adapter_shapes(A.SD_TURBO)["ip_adapter.13.to_k_ip.weight"] == (1280, 1024)


# ---- oracle ---------------------------------------------------------------------------------------------------------------------
class _NnImageProj(nn.Module):
    def __init__(self, e, d, n):
        super().__init__()
        self.proj, self.norm, self.n, self.d = nn.Linear(e, n * d), nn.LayerNorm(d), n, d

    def forward(self, x):
        return self.norm(self.proj(x).reshape(-1, self.n, self.d))


class _NnDecoupledAttention(nn.Module):
    """Both softmaxes computed separately and summed, with nn.Linear projections and scaled_dot_product_attention"""

    def __init__(self, c, kv, heads):
        super().__init__()
        self.h = heads
        self.q, self.k, self.v = (nn.Linear(c, c, bias=False), nn.Linear(kv, c, bias=False), nn.Linear(kv, c, bias=False))
        self.k_ip, self.v_ip = nn.Linear(kv, c, bias=False), nn.Linear(kv, c, bias=False)
        self.out = nn.Linear(c, c)

    def forward(self, x, ctx, tok, scale):
        b, n, c = x.shape

        def split(t):
            return t.reshape(t.shape[0], -1, self.h, c // self.h).transpose(1, 2)
        q = split(self.q(x))
        txt = F.scaled_dot_product_attention(q, split(self.k(ctx)), split(self.v(ctx)))
        img = F.scaled_dot_product_attention(q, split(self.k_ip(tok)).expand(b, -1, -1, -1), split(self.v_ip(tok)).expand(b, -1, -1, -1))
        return self.out((txt + scale * img).transpose(1, 2).reshape(b, n, c))


def test_oracle_matches_an_independent_nn_build():
    from oracle import ip_adapter as OI
    from oracle import unet as OU
    text_only = OU.attention
    torch.manual_seed(0)
    e, d, n_tok, c, heads = 48, 32, 4, 40, 5
    proj = _NnImageProj(e, d, n_tok).double()
    with torch.no_grad():
        proj.norm.weight.normal_(1, 0.1)
        proj.norm.bias.normal_(0, 0.1)
    emb = torch.randn(1, e, dtype=torch.float64)
    got_tok = OI.image_proj(proj.proj.weight, proj.proj.bias, proj.norm.weight, proj.norm.bias, emb).double()
    ref_tok = proj(emb)
    assert (got_tok - ref_tok.float().double()).abs().max() < 1e-5
    attn = _NnDecoupledAttention(c, d, heads).double()
    p = "blk.attn2."
    sd = {p + "to_q.weight": attn.q.weight, p + "to_k.weight": attn.k.weight, p + "to_v.weight": attn.v.weight,
          p + "to_k_ip.weight": attn.k_ip.weight, p + "to_v_ip.weight": attn.v_ip.weight,
          p + "to_out.0.weight": attn.out.weight, p + "to_out.0.bias": attn.out.bias}
    sd = {k: v.detach() for k, v in sd.items()}
    x, ctx = torch.randn(3, 24, c, dtype=torch.float64), torch.randn(3, 7, d, dtype=torch.float64)
    tok = ref_tok.detach()
    with torch.no_grad():
        for scale in (0.0, 0.6, 1.0):
            ref = attn(x, ctx, tok, scale)
            got = OI.decoupled_attention(sd, p, heads, x, ctx, tok, scale)
            assert (got - ref).abs().max() < 1e-10, scale
            with OI.image_prompt(tok, scale):
                hooked = OU.attention(sd, p, heads, x, ctx)
            assert (hooked - ref).abs().max() < 1e-10
        # the hook leaves cross-attentions without IP weights (the ControlNet's) text-only, and is removed on exit
        plain = {k: v for k, v in sd.items() if "_ip" not in k}
        with OI.image_prompt(tok, 1.0):
            assert (OU.attention(plain, p, heads, x, ctx) - attn(x, ctx, tok, 0.0)).abs().max() < 1e-10
        assert OU.attention is text_only


# ---- blob recipe -------------------------------------------------------------------------------------------------------------
def test_blob_path_changes_with_the_adapter_file(tmp_path):
    from ai_rtc_agent_b200.host import weights as W
    sd = I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=64)
    path = _save(sd, tmp_path / "ip-adapter_sd15.safetensors")

    def blob(ip):
        return W.packed_blob_path(tmp_path, "tiny-sd15", "tiny-sd15", True, None, None, None, synthetic=True, ip_adapter=ip)
    a = blob(None)
    b = blob(path)
    assert blob(str(tmp_path)) != a and b != a
    sd["image_proj.proj.bias"] = sd["image_proj.proj.bias"] + 1
    _save(sd, path)
    os.utime(path, (1, 1))
    assert blob(path) != b, "a replaced adapter file must not hit the old blob"
    assert blob(None) == a, "without an adapter the recipe (and every existing blob name) is unchanged"


# ---- images ---------------------------------------------------------------------------------------------------------------------
def test_image_prompt_is_never_a_path(tmp_path):
    for bad in ("/etc/passwd", b"/etc/passwd", tmp_path):
        with pytest.raises(TypeError, match="not a path"):
            I.image_array(bad)
    with pytest.raises(TypeError):
        I.image_array(np.zeros((4, 4), dtype=np.uint8))
    arr = np.random.default_rng(0).integers(0, 255, (8, 6, 3), dtype=np.uint8)
    enc = I.SyntheticImageEncoder(16)
    assert torch.equal(enc(arr), enc(torch.from_numpy(arr))) and not torch.equal(enc(arr), enc(arr[::-1].copy()))


# ---- host routing over the recording fake of libb200sd ----------------------------------------------------------------------------
class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("b2sd_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name[5:],) + tuple(a.value if isinstance(a, ctypes.c_void_p) else a for a in args))
            return 0
        return call

    def named(self, name):
        return [c for c in self.calls if c[0] == name]


@pytest.fixture
def host(monkeypatch):
    from ai_rtc_agent_b200.host import stream as S
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder
    monkeypatch.setattr(S, "_on_device", lambda t, device: t.contiguous())
    monkeypatch.setattr(S, "_encode_beside", lambda eng, prompt: eng._encode(prompt)[0])
    lib = FakeLib()
    adapter = I.adapter_from_state_dict(I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=64), A.TINY_SD15)
    eng = object.__new__(S.StreamDiffusion)
    eng.__dict__.update(
        _lib=lib, _handle=ctypes.c_void_p(1), lanes=[], styles=[], _states=weakref.WeakSet(), _prepared=True, _ev=None,
        arch=types.SimpleNamespace(ctx_tokens=77, cross_attention_dim=64), prompt_encoder=SyntheticPromptEncoder(64),
        device=torch.device("cpu"), dtype=torch.float16, t_list=[20, 40], denoising_steps_num=2, batch_size=2, frame_bff_size=1,
        cfg_type="self", latent_height=2, latent_width=2, generator=None, ip_adapter=adapter)
    eng._stream = lambda: 0
    eng.prepare("global", guidance_scale=0.0)
    lane = object.__new__(S.StreamDiffusion)
    lane.__dict__.update(eng.__dict__, _handle=ctypes.c_void_p(2), lanes=[], styles=[])
    lane._stream = lambda: 0
    eng.lanes.append(lane)
    states = []

    def new_state():
        st = object.__new__(S.StreamState)
        st.__dict__.update(_engine=eng, _lib=lib, _handle=ctypes.c_void_p(100 + len(states)))
        states.append(st)
        eng._states.add(st)
        return st
    lib.calls.clear()
    return eng, new_state, lib


def test_global_image_prompt_reaches_the_family_and_resets_viewers(host):
    eng, new_state, lib = host
    a, b = new_state(), new_state()
    img = np.full((16, 16, 3), 7, dtype=np.uint8)
    a.set_prompt("a's prompt")
    a.set_image_tokens(eng.image_tokens(img), 0.5)
    b.set_image_tokens(eng.image_tokens(img[:8]), 0.8)
    lib.calls.clear()
    eng.set_image_tokens(eng.image_tokens(img), 0.7)
    sets = lib.named("set_image_embeds")
    assert [c[1] for c in sets] == [1, 2] and all(c[3] == 4 and c[4] == pytest.approx(0.7) for c in sets)
    assert a.own_image is None and b.own_image is None, "the global call resets every viewer's own image prompt"
    assert a.own_prompt == "a's prompt", "... and keeps their own prompts"
    assert [c[2] for c in lib.named("state_clear_conditioning")] == [0, 0]
    assert [c[2] for c in lib.named("state_set_prompt_embeds")] == [100], "a's own prompt is computed again"
    assert not lib.named("state_set_image_embeds")


def test_global_prompt_keeps_viewers_own_image_prompts(host):
    eng, new_state, lib = host
    a = new_state()
    tok = eng.image_tokens(np.zeros((4, 4, 3), dtype=np.uint8))
    a.set_image_tokens(tok, 0.9)
    lib.calls.clear()
    eng.update_prompt("new global")
    assert a.own_image is not None and a.own_prompt is None
    (c,) = lib.named("state_set_image_embeds")
    assert c[1:3] == (1, 100) and c[4] == 4 and c[5] == pytest.approx(0.9)


def test_none_clears(host):
    eng, new_state, lib = host
    a = new_state()
    a.set_prompt("own")
    a.set_image_tokens(eng.image_tokens(np.zeros((4, 4, 3), dtype=np.uint8)))
    lib.calls.clear()
    a.set_image_tokens(None)
    assert a.own_image is None and a.own_prompt == "own"
    assert [c[0] for c in lib.calls] == ["state_clear_conditioning", "state_set_prompt_embeds"]
    lib.calls.clear()
    eng.set_image_tokens(None)
    assert [c[1:4] for c in lib.named("set_image_embeds")] == [(1, None, 0), (2, None, 0)]
    assert eng.image_prompt is None


def test_pipeline_and_track_route_image_prompts_and_refuse_paths(monkeypatch):
    from ai_rtc_agent_b200.host import pipeline as P
    from ai_rtc_agent_b200.host import tracks as T
    log = []

    class Eng:
        def image_tokens(self, image):
            return ("tokens", I.image_array(image).shape)

        def set_image_tokens(self, tokens, scale):
            log.append(("global", tokens, scale))

    pipe = object.__new__(P.StreamDiffusionPipeline)
    pipe.model = types.SimpleNamespace(stream=Eng())
    pipe._quiesce = lambda: "cur"
    pipe._release = lambda cur: log.append(("release", cur))
    img = np.zeros((5, 7, 3), dtype=np.uint8)
    pipe.update_image_prompt(img, 0.3)
    pipe.update_image_prompt(None)
    assert log == [("global", ("tokens", (5, 7, 3)), 0.3), ("release", "cur"), ("global", None, 1.0), ("release", "cur")]
    with pytest.raises(TypeError, match="not a path"):
        pipe.update_image_prompt("/etc/passwd")
    assert len(log) == 4, "a refused image changes nothing"

    class Peer:
        def update_image_prompt(self, image, scale):
            log.append(("peer", image, scale))
    track = object.__new__(T.VideoStreamTrack)
    track.__dict__.update(_stopped=False, _per_peer=True, _peer=Peer(), pipeline=pipe)
    track.update_image_prompt(img, 0.5)
    assert log[-1] == ("peer", img, 0.5)


# ---- the CLIP vision encoder of a real adapter ------------------------------------------------------------------------------
def _tiny_clip(root, projection_dim=16):
    """a tiny CLIPVisionModelWithProjection + CLIPImageProcessor saved as <root>/image_encoder, as beside a real adapter"""
    from transformers import CLIPImageProcessor, CLIPVisionConfig, CLIPVisionModelWithProjection
    cfg = CLIPVisionConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=2, image_size=32,
                           patch_size=8, projection_dim=projection_dim)
    torch.manual_seed(0)
    d = os.path.join(str(root), "image_encoder")
    CLIPVisionModelWithProjection(cfg).save_pretrained(d)
    CLIPImageProcessor(size={"shortest_edge": 32}, crop_size={"height": 32, "width": 32}).save_pretrained(d)
    return d


def test_real_image_encoder_loads_beside_the_adapter(tmp_path):
    from transformers import CLIPImageProcessor, CLIPVisionModelWithProjection
    enc_dir = _tiny_clip(tmp_path)
    path = _save(I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=16), tmp_path / "ip-adapter_sd15.safetensors")
    img = np.random.default_rng(0).integers(0, 256, (40, 50, 3), dtype=np.uint8)
    for where in (str(tmp_path), path):   # the adapter directory, or the adapter file beside image_encoder/
        enc = I.make_image_encoder(where, 16, device="cpu")
        assert isinstance(enc, I.ClipImageEncoder)
        assert all(p.dtype == torch.float16 for p in enc.model.parameters()), "the encoder runs in fp16"
        got = enc(img)
        assert got.shape == (1, 16) and got.dtype == torch.float16
    # the same embedding from the saved model in fp32, within fp16 rounding
    ref_model = CLIPVisionModelWithProjection.from_pretrained(enc_dir).eval()
    px = CLIPImageProcessor.from_pretrained(enc_dir)(images=img, return_tensors="pt").pixel_values
    with torch.no_grad():
        ref = ref_model(px).image_embeds
    assert (got.float() - ref).abs().max() <= 2e-2 * ref.abs().max() + 1e-3
    ad = I.load_adapter(path, A.TINY_SD15)
    assert ad.tokens(got).shape == (1, I.IP_TOKENS, A.TINY_SD15.cross_attention_dim)
    with pytest.raises(ValueError, match="projection_dim 16, the adapter expects 1024"):
        I.make_image_encoder(str(tmp_path), 1024, device="cpu")


def test_real_adapter_without_an_encoder_is_refused(tmp_path):
    path = _save(I.synthetic_adapter_state_dict(A.TINY_SD15, embed_dim=16), tmp_path / "ip-adapter_sd15.safetensors")
    with pytest.raises(FileNotFoundError, match="no image_encoder/"):
        I.make_image_encoder(path, 16, device="cpu")
    assert isinstance(I.make_image_encoder(path, 16, device="cpu", allow_synthetic=True), I.SyntheticImageEncoder)
