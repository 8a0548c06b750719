"""The engine at the edges of the configuration space it accepts (stream batch 1 .. 16, sides 64 .. 1024): each configuration
launch-audited (every kernel launch of one frame and of the prompt / timestep refresh against a float64 recomputation,
tests/test_launch_audit_gpu.py) and then run for T + 2 frames through the stream loop against the oracle: the u8 image within
2 LSB and, for T > 1, the stream-batch latent buffer.  The CPU oracle checks tiny models up to 256 px, the fp32 GPU oracle
(oracle/torch_gpu.py) larger sizes and the full-size models.

The list is chosen by tests/test_config_space.py: each entry reaches a contraction, attention or stream-batch regime that no
other engine configuration reaches.  Each entry also checks that model: the regimes the audit records include every regime
the CPU model predicts for the configuration."""
from __future__ import annotations

import gc

import pytest
import torch

from tests import test_config_space as CS
from tests.test_engine_gpu import _cmp, _u8_check
from tests.test_launch_audit_gpu import _audit

pytestmark = pytest.mark.gpu


def _entry(turbo, t, hw, full=False):
    tl = [32] if t == 1 else [int(10 + 35 * i / (t - 1)) for i in range(t)]   # increasing t_index_list of T steps
    size = str(hw) if isinstance(hw, int) else f"{hw[0]}x{hw[1]}"
    name = f"{'' if full else 'tiny-'}{'turbo' if turbo else 'sd15'}-T{t}-{size}"
    return pytest.param(dict(turbo=turbo, tl=tl, hw=hw, full=full), id=name)


# Chosen by tests/test_config_space.py (each reaches a regime no other engine configuration reaches).  Full-size models where
# only their channel counts take the swapped orientation (K-heavy contractions of <= 64 pixels).
SWEEP = [
    _entry(True, 1, 64),                    # 1 x 1 deepest level: 1-token self-attention, GroupNorm over 1 pixel
    _entry(False, 4, 64),                   # four 1-pixel images: 1-token attention with V^T padded per image to 8 columns
    _entry(False, 5, (704, 320)),           # 11 x 5 level: 2 images per tile, the last one a phantom; V^T per image at 55 tokens
    _entry(False, 16, 128),                 # the largest stream batch
    _entry(True, 1, (128, 576)),            # 16-wide tiles with a partial last column tile, 8-wide tiles
    _entry(False, 3, (64, 320)),            # several images per 16- / 8-wide tile, phantom images
    _entry(False, 3, (64, 768)),
    _entry(False, 3, (192, 768)),
    _entry(False, 2, (704, 960)),           # 10560-token self-attention whose last KV tile reaches the next image
    _entry(False, 2, (64, 576), full=True),  # swapped orientation: 8 x 8 pixel tiles, partial in w and h
    _entry(True, 1, (64, 256), full=True),   # swapped: 16-wide pixel tiles, the 128-pixel row tile
    _entry(False, 2, (64, 1024), full=True),
    _entry(True, 1, (64, 768), full=True),
    _entry(True, 1, (768, 64), full=True),
]


def _release():
    gc.collect()
    torch.cuda.empty_cache()


def _stream_loop(cfg):
    """T + 2 frames through the stream loop of a fresh engine against the oracle (CPU for tiny models up to 256 px, fp32 GPU
    otherwise)"""
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import pipeline as opipe
    from oracle import stream as ostream
    from oracle import torch_gpu as tg
    from oracle import unet as ounet
    from oracle import weights as ow
    turbo, tl, hw, full = cfg["turbo"], cfg["tl"], cfg["hw"], cfg["full"]
    height, width = (hw, hw) if isinstance(hw, int) else hw
    if full:
        ucfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
    else:
        ucfg, arch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15)
    usd16, vsd16 = ow.make_unet_weights(ucfg), ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(ucfg.cross_attention_dim)
    sd = StreamDiffusion(arch, usd16, vsd16, tl, lambda p: emb, width=width, height=height, device="cuda")
    sd.prepare("p", guidance_scale=0.0)
    on_gpu = full or max(height, width) > 256
    if on_gpu:
        orc = tg.build(ucfg, usd16, vsd16, tl, height, emb, sd.init_noise, torch.float32, width=width)
    else:
        orc = ostream.StreamOracle(ow.to_float(usd16), ucfg, ow.to_float(vsd16), tl, width, height)
        orc.prepare(emb.float(), guidance_scale=0.0, init_noise=sd.init_noise.float())
    T = len(tl)
    for i in range(T + 2):
        frame = ow.make_frame(height, width, seed=40 + i)
        out = sd.step_u8(frame.cuda())
        with torch.no_grad():
            ref = opipe.frame_to_u8(orc, frame.cuda() if on_gpu else frame)
        _u8_check(out, ref, f"frame {i}")
        if T > 1:
            rows = []
            e, c = _cmp("buffer", sd.get_tensor("unet_in")[1:].cpu(), orc.x_t_latent_buffer.cpu(), rows)
            assert e <= 2e-2 and c >= 0.999, f"frame {i}: x_t_latent_buffer relerr {e:.3e} cos {c:.6f}"


@pytest.mark.parametrize("cfg", SWEEP)
def test_config_space_engine(cuda, request, cfg):
    name = request.node.callspec.id
    audit_cfg = {k: v for k, v in cfg.items() if k != "full"}
    aud = _audit(cuda, name, audit_cfg, full=cfg["full"])
    want = CS.engine_regimes(cfg, cfg["full"])
    got = {"contraction": {CS.contraction_regime(*t) for t in aud.tiles},
           "attention": {CS.attention_regime(nb, sq) for nb, sq in aud.self_attn},
           "batch": {CS.batch_regime(t) for t in aud.stream_batch}}
    print(f"{name}: " + "; ".join(f"{k} {sorted(v)}" for k, v in got.items()))
    for k in CS.ENGINE_CLASSES:
        assert want[k] <= got[k], f"{k} regimes predicted, never launched: {sorted(want[k] - got[k])}"
    _stream_loop(cfg)
    _release()
