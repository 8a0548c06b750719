"""CPU tests of the host side (no GPU): C-ABI surface, reference-shaped argument validation, schedule tables,
weight plumbing, frame-type handling, and the multi-process weight broadcast over gloo."""
import ctypes
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shared_library_exports_every_declared_symbol():
    from ai_rtc_agent_b200.host import capi
    lib = capi.lib()
    header = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    names = sorted(set(re.findall(r"\b(b2sd_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/b200sd.h but not exported by libb200sd.so"
    assert lib.b2sd_version() >= 1
    assert isinstance(lib.b2sd_last_error(), (bytes, type(None)))


def _ctypes_mirrors():
    """C struct name -> its ctypes mirror in host/capi.py"""
    from ai_rtc_agent_b200.host import capi
    return {"b2sd_act_view": capi.ActView, "b2sd_igemm_desc": capi.IgemmDesc, "b2sd_igemm_plan_info": capi.IgemmPlanInfo,
            "b2sd_attn_desc": capi.AttnDesc, "b2sd_config": capi.EngineConfig, "b2sd_groupnorm_args": capi.GroupNormArgs,
            "b2sd_layernorm_args": capi.LayerNormArgs, "b2sd_smallconv_args": capi.SmallConvArgs,
            "b2sd_upsample2x_args": capi.Upsample2xArgs, "b2sd_maxpool2x2_args": capi.MaxPool2x2Args,
            "b2sd_hed_project_args": capi.HedProjectArgs, "b2sd_hed_fuse_args": capi.HedFuseArgs,
            "b2sd_lcm_step_args": capi.LcmStepArgs, "b2sd_post_u8_args": capi.PostU8Args,
            "b2sd_small_linear_args": capi.SmallLinearArgs, "b2sd_timestep_embedding_args": capi.TimestepEmbeddingArgs,
            "b2sd_launch_record": capi.LaunchRecord}


def test_ctypes_struct_layout_matches_the_c_header(tmp_path):
    """Compile include/b200sd.h with gcc (plain C: the header must stay C-clean) and compare, for every struct it declares,
    sizeof() and the offsetof() of every field with the ctypes mirror: a mismatch makes the host read garbage descriptors."""
    import subprocess
    header = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    declared = re.findall(r"^typedef struct\s*\{.*?\}\s*(b2sd_[a-z0-9_]+)\s*;", header, re.M | re.S)
    mirrors = _ctypes_mirrors()
    assert len(declared) >= 17 and sorted(declared) == sorted(mirrors), "every struct of b200sd.h needs a ctypes mirror"
    lines, want = [], []
    for name, cls in mirrors.items():
        lines.append(f'printf("%zu\\n", sizeof({name}));')
        want.append((name, "sizeof", ctypes.sizeof(cls)))
        for field, _ in cls._fields_:
            lines.append(f'printf("%zu\\n", offsetof({name}, {field}));')
            want.append((name, field, getattr(cls, field).offset))
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sd.h"\nint main(void){\n' + "\n".join(lines) +
                   "\nreturn 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert len(got) == len(want)
    bad = [(n, f, c, g) for (n, f, c), g in zip(want, got) if c != g]
    assert not bad, "(struct, field, ctypes, C): " + repr(bad)


def test_no_cpu_fallback():
    """Without a GPU the product path must fail loudly, not fall back to the oracle."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ai_rtc_agent_b200.host import capi
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    with pytest.raises(capi.B2Error):
        StreamDiffusionWrapper("tiny-turbo", [10])
    src = ""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "ai-rtc-agent_b200")):
        for f in files:
            if f.endswith(".py"):
                src += open(os.path.join(dirpath, f)).read()
    for mod in ("lib/pipeline.py", "lib/wrapper.py"):
        src += open(os.path.join(ROOT, mod)).read()
    assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), "product code must never import the oracle"


def test_wrapper_validation_matches_reference_errors():
    from ai_rtc_agent_b200.host.wrapper import StreamDiffusionWrapper
    with pytest.raises(ValueError, match="txt2img mode accepts only cfg_type = 'none'"):   # lib/wrapper.py:135-139
        StreamDiffusionWrapper("m", [1], mode="txt2img")
    with pytest.raises(ValueError, match="frame_buffer_size > 1"):                          # lib/wrapper.py:140-144
        StreamDiffusionWrapper("m", [1], mode="txt2img", cfg_type="none", frame_buffer_size=2)
    with pytest.raises(NotImplementedError, match="img2img mode must use denoising batch"):  # lib/wrapper.py:146-150
        StreamDiffusionWrapper("m", [1], use_denoising_batch=False)
    with pytest.raises(NotImplementedError):
        StreamDiffusionWrapper("m", [1], use_safety_checker=True)
    with pytest.raises(FileNotFoundError):
        os.environ.pop("B200SD_SYNTHETIC_WEIGHTS", None)
        StreamDiffusionWrapper("no/such-model", [1])


def test_reference_import_surface():
    sys.path.insert(0, ROOT)
    import lib.pipeline as P
    import lib.wrapper as Wm
    assert P.DEFAULT_PROMPT == "fireworks in the night sky" and P.DEFAULT_T_INDEX_LIST == [18, 26, 35, 45]
    assert P.DEFAULT_NUM_INFERENCE_STEPS == 50 and P.DEFAULT_GUIDANCE_SCALE == 0.0
    for m in ("update_prompt", "update_t_index_list", "preprocess", "predict", "postprocess", "__call__"):
        assert callable(getattr(P.StreamDiffusionPipeline, m))
    for m in ("prepare", "img2img", "txt2img", "preprocess_image", "postprocess_image", "update_t_index_list", "__call__"):
        assert callable(getattr(Wm.StreamDiffusionWrapper, m))
    import inspect
    sig = inspect.signature(Wm.StreamDiffusionWrapper.__init__)
    ref_kwargs = ["model_id_or_path", "t_index_list", "controlnet_id_or_path", "controlnet_processor_id", "lora_dict", "mode",
                  "output_type", "lcm_lora_id", "vae_id", "device", "dtype", "frame_buffer_size", "width", "height", "warmup",
                  "acceleration", "do_add_noise", "device_ids", "use_lcm_lora", "use_tiny_vae", "enable_similar_image_filter",
                  "similar_image_filter_threshold", "similar_image_filter_max_skip_frame", "use_denoising_batch", "cfg_type",
                  "seed", "use_safety_checker", "engine_dir", "cuda_stream_handle"]
    assert list(sig.parameters)[1:] == ref_kwargs                       # lib/wrapper.py:35-66, same order
    d = {k: v.default for k, v in sig.parameters.items()}
    assert d["width"] == 512 and d["height"] == 512 and d["acceleration"] == "tensorrt" and d["cfg_type"] == "self"
    assert d["seed"] == 2 and d["engine_dir"] == "engines" and d["output_type"] == "pil" and d["warmup"] == 10
    assert Wm.CudaStreamPtr(1234).ptr == 1234


def test_invalid_frame_type_raises_like_reference():
    from ai_rtc_agent_b200.host.pipeline import StreamDiffusionPipeline
    p = StreamDiffusionPipeline.__new__(StreamDiffusionPipeline)
    p.device = "cuda"
    with pytest.raises(Exception, match="invalid frame type"):          # lib/pipeline.py:51-52
        p.preprocess("not a frame")
    with pytest.raises(Exception, match="invalid frame type"):
        p(torch.zeros(1, 8, 8, 3, dtype=torch.uint8))                   # CPU tensor is neither NVDEC nor av frame


def test_schedule_tables_agree_with_oracle():
    from ai_rtc_agent_b200.host import stream as hs
    from oracle import stream as ostream
    assert hs.lcm_timestep_table(50) == ostream.lcm_timesteps(50)
    assert hs.lcm_timestep_table(10) == ostream.lcm_timesteps(10)
    assert torch.equal(hs.scaled_linear_alphas_cumprod(), ostream.alphas_cumprod())
    for t in (99, 299, 479, 639, 999):
        a, b = hs.lcm_boundary_scalings(t), ostream.boundary_scalings(t)
        assert abs(a[0] - b[0]) < 1e-12 and abs(a[1] - b[1]) < 1e-12


def test_two_independent_parameter_inventories_agree():
    """host/arch.py and oracle/unet.py enumerate the checkpoint layout independently."""
    from ai_rtc_agent_b200.host import arch as A
    from oracle import taesd as otaesd
    from oracle import unet as ounet
    assert A.unet_param_shapes(A.SD15) == ounet.param_shapes(ounet.SD15)
    assert A.unet_param_shapes(A.SD_TURBO) == ounet.param_shapes(ounet.SD_TURBO)
    assert A.unet_param_shapes(A.TINY_TURBO) == ounet.param_shapes(ounet.tiny_config(True))
    assert A.unet_param_shapes(A.TINY_SD15) == ounet.param_shapes(ounet.tiny_config(False))
    assert A.taesd_param_shapes() == otaesd.param_shapes()
    assert A.arch_for("stabilityai/sd-turbo") is A.SD_TURBO and A.arch_for("lykon/dreamshaper-8") is A.SD15


def test_fuse_lora_math():
    from ai_rtc_agent_b200.host.weights import fuse_lora
    g = torch.Generator().manual_seed(0)
    w = torch.randn(8, 6, generator=g).half()
    down, up = torch.randn(2, 6, generator=g), torch.randn(8, 2, generator=g)
    sd = {"down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.weight": w.clone()}
    lora = {"unet.down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.lora_A.weight": down,
            "unet.down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.lora_B.weight": up,
            "unet.down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.alpha": torch.tensor(4.0)}
    assert fuse_lora(sd, lora, scale=0.5) == 1
    ref = (w.float() + 0.5 * (4.0 / 2) * (up @ down)).half()
    assert torch.equal(list(sd.values())[0], ref)


def test_synthetic_weights_are_seeded_and_scaled():
    from ai_rtc_agent_b200.host import arch as A
    s1 = A.synthetic_state_dict(A.unet_param_shapes(A.TINY_TURBO), seed=7)
    s2 = A.synthetic_state_dict(A.unet_param_shapes(A.TINY_TURBO), seed=7)
    assert all(torch.equal(s1[k], s2[k]) for k in s1)
    w = s1["down_blocks.0.resnets.0.conv1.weight"].float()
    assert abs(w.std().item() * (w[0].numel() ** 0.5) - 1.0) < 0.1
    A.validate_state_dict(s1, A.unet_param_shapes(A.TINY_TURBO), "tiny")
    with pytest.raises(ValueError):
        A.validate_state_dict({}, A.unet_param_shapes(A.TINY_TURBO), "empty")


def _bcast_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host import dist as bd
    bd.init(backend="gloo")
    shapes = A.taesd_param_shapes()
    sd = A.synthetic_state_dict(shapes, seed=11, relu_net=True) if rank == 0 else None
    out = bd.broadcast_state_dict(sd, shapes, torch.device("cpu"))
    digest = sum(float(v.float().abs().sum()) for v in out.values())
    q.put((rank, digest, len(out)))
    dist.barrier()
    dist.destroy_process_group()


def test_weight_broadcast_world_size_2_gloo():
    """N>1 path on CPU: rank 0 owns the weights, every rank ends with identical copies, one broadcast."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_bcast_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0][1] == res[1][1] and res[0][2] == res[1][2] > 50


def _write_tiny_checkpoint(root, with_lora=True):
    """A diffusers-layout checkpoint tree on disk (the files download.py:17-25 would fetch), tiny-width: unet/, TAESD repo,
    an LCM-LoRA in peft naming and a style LoRA in kohya naming."""
    import torch
    from safetensors.torch import save_file
    from ai_rtc_agent_b200.host import arch as A
    from oracle import unet as ounet
    from oracle import weights as ow
    # the oracle's generator (fan-in scaling with damped residual branches keeps fp16 error growth like a trained net's)
    unet = ow.make_unet_weights(ounet.tiny_config(False), seed=5)
    vae = ow.make_taesd_weights(seed=6)
    assert set(unet) == set(A.unet_param_shapes(A.TINY_SD15)) and set(vae) == set(A.taesd_param_shapes())
    model_dir = os.path.join(root, "tiny-sd15-ckpt")
    os.makedirs(os.path.join(model_dir, "unet"))
    save_file({k: v.contiguous() for k, v in unet.items()}, os.path.join(model_dir, "unet", "diffusion_pytorch_model.fp16.safetensors"))
    taesd_dir = os.path.join(root, "taesd")
    os.makedirs(taesd_dir)
    save_file({k: v.contiguous() for k, v in vae.items()}, os.path.join(taesd_dir, "diffusion_pytorch_model.safetensors"))
    g = torch.Generator().manual_seed(9)
    tq = "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q"
    ff = "mid_block.attentions.0.transformer_blocks.0.ff.net.2"
    lcm = {f"unet.{tq}.lora_A.weight": torch.randn(4, 64, generator=g).half(), f"unet.{tq}.lora_B.weight": torch.randn(64, 4, generator=g).half(),
           f"unet.{ff}.lora_A.weight": torch.randn(4, 1024, generator=g).half(), f"unet.{ff}.lora_B.weight": torch.randn(256, 4, generator=g).half()}
    lcm_dir = os.path.join(root, "lcm-lora")
    os.makedirs(lcm_dir)
    save_file(lcm, os.path.join(lcm_dir, "pytorch_lora_weights.safetensors"))
    kohya = "lora_unet_" + "up_blocks.3.resnets.0.conv1".replace(".", "_")
    style = {kohya + ".lora_down.weight": torch.randn(2, 192, 3, 3, generator=g).half(), kohya + ".lora_up.weight": torch.randn(64, 2, 1, 1, generator=g).half(),
             kohya + ".alpha": torch.tensor(1.0)}
    style_path = os.path.join(root, "style.safetensors")
    save_file(style, style_path)
    return model_dir, taesd_dir, lcm_dir, style_path, unet, vae, lcm, style


def test_checkpoint_on_disk_lora_fusing_end_to_end(tmp_path):
    """load_unet / load_taesd / fuse_lora (lib/wrapper.py:645-707) on a real directory tree: peft (`lora_A/B`) and kohya
    (`lora_unet_*`, alpha) key styles must land on the right parameters, with W += scale * alpha/rank * up @ down."""
    import torch
    from ai_rtc_agent_b200.host import weights as W
    model_dir, taesd_dir, lcm_dir, style_path, unet, vae, lcm, style = _write_tiny_checkpoint(str(tmp_path))
    arch, usd, vsd, repo = W.resolve_weights(model_dir, taesd_dir, lcm_dir, True, {style_path: 0.5}, sd_turbo=False)
    assert repo == model_dir and arch.name in ("sd15", "tiny-sd15")
    assert set(usd) == set(unet) and set(vsd) == set(vae)
    tq = "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.weight"
    want = unet[tq].float() + lcm["unet." + tq[:-7] + ".lora_B.weight"].float() @ lcm["unet." + tq[:-7] + ".lora_A.weight"].float()
    assert torch.allclose(usd[tq].float(), want.half().float(), atol=2e-3)
    ck = "up_blocks.3.resnets.0.conv1.weight"
    kohya = "lora_unet_" + ck[:-7].replace(".", "_")
    delta = (style[kohya + ".lora_up.weight"].float().flatten(1) @ style[kohya + ".lora_down.weight"].float().flatten(1)) * (0.5 * 1.0 / 2)
    assert torch.allclose(usd[ck].float(), (unet[ck].float() + delta.reshape(unet[ck].shape)).half().float(), atol=2e-3)
    untouched = "conv_in.weight"
    assert torch.equal(usd[untouched], unet[untouched])


def test_lora_that_does_not_apply_is_an_error(tmp_path):
    """A LoRA whose module names match nothing must not be skipped silently (an un-fused LCM-LoRA leaves SD-1.5
    un-distilled while it is run at 4 steps)."""
    import torch
    from ai_rtc_agent_b200.host.weights import fuse_lora
    sd = {"mid_block.resnets.0.conv1.weight": torch.zeros(8, 8, 3, 3, dtype=torch.float16)}
    bad = {"unet.some.other.module.lora_A.weight": torch.zeros(2, 8), "unet.some.other.module.lora_B.weight": torch.zeros(8, 2)}
    with pytest.raises(KeyError, match="matched 0 of 1"):
        fuse_lora(sd, bad)
    assert fuse_lora(sd, bad, strict=False) == 0
    te_only = {"lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": torch.zeros(2, 8),
               "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_up.weight": torch.zeros(8, 2)}
    with pytest.raises(KeyError):      # nothing for the UNet at all
        fuse_lora(sd, te_only)


def test_real_checkpoint_needs_its_text_encoder(tmp_path):
    """make_prompt_encoder: a checkpoint directory without a loadable text_encoder/ is an error, never a silent fallback
    to hash-seeded embeddings."""
    from ai_rtc_agent_b200.host.prompt import SyntheticPromptEncoder, make_prompt_encoder
    d = tmp_path / "ckpt"
    d.mkdir()
    with pytest.raises(FileNotFoundError):
        make_prompt_encoder(str(d), 768, "cpu")
    (d / "text_encoder").mkdir()
    with pytest.raises(Exception):     # present but not loadable
        make_prompt_encoder(str(d), 768, "cpu")
    assert isinstance(make_prompt_encoder(None, 768, "cpu"), SyntheticPromptEncoder)
    assert isinstance(make_prompt_encoder(str(tmp_path / "nope"), 768, "cpu", allow_synthetic=True), SyntheticPromptEncoder)


def test_packed_blob_path_follows_the_reference_cache_naming():
    from ai_rtc_agent_b200.host import weights as W
    a = W.packed_blob_path("./models/engines", "lykon/dreamshaper-8", "sd15", True, None, {"ghibli.safetensors": 1.0}, None, False)
    b = W.packed_blob_path("./models/engines", "lykon/dreamshaper-8", "sd15", True, None, {"ghibli.safetensors": 0.8}, None, False)
    c = W.packed_blob_path("./models/engines", "lykon/dreamshaper-8", "sd15", True, None, None, None, False)
    assert os.path.dirname(a) == os.path.join("./models/engines", "engines--lykon--dreamshaper-8")   # lib/wrapper.py:593
    assert a.endswith(".b2pack") and len({a, b, c}) == 3, "the LoRA recipe is part of the key"
    # batch / resolution do not change the blob, except stream batches whose attention levels have ragged token counts
    assert W.layout_variant(1, 512, 512) == W.layout_variant(4, 512, 512) == W.layout_variant(4, 768, 768) == ""
    assert W.layout_variant(4, 128, 128) == "ragged3" and W.layout_variant(1, 128, 128) == ""
    d = W.packed_blob_path("./e", "m", "sd15", True, None, None, None, False, variant=W.layout_variant(4, 128, 128))
    assert d != W.packed_blob_path("./e", "m", "sd15", True, None, None, None, False)


def test_pack_cli_argument_parsing():
    from ai_rtc_agent_b200 import pack
    assert pack.parse_lora(["a.safetensors:0.5", "/x/y.safetensors"]) == {"a.safetensors": 0.5, "/x/y.safetensors": 1.0}
    with pytest.raises(SystemExit):
        pack.parse_lora(["a.safetensors:fast"])


def _write_tiny_clip(model_dir, hidden=64):
    """text_encoder/ + tokenizer/ of a diffusers checkpoint (lib/wrapper.py:468-473 loads exactly these two sub-folders):
    a 2-layer CLIPTextModel with random weights and a character-level BPE vocabulary, saved with save_pretrained."""
    import json
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTokenizer
    vocab = {"<|startoftext|>": 0, "<|endoftext|>": 1}
    for c in "abcdefghijklmnopqrstuvwxyz":
        vocab[c] = len(vocab)
    for c in "abcdefghijklmnopqrstuvwxyz":
        vocab[c + "</w>"] = len(vocab)
    tok_dir, te_dir = os.path.join(model_dir, "tokenizer"), os.path.join(model_dir, "text_encoder")
    os.makedirs(tok_dir, exist_ok=True)
    json.dump(vocab, open(os.path.join(tok_dir, "vocab.json"), "w"))
    open(os.path.join(tok_dir, "merges.txt"), "w").write("#version: 0.2\n")
    CLIPTokenizer(os.path.join(tok_dir, "vocab.json"), os.path.join(tok_dir, "merges.txt"), model_max_length=77).save_pretrained(tok_dir)
    torch.manual_seed(3)
    cfg = CLIPTextConfig(vocab_size=len(vocab), hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=2,
                         num_attention_heads=2, max_position_embeddings=77, projection_dim=hidden, bos_token_id=0, eos_token_id=1,
                         pad_token_id=1)
    CLIPTextModel(cfg).save_pretrained(te_dir)


def test_clip_prompt_encoder_from_a_checkpoint_directory(tmp_path):
    """SURVEY 8f-4: the text encoder on the update path (lib/wrapper.py:468-473, lib/pipeline.py:44-45) -- tokenizer +
    CLIPTextModel from the checkpoint's sub-folders, (1,77,D) fp16 last_hidden_state, padded / truncated to 77 tokens."""
    from transformers import CLIPTextModel, CLIPTokenizer
    from ai_rtc_agent_b200.host.prompt import ClipPromptEncoder, make_prompt_encoder
    d = str(tmp_path / "ckpt")
    os.makedirs(d)
    _write_tiny_clip(d, hidden=64)
    enc = make_prompt_encoder(d, 64, "cpu")
    assert isinstance(enc, ClipPromptEncoder)
    a, b, a2 = enc("fireworks in the night sky"), enc("a cat"), enc("fireworks in the night sky")
    assert a.shape == (1, 77, 64) and a.dtype == torch.float16
    assert torch.equal(a, a2) and not torch.equal(a, b)
    long_prompt = enc("word " * 200)          # truncation to model_max_length
    assert long_prompt.shape == (1, 77, 64)
    tok = CLIPTokenizer.from_pretrained(os.path.join(d, "tokenizer"))
    ref = CLIPTextModel.from_pretrained(os.path.join(d, "text_encoder"))
    ids = tok("a cat", padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
    assert torch.allclose(b.float(), ref(ids)[0].float(), atol=2e-2)
    with pytest.raises(ValueError, match="hidden size"):
        make_prompt_encoder(d, 768, "cpu")    # encoder / UNet mismatch must not pass silently


def test_bench_helpers(tmp_path, monkeypatch):
    """bench.py's host-side helpers: NCCL log summary (what the multi-GPU line reports as evidence of the communicator), core
    count for the CPU arm (torchrun's OMP_NUM_THREADS=1 must not decide it), one config dict for every arm."""
    sys.path.insert(0, ROOT)
    import bench
    log = tmp_path / "nccl_n2_host_123.log"
    log.write_text("host:123:123 [0] NCCL INFO NCCL version 2.28.9+cuda12.9\n"
                   "host:123:456 [0] NCCL INFO Channel 00/0 : 0[0] -> 1[1] via P2P/CUMEM\n"
                   "host:123:456 [0] NCCL INFO comm 0x1 rank 0 nranks 2 cudaDev 0 nvmlDev 0 busId 1b000 commId 0x2 - Init COMPLETE\n")
    s = bench.nccl_log_summary(str(tmp_path / "nccl_n2_*_*.log"))
    assert s["init_complete_nranks"] == [2] and s["version"] == "2.28.9" and s["p2p_seen"] and not s["nvls_seen"]
    monkeypatch.setenv("OMP_NUM_THREADS", "1")
    assert 1 <= bench.physical_cores() <= (os.cpu_count() or 1)
    assert bench.bench_config(1)["workload"] == bench.bench_config(8)["workload"]
    assert set(bench.bench_config(1)) == set(bench.bench_config(8))
    assert bench.pin_to_gpu_numa_node(0) is None or "numa_node" in bench.pin_to_gpu_numa_node(0)
