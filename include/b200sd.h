/*
 * libb200sd -- C ABI of the B200-native per-frame img2img path.
 *
 * The reference (yondonfu/ai-rtc-agent) has no C/FFI boundary of its own: its drop-in boundary is
 * two Python classes (lib/pipeline.py:17-96 StreamDiffusionPipeline, lib/wrapper.py:34-407
 * StreamDiffusionWrapper) that reach the GPU through TensorRT engines built by the un-vendored
 * `streamdiffusion` package.  This header is what the Python shim in
 * ai-rtc-agent_b200/host/ binds with ctypes (see INTEGRATION.md); every entry point names the
 * reference call it stands in for.
 *
 * Conventions: plain pointers and sizes only (no torch types); all device pointers are CUDA device
 * memory of the current device; `stream` is a cudaStream_t passed as void*; every function returns 0
 * on success and non-zero on failure, with the message available from b2sd_last_error().
 * No function synchronises the device unless its comment says so.
 */
#ifndef B200SD_H
#define B200SD_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* b2sd_last_error(void);
int b2sd_version(void);

/* ------------------------------------------------------------------------------------------------
 * Operator level (the contractions inside the reference's unet.engine / vae_*.engine,
 * lib/wrapper.py:445-466): used by the parity tests and by the engine below.
 * ---------------------------------------------------------------------------------------------- */

/* NHWC fp16 view: element (n,h,w,c) at ptr[((n*H + h)*W + w)*ld + c] */
typedef struct {
    const void* ptr;
    int n, h, w, c;
    int ld;
} b2sd_act_view;

enum {
    B2SD_IG_RELU = 1,
    B2SD_IG_GEGLU = 2,
    B2SD_IG_SILU = 8,        /* x * sigmoid(x) after bias / residual (ControlNet conditioning embedding); single CTAs with
                                bn 16 / 32 / 64 / 128 only, not with B2SD_IG_TCONV or B2SD_IG_PAIR */
    B2SD_IG_PAD0 = 16,       /* 3x3 taps at input (stride*out + tap) instead of (stride*out + tap - 1): F.pad(x, (0,1,0,1)) then
                                an unpadded conv, the AutoencoderKL encoder's Downsample2D; single CTAs, bn 64 / 128 / 256, not
                                with B2SD_IG_TCONV, B2SD_IG_PAIR, B2SD_IG_SILU or swap */
    B2SD_IG_TCONV = 64,      /* run the persistent halo-tile kernel (stride-1 3x3, 64 -> 64 channels: the TAESD body) */
    B2SD_IG_PAIR = 128       /* CTA pairs: tcgen05.mma.cta_group::2 (M = 256 per MMA), each CTA stages half of the weight tile;
                                normal orientation, bn % 32 == 0, splits <= 4 */
};

/* conv3x3 / conv1x1 / Linear as one implicit GEMM:
 *   out[row][j] = acc_scale_b[b] * acc_scale * (sum_seg sum_tap sum_c src[seg](row, tap, c) * w[j][k] + colbias[b][j])
 *                 + res_scale * res[row][j]        (then ReLU / SiLU / GEGLU per flags)
 * K order of the packed weight rows = segments in sequence, each [tap][c]. */
typedef struct {
    b2sd_act_view src[3];
    int ntap[3];       /* 1 or 9 (3x3, pad 1) */
    int nseg;
    const void* w;     /* fp16 [w_rows][w_ld] */
    int w_rows, w_ld;
    int stride;        /* 1 or 2 */
    int nb, ho, wo;    /* output extents */
    int bn;            /* N tile, 0 = auto */
    int splits;        /* split-K factor (1, 2, 4 or 8 K slices reduced inside a thread-block cluster), <=1 = off */
    void* partial;     /* no workspace is needed (cluster split-K); optional int64 [ctas][8] debug timeline, else NULL */
    void* out;         /* fp16 [nb*ho*wo][ldc] */
    int ldc;
    const float* colbias;
    int colbias_bstride;
    const void* res;   /* fp16, indexed like out with pitch ldr */
    int ldr;
    float acc_scale, res_scale;
    int flags;
    int n_valid;       /* output channels */
    int swap;          /* 1: swapped orientation (output channels on the MMA M side, bn = 64/128/256 pixels on N) */
    /* LayerNorm without a LayerNorm launch (BasicTransformerBlock norm1/2/3), all optional (NULL / 0 = off):
     * rowstat_out  producer: also accumulate (sum, sum of squares) of every stored fp16 output row as 2^20 fixed point into
     *              uint64 [rows][2] with integer atomics (order independent => bit reproducible); caller zeroes it;
     * rowstat_in   consumer: those statistics for this GEMM's A rows; with colsum[n] = sum_k w[n][k] (w = W diag(gamma)) and
     *              colbias[n] = sum_k W[n][k] beta[k] + b[n] the epilogue computes rstd*(acc - mean*colsum) + colbias,
     *              i.e. LayerNorm(A) W^T + b, mean/var over ln_c columns with eps ln_eps;
     * out2         columns >= col2 are stored transposed, out2[(col - col2)*ld2 + row] (V^T block of a fused q/k/v projection). */
    void* rowstat_out;
    const void* rowstat_in;
    const float* colsum;
    int ln_c;
    float ln_eps;
    void* out2;
    int ld2, col2;
    /* acc_scale_b  optional fp32 [nb] in device memory, read when the kernel runs: a factor of batch item b's contraction term
     *              (NULL = 1).  Normal orientation (swap = 0), bn 16 / 32 / 64 / 128 / 160 / 256 (CTA pairs from 32), split-K
     *              (applied once, after the reduction); not with GEGLU, SiLU, tap origin 0, the LayerNorm fold or
     *              B2SD_IG_TCONV (the halo-tile kernel refuses it). */
    const float* acc_scale_b;
} b2sd_igemm_desc;

int b2sd_op_igemm(const b2sd_igemm_desc* d, void* stream);

/* Host-only planning (no GPU, no driver call): what b2sd_op_igemm (autotile = 0: the descriptor's bn / splits / swap / flags as
 * given) or the engine's tile policy (autotile = 1: latency policy of a single frame in flight; 2: throughput policy of >= 4
 * frames in flight; allow_swap = the contraction may use the swapped orientation) would launch for this contraction.  Pointers in the descriptor only need plausible alignment.  For tests of the host logic. */
typedef struct {
    int mode;          /* 0 = igemm_kernel on single CTAs, 1 = CTA pairs (2-CTA clusters); the halo-tile kernel is requested with B2SD_IG_TCONV */
    int swap, bn, splits;
    int grid_x, grid_y, grid_z;
    int num_stages;    /* operand ring depth */
    int acc_bufs;      /* 2 = persistent over M tiles (double-buffered TMEM accumulator) */
    int total_kb, kb_per_split;   /* K in 64-channel blocks, per cluster rank */
    int tmem_cols;
    int m_tiles;       /* 128-row output tiles */
    int64_t smem_bytes, rows_total;
    int tw, th, tn;    /* pixel tile: tn images x th rows x tw columns of the output (swapped orientation: the N-side tile) */
} b2sd_igemm_plan_info;
int b2sd_igemm_plan_dry(const b2sd_igemm_desc* d, int autotile, int allow_swap, b2sd_igemm_plan_info* out);

/* Host-only: launch shape of GroupNorm over [ca | cb] channels, hw pixels per image: cluster = CTAs per (image, group) of the
 * cluster kernel (0 = the non-cluster kernels: fused cooperative, or statistics + apply), threads per CTA of the cluster kernel,
 * pixels per CTA (cluster = 0: pixels per chunk of the non-cluster kernels). */
int b2sd_groupnorm_plan_dry(int ca, int cb, int groups, int hw, int* cluster, int* threads, int* pixels_per_cta);
uint64_t b2sd_igemm_partial_floats(int splits, int64_t rows_total, int n_valid);   /* legacy sizing helper, unused by the cluster split-K */

/* Flash attention (self / cross) of BasicTransformerBlock.attn1 / attn2 (inside unet.engine), and with dp = d_real = 512 the
 * single-head attention of the AutoencoderKL mid blocks (pitches, V^T batch stride multiples of 8, 16-byte aligned pointers).
 * q: [nb*sq][ldq], head h at columns [h*dp, (h+1)*dp); k likewise (batch b at row b*k_bstride, 0 = shared);
 * vt = V^T: [heads*dp][ldvt] with the key index contiguous (batch b at column b*vt_bstride);
 * out: [nb*sq][ldo], head h at columns [h*d_real, (h+1)*d_real). softmax scale = d_real^-0.5. */
typedef struct {
    const void* q; int ldq;
    const void* k; int ldk; int64_t k_bstride; int64_t k_rows;
    const void* vt; int ldvt; int64_t vt_bstride; int64_t vt_cols;
    void* out; int ldo;
    int nb, heads, sq, skv, d_real, dp;   /* dp: 64, 128, 192 (zero-padded heads) or 512 (d_real 512) */
} b2sd_attn_desc;
int b2sd_op_attention(const b2sd_attn_desc* d, void* stream);
/* The same (dp 64 / 128 / 192) with IP-Adapter's decoupled image segment, shared by every batch item:
 *   out = softmax(Q K^T / sqrt(d_real)) V + softmax(Q Kip^T / sqrt(d_real)) Vip
 * over the first *n_ip image keys (device int, 0..64, read by the kernel; 0 = b2sd_op_attention's result, bit for bit).
 * k_ip: [64][ldk] with k's head layout; vt_ip = Vip^T: [heads*dp][64]; both 16-byte aligned, whole 64-key blocks whose keys
 * past n_ip must be finite (zeroed).  A scale on the image term is folded into vt_ip. */
int b2sd_op_attention_ip(const b2sd_attn_desc* d, const void* k_ip, const void* vt_ip, const int* n_ip, void* stream);

/* GroupNorm(+SiLU) over the channel concatenation [xa | xb] (xb may be NULL), NHWC fp16.  y must not overlap xa or xb
 * (the statistics are centred on a value of x that other CTAs read after some have written y): refused. */
int b2sd_op_groupnorm(const void* xa, int ca, int lda, const void* xb, int cb, int ldb, const float* gamma,
                      const float* beta, void* y, int ldy, int nb, int hw, int groups, float eps, int silu,
                      void* stream);
/* Kernel path of the most recent GroupNorm launch issued on the calling thread: 0 = one thread-block cluster per
 * (image, group), 1 = cooperative single-launch kernel, 2 = statistics + apply launches, -1 = none yet. */
int b2sd_groupnorm_last_path(void);
int b2sd_op_layernorm(const void* x, int ldx, const float* gamma, const float* beta, void* y, int ldy,
                      int64_t rows, int c, float eps, void* stream);
int b2sd_op_upsample2x(const void* x, void* y, int nb, int h, int w, int c, void* stream);
/* direct 3x3 conv for Cin in {3,4}; flags: 1 = input is u8 NHWC scaled by 1/255 (lib/pipeline.py:61),
 * 2 = tanh(x/3)*3 on the input (DecoderTiny), 4 = ReLU on the output */
int b2sd_op_smallconv(const void* x, const void* w_oihw, const float* bias, void* y, int ldy, int nb, int h,
                      int w, int cin, int cout, int in_h, int in_w, int flags, void* stream);
/* Same, plus flag 32 = SiLU on the output, flag 64 = input on the 0..255 scale minus in_off[c] (device fp32 [3]; HED's first
 * conv, zero padding in the shifted domain), cout a multiple of 16 (columns cout..ldy-1 of y are not written), and an optional
 * fp16 NHWC residual added after the bias: item n at res + n * res_bstride (0 = one residual for every item), pitch ldr
 * (res 4-byte aligned, ldr and res_bstride even).  b2sd_op_smallconv is this with res = in_off = NULL. */
int b2sd_op_smallconv_ex(const void* x, const void* w_oihw, const float* bias, void* y, int ldy, int nb, int h, int w,
                         int cin, int cout, int in_h, int in_w, int flags, const void* res, int ldr, int64_t res_bstride,
                         const float* in_off, void* stream);
/* HED edge detector pieces: 2x2/2 max-pool (NHWC fp16, even h / w / c); per-pixel projection C -> 1 (fp32 weights [c],
 * bias [1], fp32 out [npix]); fusion of `levels` fp32 side outputs (maps[k] of hs[k] x ws[k]) into the u8 edge image
 * [h][w][3] (bilinear half-pixel upsampling, mean, sigmoid, * 255, truncation); edge_f16 (optional) gets the value as fp16. */
int b2sd_op_maxpool2x2(const void* x, void* y, int nb, int h, int w, int c, void* stream);
int b2sd_op_hed_project(const void* x, int ldx, int c, int64_t npix, const float* w, const float* bias, float* out, void* stream);
int b2sd_op_hed_fuse(const float* const* maps, const int* hs, const int* ws, int levels, int h, int w, void* out_u8,
                     void* edge_f16, void* stream);
/* StreamDiffusion scheduler_step_batch + stream-batch buffer update (see elementwise.cuh) */
int b2sd_op_lcm_step(void* x, const void* eps, const void* noise, const float* coef, void* out_latent, int T,
                     int hw, int do_add_noise, void* stream);
/* Codec boundary (SURVEY.md 8f-1; the reference's aiortc fork decodes with NVDEC / encodes with NVENC, requirements.txt:12-13,
 * and exchanges RGB tensors in HBM with lib/pipeline.py:50-51,83,96).  NV12 surface (Y plane + interleaved UV plane, pitches in
 * bytes) <-> the frame formats of b2sd_step: u8 NHWC RGB in, u8 NCHW RGB out.  flags: 0 = BT.709 limited range,
 * B2SD_CSC_BT601, B2SD_CSC_FULL_RANGE.  b2sd_codec_probe: bit 0 = libnvcuvid loadable, bit 1 = libnvidia-encode loadable. */
enum { B2SD_CSC_BT601 = 1, B2SD_CSC_FULL_RANGE = 2 };
int b2sd_op_nv12_to_rgb(const void* y, int y_pitch, const void* uv, int uv_pitch, void* rgb_nhwc, int h, int w, int flags, void* stream);
int b2sd_op_rgb_to_nv12(const void* rgb_nchw, void* y, int y_pitch, void* uv, int uv_pitch, int h, int w, int flags, void* stream);
int b2sd_codec_probe(void);
/* decoder tail + lib/pipeline.py:72-74 on the fp16 grid -> u8 NCHW */
int b2sd_op_post_u8(const void* y_nhwc, int ldy, void* out_nchw_u8, int nb, int h, int w, void* stream);
/* the float entry's tail: y * 2 - 1 in fp16 -> fp16 NCHW */
int b2sd_op_post_f16(const void* y_nhwc, int ldy, void* out_nchw_f16, int nb, int h, int w, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Engine level: one handle == one temporal stream (one StreamDiffusion instance, lib/wrapper.py:168).
 * Replaces StreamDiffusion + UNet2DConditionModelEngine + AutoencoderKLEngine
 * (lib/wrapper.py:445-466, 494-504) for mode="img2img", use_denoising_batch=True, frame_buffer_size=1,
 * cfg_type="self" with guidance_scale <= 1 (the only configuration lib/pipeline.py:23-42 builds).
 * ---------------------------------------------------------------------------------------------- */
typedef struct b2sd_engine* b2sd_handle;
#define B2SD_MAX_CONTROLNETS 4

typedef struct {
    int block_out_channels[4];   /* (320,640,1280,1280) */
    int heads[4];                /* SD-1.5: 8,8,8,8   SD-Turbo: 5,10,20,20 */
    int down_attn[4];            /* 1,1,1,0 */
    int cross_attention_dim;     /* 768 | 1024 */
    int layers_per_block;        /* 2 */
    int norm_groups;             /* 32 */
    int ctx_tokens;              /* 77 */
    int batch;                   /* len(t_index_list) * frame_buffer_size (lib/wrapper.py:159-163) */
    int height, width;           /* image size, multiples of 64 */
    int do_add_noise;            /* lib/wrapper.py:53 */
    int use_cuda_graph;          /* replay the frame program as one CUDA graph */
    int controlnet;              /* 1: a ControlNet (weights under "controlnet." + diffusers ControlNetModel keys) conditions
                                    every stream-batch slot on the current frame (control image = frame / 255 at the engine's
                                    size); its 12 + 1 residuals are added to the UNet's skips and mid-block output.  0: none.
                                    2..B2SD_MAX_CONTROLNETS: that many nets (control_processor_more).  A lane inherits its
                                    parent's value. */
    int control_processor;       /* with controlnet = 1: B2SD_CONTROL_FRAME (0), B2SD_CONTROL_HED (1): the control image is the
                                    HED edge map of the frame (controlnet_aux HEDdetector at the engine's size; weights under
                                    "hed." + ControlNetHED.pth keys, e.g. "hed.block1.convs.0.weight", "hed.norm"), or
                                    B2SD_CONTROL_CANNY (2): the Canny edge map of the frame (controlnet_aux CannyDetector,
                                    cv2.Canny with aperture 3 and the L1 gradient, at the engine's size; no weights; thresholds
                                    b2sd_set_canny_thresholds).  Inherited by lanes. */
    int vae;                     /* B2SD_VAE_TINY (0): TAESD (weights "vae." + AutoencoderTiny keys).  B2SD_VAE_KL (1): the model's
                                    own AutoencoderKL (weights "vae." + diffusers AutoencoderKL keys, e.g.
                                    "vae.encoder.down_blocks.0.resnets.0.conv1.weight", "vae.quant_conv.weight"; mid-block attention
                                    as to_q / to_k / to_v / to_out.0 with q/k/v as [512][512]); the latent is scaling_factor times the
                                    mean of the encoder's distribution (not a sample).  Inherited by lanes. */
    float vae_scaling_factor;    /* with vae = B2SD_VAE_KL: vae/config.json scaling_factor; 0 = 0.18215 */
    int ip_tokens;               /* IP-Adapter image prompts: 0 = off; else the most image tokens a prompt may have, 1..64.  The
                                    UNet's cross-attentions (not the ControlNet's) then add a decoupled attention over the image
                                    tokens' K / V (weights "...attn2.to_k_ip.weight" / "...attn2.to_v_ip.weight" beside to_k /
                                    to_v), see b2sd_set_image_embeds.  Inherited by lanes and styles. */
    int control_processor_more[B2SD_MAX_CONTROLNETS - 1];
                                 /* multi-ControlNet: controlnet = N (1..B2SD_MAX_CONTROLNETS) nets, net 0 with the weights and
                                    processor above, net i >= 1 with weights under "controlnet<i>." (e.g.
                                    "controlnet1.controlnet_mid_block.weight") and processor control_processor_more[i - 1]
                                    (0 for the entries past the last net).  The HED and Canny edge maps are each computed once
                                    per frame however many nets read them.  Each net's residuals are scaled by its own per-slot scales
                                    (b2sd_set_control_scales) and summed into the UNet's skips in net order,
                                    ((skip + r_0) + r_1) + ...  Inherited by lanes and styles. */
} b2sd_config;
enum { B2SD_CONTROL_FRAME = 0, B2SD_CONTROL_HED = 1, B2SD_CONTROL_CANNY = 2 };
enum { B2SD_VAE_TINY = 0, B2SD_VAE_KL = 1 };

int b2sd_create(const b2sd_config* cfg, b2sd_handle* out);
int b2sd_destroy(b2sd_handle h);
/* A "lane": a second engine over the SAME parameters as `parent` (one copy of the weights in HBM), with its own activations,
 * stream state and CUDA graph, so that several frames can be in flight on different CUDA streams.  cfg = NULL copies the
 * parent's; otherwise only batch / height / width may differ.  Prepare it like any engine (after the parent's first
 * b2sd_prepare, which lays the weights out).  With a 1-step stream batch (SD-Turbo) consecutive frames of ONE video stream are
 * independent, so alternating them over two lanes overlaps frame n+1 with frame n and yields bit-identical output; lanes are
 * also how several independent video streams share one GPU.  (The reference serialises everything behind a per-frame
 * torch.cuda.synchronize(), SURVEY.md 8 a-10.) */
int b2sd_create_lane(b2sd_handle parent, const b2sd_config* cfg, b2sd_handle* out);

/* Weights under diffusers state-dict names: UNet keys as-is ("down_blocks.0.resnets.0.conv1.weight"),
 * TAESD keys prefixed "vae." ("vae.encoder.layers.0.weight"), ControlNet keys prefixed "controlnet."
 * ("controlnet.controlnet_cond_embedding.conv_in.weight").  ptr may be host or device memory.
 * dtype: 0 = fp16, 1 = fp32.  Replaces the ONNX export + TensorRT build of lib/wrapper.py:785-910.
 * After the first b2sd_prepare the raw copies of parameters that only feed the packing kernels are released (set
 * B2_KEEP_RAW=1 to keep them); loading further tensors into such an engine is an error.  So is loading into a prepared
 * engine with live parameters (b2sd_set_live_params): b2sd_apply_lora changes those. */
int b2sd_load_tensor(b2sd_handle h, const char* key, const void* ptr, int dtype, const int64_t* shape, int ndim);

/* Live parameters: LoRAs switched on a running engine (b2sd_apply_lora).  on = 1 puts h's weight store in live mode; call it
 * before the store's first b2sd_prepare, on parameters loaded with b2sd_load_tensor.  Lanes share the store and so the mode.
 * The first prepare then keeps the loaded (base) UNet parameters: the raw copies of the pack-only ones are not released, and
 * every UNet matrix a kernel reads as loaded gets a second, base copy.  b2sd_import_packed refuses a live store (a blob does
 * not carry the base). */
int b2sd_set_live_params(b2sd_handle h, int on);
/* One LoRA pair on one UNet matrix: delta = scale * up @ down, with up [rows][rank] and down [rank][cols] in DEVICE memory,
 * rows = the parameter's first dimension and cols = the product of the others (Cin * kh * kw for a convolution, as
 * W.flatten(1)).  scale is the LoRA's scale times alpha / rank. */
typedef struct b2sd_lora_factor {
    const char* key;      /* the parameter, e.g. "up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k.weight" */
    const void* up;
    const void* down;
    int rank;
    int dtype;            /* of both factors: 0 = fp16, 1 = fp32 */
    float scale;
} b2sd_lora_factor;
/* Re-fuse the live UNet parameters of h's weight store: every key of f becomes base + the deltas of its factors, in the given
 * order, rounded to fp16 after each (as fusing LoRAs one after another on the host does); every other parameter reverts to its
 * base value, which is never written (n = 0: the base weights).  The deltas run on the tensor cores; every packed and fp32
 * entry derived from a changed parameter is rebuilt in place, so addresses, frame programs and CUDA graphs stay valid.  All of
 * it is enqueued on `stream` without a host synchronisation: the caller orders it after the frames in flight on the store's
 * engines and before later ones, keeps the factors alive until it has run, and then refreshes each engine's conditioning
 * (b2sd_refresh_conditioning) and each state's own (b2sd_state_set_*).  Arguments are checked before any device work.  A store
 * scratch holds the factor operands and fused matrices; it grows only when a call needs more than any before it. */
int b2sd_apply_lora(b2sd_handle h, int n, const b2sd_lora_factor* f, void* stream);
/* Recompute h's global prompt and time blocks (cross-attention K / V^T, time embeddings, resnet time biases) from its global
 * prompt embeddings and timesteps with the current parameters, on `stream`, without a host synchronisation */
int b2sd_refresh_conditioning(b2sd_handle h, void* stream);

/* Styles: one engine's UNet with its own LoRAs beside the parent's, sharing everything a UNet LoRA does not reach.
 * b2sd_create_style makes an engine over a new weight store derived from parent's, which must be live and prepared
 * (b2sd_set_live_params before its first b2sd_prepare).  The style reads the parent's base parameters in place (they are never
 * written) and keeps the parent's store alive; it owns copies of the UNet matrices kernels read as loaded and the packed /
 * fp32 entries derived from UNet matrices, and shares by pointer the VAE, ControlNet, HED and every other entry.  It has the
 * parent's configuration and concurrency.  Prepare it and its lanes (b2sd_create_lane(style, ...)) like any engine, before its
 * first b2sd_apply_lora, which then fuses LoRAs relative to the shared base.  A store and the styles derived from it form a
 * family: a state of any of them may be stepped by an engine of any other (same batch and size), but a state's own prompt /
 * timesteps are bound only on engines of the store they were computed on (set them again after a move).
 * The style's memory is allocated and freed stream-ordered, from a pool of its own that never makes an allocation wait for a
 * free on another stream, on a stream of its own: nothing about it synchronises the device or waits for other engines' work.
 * Free its engines with b2sd_release(h, stream), whose frees run after the work queued on `stream` at the call (make it wait
 * for the last frames of every engine of the style first); the store goes with its last engine. */
int b2sd_create_style(b2sd_handle parent, b2sd_handle* out);
int b2sd_release(b2sd_handle h, void* stream);

/* Packed-weight blob: the kernel-native layouts b2sd_prepare derives from the parameters (reordered convolution
 * matrices, per-head q/k/v gathers, GEGLU interleave, fused bias vectors), written once and loaded instead of
 * b2sd_load_tensor + repacking.  Replaces the reference's cached TensorRT engine files `engines--<model>/...engine`
 * (lib/wrapper.py:593-597, 896-910; build.py:11-32).  The blob depends on the architecture and the (LoRA-fused)
 * parameter values only -- not on batch, image size or prompt.  Export after b2sd_prepare; import into a fresh engine
 * (same b2sd_config architecture fields) before b2sd_prepare.  Host synchronous. */
int b2sd_export_packed(b2sd_handle h, const char* path);
int b2sd_import_packed(b2sd_handle h, const char* path);

/* StreamDiffusion.prepare (via lib/wrapper.py:197-234): fixes per-slot scalars and noise, zeroes the
 * stream-batch latent buffer, builds the frame program.  All pointers are HOST memory:
 *   prompt_embeds  fp16 [ctx_tokens][cross_attention_dim]   (CLIP output, encoded by the caller)
 *   timesteps      fp32 [batch]                             (sub_timesteps_tensor)
 *   coef           fp32 [4][batch] = alpha_prod_t_sqrt, beta_prod_t_sqrt, c_skip, c_out
 *   init_noise     fp16 [batch][4][h/8][w/8]                (NCHW, as torch.randn produced it)
 * Synchronises `stream`. */
int b2sd_prepare(b2sd_handle h, const void* prompt_embeds, const float* timesteps, const float* coef,
                 const void* init_noise, void* stream);
/* StreamDiffusion.update_prompt (lib/pipeline.py:44-45): refresh the per-layer cross-attention K/V cache (the engine's global
 * prompt block, see b2sd_state_set_prompt_embeds) */
int b2sd_set_prompt_embeds(b2sd_handle h, const void* prompt_embeds, void* stream);
/* lib/wrapper.py:389-407 update_t_index_list: only sub_timesteps change (alpha/beta/c_skip/c_out keep the
 * values given to b2sd_prepare -- reference behaviour); refreshes the engine's global time block */
int b2sd_set_timesteps(b2sd_handle h, const float* timesteps, void* stream);

/* One StreamDiffusionPipeline.__call__ (lib/pipeline.py:76-96, NVENC branch): frame_in = device u8 NHWC
 * [in_h][in_w][3] (nearest-resized to height x width if different, SURVEY a-4), frame_out = device u8 NCHW
 * [3][height][width].  Enqueues on `stream`; no host synchronisation. */
int b2sd_step(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, void* stream);

/* Same, for the reference's split call path preprocess -> predict -> postprocess (lib/pipeline.py:50-74):
 * input may be the (3,H,W) float tensor lib/pipeline.py:65 produces; output may be the fp16 NCHW image
 * in [-1,1] that StreamDiffusion.__call__ returns (lib/wrapper.py:330). */
enum { B2SD_IN_U8_NHWC = 0, B2SD_IN_F32_NCHW = 1, B2SD_IN_F16_NCHW = 2 };
enum { B2SD_OUT_U8_NCHW = 0, B2SD_OUT_F16_NCHW = 1 };
int b2sd_step_ex(b2sd_handle h, const void* frame_in, int in_kind, int in_h, int in_w, void* frame_out,
                 int out_kind, void* stream);

/* Parity/debug taps: copies a named intermediate of the last step to host memory as fp16 NHWC.
 * Names: "x_t", "unet_in", "eps", "x0", "image", "conv_in", "down.I.J", "mid", "up.I.J"; with the AutoencoderKL also
 * "vae.enc.down.I", "vae.enc.mid", "vae.dec.mid", "vae.dec.up.I" (block outputs); with a ControlNet also "cn_cond"
 * (conditioning embedding, batch 1), "cn.conv_in" (its conv_in(x) + cn_cond), "cn.res.K" (UNet skip K, in push order 0..11,
 * plus ControlNet residual K: what the up path reads) and "cn.mid" ("mid" plus the mid-block residual); with HED also
 * "control" (the u8 edge value as fp16, [1][h][w][1]); with Canny also "canny" (the u8 edge image, [1][h][w][3], 0 / 255) and
 * "canny_class" (canny_head's class map, [1][h][w][1]: 0 none, 1 candidate, 2 strong), both as fp16.
 * Returns the element count via *count (pass dst = NULL to query).  Synchronises `stream`. */
int b2sd_get_tensor(b2sd_handle h, const char* name, void* dst, int64_t capacity, int64_t* count, int* dims4,
                    void* stream);
/* Profiling aid: eager replay of one frame with a CUDA event after every launch, averaged over `iters`;
 * writes a JSON array [{"name","ms"},...] to json_buf.  Synchronises. */
int b2sd_profile(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, int iters,
                 char* json_buf, int64_t cap, void* stream);
/* Device time of one launch class ("igemm", "attn", "groupnorm", "layernorm", ...) of the frame program, measured by
 * replaying a CUDA graph that holds only those launches (same order, buffers and weight streaming as the frame graph).
 * ms_per_replay = average over `iters` replays; launches / flops (optional) = launches and algorithmic FLOPs per replay. */
int b2sd_profile_kind(b2sd_handle h, const char* kind, int iters, double* ms_per_replay, int* launches, double* flops,
                      void* stream);
/* number of kernel launches (graph nodes) in one b2sd_step */
/* Concurrent use of b2sd_profile_kind (one host thread and CUDA stream per lane): after b2sd_profile_gate(n) the next n calls
 * wait for each other between their warm-up and their timed replays, so the timed regions overlap.  0 / 1 switches it off. */
int b2sd_profile_gate(int participants);
int b2sd_launches_per_step(b2sd_handle h);

/* Launch audit (test aid, like b2sd_profile): what each launch of the frame program computes, as it is launched.
 * kind B2SD_LAUNCH_IGEMM / _TCONV: `igemm` is the contraction with the plan's bn / splits / swap and B2SD_IG_PAIR /
 * B2SD_IG_TCONV in flags (partial = NULL), `plan` the plan (for the halo-tile kernel only bn 64, splits 1 and rows_total);
 * _ATTN: `attn`; _GROUPNORM / _LAYERNORM: the normalisation's arguments; every other kind: its launcher's arguments in the
 * member of the same name (smallconv, upsample2x, ...).  _OTHER: only `label` (the profiling label), the kind of a record that
 * nobody filled: both audit entry points fill every launch they issue. */
enum { B2SD_LAUNCH_OTHER = 0, B2SD_LAUNCH_IGEMM = 1, B2SD_LAUNCH_TCONV = 2, B2SD_LAUNCH_ATTN = 3, B2SD_LAUNCH_GROUPNORM = 4,
       B2SD_LAUNCH_LAYERNORM = 5, B2SD_LAUNCH_SMALLCONV = 6, B2SD_LAUNCH_UPSAMPLE2X = 7, B2SD_LAUNCH_MAXPOOL2X2 = 8,
       B2SD_LAUNCH_HED_PROJECT = 9, B2SD_LAUNCH_HED_FUSE = 10, B2SD_LAUNCH_LCM_STEP = 11, B2SD_LAUNCH_POST_U8 = 12,
       B2SD_LAUNCH_SMALL_LINEAR = 13, B2SD_LAUNCH_TIMESTEP_EMBEDDING = 14, B2SD_LAUNCH_CANNY_HEAD = 15,
       B2SD_LAUNCH_CANNY_CCL = 16 };
typedef struct {
    const void* xa; int ca, lda;
    const void* xb; int cb, ldb;   /* xb NULL: no second source */
    const float* gamma; const float* beta;
    void* y; int ldy;
    int nb, hw, groups;
    float eps;
    int silu;
} b2sd_groupnorm_args;
typedef struct {
    const void* x; int ldx;
    const float* gamma; const float* beta;
    void* y; int ldy;
    int64_t rows; int c;
    float eps;
} b2sd_layernorm_args;
/* direct 3x3 conv (b2sd_op_smallconv_ex): x read per flags (1 u8 NHWC / 255, 8 fp32 NCHW, 16 fp16 NCHW, else fp16 NHWC; 2 =
 * tanh(x/3)*3; 64 = u8 or NCHW value on the 0..255 scale minus in_off[c]), nearest-resized from in_h x in_w to h x w, rounded to
 * fp16, convolved with wt = fp32 [cin*9][cout] (k = tap*cin + c, pad 1), + bias, + res (item n at res + n*res_bstride, pitch
 * ldr), then 4 = ReLU / 32 = SiLU; fp16 out, columns [cout, ldy) untouched */
typedef struct {
    const void* x; const float* wt; const float* bias;
    void* y; int ldy;
    int nb, h, w, cin, cout, in_h, in_w, flags;
    const void* res; int ldr; int64_t res_bstride;
    const float* in_off;
} b2sd_smallconv_args;
/* nearest x2 upsampling, NHWC fp16 [nb][h][w][c] -> [nb][2h][2w][c] (both dense) */
typedef struct { const void* x; void* y; int nb, h, w, c; } b2sd_upsample2x_args;
/* 2x2 / 2 max-pool, NHWC fp16 [nb][h][w][c] -> [nb][h/2][w/2][c] (both dense) */
typedef struct { const void* x; void* y; int nb, h, w, c; } b2sd_maxpool2x2_args;
/* out[p] = bias[0] + sum_c x[p*ldx + c] * w[c], fp32 out [npix] */
typedef struct { const void* x; int ldx, c; int64_t npix; const float* w; const float* bias; float* out; } b2sd_hed_project_args;
/* see b2sd_op_hed_fuse */
typedef struct {
    const float* maps[5]; int hs[5], ws[5];
    int levels, h, w;
    void* out; void* edge_f16;
} b2sd_hed_fuse_args;
/* see b2sd_op_lcm_step: x (rewritten in place: slots 1..T-1) and eps fp16 [T][hw][4], coef fp32 [4][T] */
typedef struct {
    void* x; const void* eps; const void* noise; const float* coef; void* out_latent;
    int T, hw, do_add_noise;
} b2sd_lcm_step_args;
/* see b2sd_op_post_u8 */
typedef struct { const void* y; int ldy; void* out; int nb, h, w; } b2sd_post_u8_args;
/* out[b*out_ld + j] = bias[j] + sum_i act(in[b*in_ld + i]) * w[j*k + i] (w fp16 [n][k], act = SiLU when silu_in), b < nb */
typedef struct {
    const float* in; int in_ld;
    const void* w; const float* bias;
    float* out; int out_ld;
    int nb, n, k, silu_in;
} b2sd_small_linear_args;
/* out[b] = [cos | sin](t[b] * exp(-ln(10000) * j / (dim/2))), j < dim/2: fp32 [nb][dim] */
typedef struct { const float* t; float* out; int nb, dim; } b2sd_timestep_embedding_args;
/* Canny's input head: the frame x (in_flags 1 u8 NHWC, 8 fp32 NCHW, 16 fp16 NCHW, nearest-resized from in_h x in_w to h x w,
 * floats as rint(clamp(v, 0, 1) * 255)) classified per pixel into cls u8 [h][w] (0 none, 1 candidate, 2 strong) with the
 * integer thresholds low / high (swapped when reversed, floored, clamped to [-1, 2041]) */
typedef struct b2sd_canny_head_args { const void* x; int in_flags, in_h, in_w, h, w, low, high; void* cls; } b2sd_canny_head_args;
/* Canny's hysteresis, stage 0..3 (local labels, border merges, root flags, output): cls [h][w] -> out u8 [h][w][3], with the
 * scratch parent int [h][w] and flag u8 [h][w] */
typedef struct b2sd_canny_ccl_args { const void* cls; void* parent; void* flag; void* out; int h, w, stage; } b2sd_canny_ccl_args;
typedef struct {
    int kind;
    const char* label;
    b2sd_igemm_desc igemm;
    b2sd_igemm_plan_info plan;
    b2sd_attn_desc attn;
    b2sd_groupnorm_args groupnorm;
    b2sd_layernorm_args layernorm;
    b2sd_smallconv_args smallconv;
    b2sd_upsample2x_args upsample2x;
    b2sd_maxpool2x2_args maxpool2x2;
    b2sd_hed_project_args hed_project;
    b2sd_hed_fuse_args hed_fuse;
    b2sd_lcm_step_args lcm_step;
    b2sd_post_u8_args post_u8;
    b2sd_small_linear_args small_linear;
    b2sd_timestep_embedding_args timestep_embedding;
    /* _ATTN with IP-Adapter's image segment: b2sd_op_attention_ip's k_ip, vt_ip and n_ip (device memory); NULL otherwise */
    const void* attn_k_ip;
    const void* attn_vt_ip;
    const int* attn_n_ip;
    b2sd_canny_head_args canny_head;
    b2sd_canny_ccl_args canny_ccl;
} b2sd_launch_record;
/* One b2sd_step with the frame program run eagerly (no CUDA graph) and `fn` called around every kernel launch: `stream` is
 * synchronised, fn(user, index, 0, rec) runs, the launch is enqueued, `stream` is synchronised, fn(user, index, 1, rec) runs.
 * index counts kernel launches (0 .. b2sd_launches_per_step - 1, in launch order, the frame's input heads first and the u8
 * tail last); the frame program's memset of the LayerNorm statistics is not a kernel launch and gets no call.  A non-zero
 * return from fn aborts the step with an error.  The output equals b2sd_step's. */
typedef int (*b2sd_audit_fn)(void* user, int index, int after, const b2sd_launch_record* rec);
int b2sd_audit_step(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, b2sd_audit_fn fn, void* user,
                    void* stream);
/* The prompt / timestep refresh of b2sd_prepare (the cross-attention K / V^T projections of the current prompt, then the
 * timestep embedding, the time MLPs and every resnet's per-slot time bias) run eagerly with the same callback protocol as
 * b2sd_audit_step; index counts the refresh's kernel launches.  It recomputes what b2sd_prepare computed from the same inputs. */
int b2sd_audit_refresh(b2sd_handle h, b2sd_audit_fn fn, void* user, void* stream);

/* Stream states: the stream-batch state of one temporal stream (x_t_latent_buffer, slots 1 .. T-1 of the UNet input batch,
 * (T-1) * (h/8) * (w/8) * 4 fp16 values; nothing at T = 1) kept apart from the engines that step it.  Any engine of the
 * state's weight store with the state's batch and size can step it, so several video streams (one state each) share a pool
 * of lanes: frames of different states overlap completely, and consecutive frames of one state are stage-pipelined across
 * lanes -- the frame program is cut into encoder body | last encoder conv + UNet + scheduler step | decoder, and only the
 * middle stage is serialised per state, so the encoder of frame n+1 and the decoder of frame n-1 overlap the UNet of frame n.
 * This is how one stateful stream (T > 1, where frame n+1 needs frame n's latent buffer) runs on several lanes: step one
 * state on each in turn.  A state carries one CUDA event that orders its steps; submit the frames of one state in order from
 * one host thread. */
typedef struct b2sd_state* b2sd_state_handle;
/* a zeroed state sized for h's batch and size (h prepared); allocated stream-ordered on `stream` */
int b2sd_state_create(b2sd_handle h, b2sd_state_handle* out, void* stream);
/* zero the state (what b2sd_prepare does to an engine's own latent buffer), after its last step, on `stream` */
int b2sd_state_reset(b2sd_state_handle state, void* stream);
/* free the state (and its conditioning overrides) on `stream` after its last step, without a host synchronisation; NULL is a
 * no-op */
int b2sd_state_destroy(b2sd_state_handle state, void* stream);
/* b2sd_step_ex on `state`: input heads, encoder body | wait for the state's previous step, copy the state into slots 1 .. T-1,
 * latent conv + UNet (+ ControlNet) + scheduler step, copy slots 1 .. T-1 back, record the state's event | decoder, tail.
 * At T = 1 the state is empty and this is b2sd_step_ex. */
int b2sd_step_state(b2sd_handle h, b2sd_state_handle state, const void* frame_in, int in_kind, int in_h, int in_w,
                    void* frame_out, int out_kind, void* stream);

/* Per-state conditioning: a state may carry its own prompt and its own timesteps, so each viewer of a lane pool sees its own
 * prompt and t_index_list.  An engine keeps what its frame program reads of the conditioning in two contiguous blocks: the
 * prompt block (every cross-attention K / V^T cache, UNet and ControlNet) and the time block (every resnet's per-slot time
 * bias).  A state's override of a block is a device copy of it computed for that state.  Before the UNet stage of a step, each
 * block is made to hold what the state is stepped with -- its override, or the engine's global values (b2sd_prepare /
 * b2sd_set_prompt_embeds / b2sd_set_timesteps) -- with one device-to-device copy when it holds something else; so lanes whose
 * states never override copy nothing.  b2sd_step_ex and the other calls without a state use the global values.
 * An override is immutable: an update makes a new one, and the one it replaces is freed after the last step that copies it.
 * The calls refuse what b2sd_step_state refuses (null handles, a state of another store / batch / size, an unprepared
 * engine).  A state's bookkeeping is host state without a lock: calls that take one state (b2sd_step_state and the three
 * below) must not run concurrently, from whichever engine or thread; calls on different states may.  The overrides of a weight store's states share a memory pool that keeps a few blocks' worth of
 * memory across synchronisations; it is released when the last engine of the store and the last override are gone. */
/* Compute `state`'s prompt block from embeddings in DEVICE memory, fp16 [ctx_tokens][cross_attention_dim], on engine h (any
 * engine that may step the state), stream-ordered on `stream` after the frames queued there, without a host synchronisation.
 * Steps of the state submitted after this call use it, on any engine. */
int b2sd_state_set_prompt_embeds(b2sd_handle h, b2sd_state_handle state, const void* prompt_embeds, void* stream);
/* The same for the time block from the state's per-slot timesteps in DEVICE memory, fp32 [batch]; as b2sd_set_timesteps, only
 * the time embedding changes (alpha / beta / c_skip / c_out keep their b2sd_prepare values). */
int b2sd_state_set_timesteps(b2sd_handle h, b2sd_state_handle state, const float* timesteps, void* stream);
/* IP-Adapter image prompt (an engine with ip_tokens > 0), shared by the frame's cross-attentions like the prompt:
 * tokens_f16 fp16 [n_tok][cross_attention_dim] (host or device memory, 1 <= n_tok <= ip_tokens; NULL clears the image prompt),
 * scale (finite) multiplies the image attention term (folded into the image V^T).  b2sd_set_image_embeds refreshes the engine's
 * global prompt block, as b2sd_set_prompt_embeds does; b2sd_state_set_image_embeds computes the state's prompt block (its own
 * prompt if it has one computed on h's weight store, else the engine's) with this image prompt, as
 * b2sd_state_set_prompt_embeds does (tokens in DEVICE memory, stream-ordered, no host synchronisation), and
 * b2sd_state_set_prompt_embeds keeps the state's image prompt likewise.  A state's image prompt without a prompt of its own
 * takes the text part from the engine's global block at the call, so a global refresh (b2sd_set_prompt_embeds,
 * b2sd_refresh_conditioning) is followed by setting the state's image prompt again, as its own prompt is.  After a move to another store of the family set the
 * state's prompt, then its image prompt, again.  Clearing the state's prompt block (b2sd_state_clear_conditioning(state, 0))
 * drops both.  Neither call recaptures a CUDA graph. */
int b2sd_set_image_embeds(b2sd_handle h, const void* tokens_f16, int n_tok, float scale, void* stream);
int b2sd_state_set_image_embeds(b2sd_handle h, b2sd_state_handle state, const void* tokens_f16, int n_tok, float scale,
                                void* stream);
/* ControlNet conditioning scale (an engine with controlnet = 1), per stream-batch slot: each slot's ControlNet residuals
 * (every zero conv's output, bias included) are multiplied by its scale before they are added to the UNet's skips, as diffusers'
 * controlnet_conditioning_scale does; a guidance window (control_guidance_start / _end) is a scale of 0 on the slots outside
 * it.  The scales live in the time block beside the time biases, so a change is one small device write: no graph recapture, no
 * parameter changes.  b2sd_set_control_scale sets the engine's global scales from host memory, fp32 [batch], finite (1 after
 * b2sd_create), stream-ordered on `stream` without a host synchronisation; it keeps the global time biases, and
 * b2sd_set_timesteps keeps the global scales.  b2sd_state_set_control_scale computes the state's time block with scales in
 * DEVICE memory (which the caller checks: they are not read on the host), as b2sd_state_set_timesteps does: it keeps the state's
 * own timesteps if it has some computed on h's weight store, and b2sd_state_set_timesteps keeps the state's own scales likewise.
 * Scales or timesteps of a state without the other part of its own take that part from the engine's global block at the
 * call, so a global refresh is followed by setting them again; after a move to another store of the family set the state's
 * timesteps, then its scales, again.  Clearing the state's time block (b2sd_state_clear_conditioning(state, 1)) drops both.
 * Both calls refuse an engine without a ControlNet, and one with several (use b2sd_set_control_scales). */
int b2sd_set_control_scale(b2sd_handle h, const float* scale_per_slot, void* stream);
int b2sd_state_set_control_scale(b2sd_handle h, b2sd_state_handle state, const float* scale_per_slot, void* stream);
/* The same for an engine with any number of ControlNets: per_net_slot is fp32 [controlnet][batch], row i net i's per-slot
 * scales.  Same memory, ordering and keeping rules as the single-net calls above, which these equal with one net. */
int b2sd_set_control_scales(b2sd_handle h, const float* per_net_slot, void* stream);
int b2sd_state_set_control_scales(b2sd_handle h, b2sd_state_handle state, const float* per_net_slot, void* stream);
/* Drop the state's override of the prompt (which = 0) or time (which = 1) block: later steps use the engines' global values.
 * No device work; the override is freed after the steps already submitted with it. */
int b2sd_state_clear_conditioning(b2sd_state_handle state, int which);
/* Canny thresholds (an engine with a ControlNet whose processor is B2SD_CONTROL_CANNY; others are refused): cv2.Canny's
 * threshold1 / threshold2, finite, swapped when low > high and floored; a pixel is a candidate when its L1 gradient magnitude
 * is > low and strong when > high (100 / 200 after b2sd_create, controlnet_aux's defaults).  One pair per frame, shared by
 * every Canny net.  They are host values that canny_head takes as kernel arguments when a step launches it, so a change needs
 * no device work, no graph recapture and no synchronisation: steps submitted before the call keep the old values.
 * b2sd_set_canny_thresholds sets the engine's global pair; b2sd_state_set_canny_thresholds the state's own pair, used by any
 * engine that steps the state (lanes and styles alike, and nothing else about the state changes it);
 * b2sd_state_clear_canny_thresholds makes the state follow the stepping engine's global pair again. */
int b2sd_set_canny_thresholds(b2sd_handle h, double low, double high);
int b2sd_state_set_canny_thresholds(b2sd_state_handle state, double low, double high);
int b2sd_state_clear_canny_thresholds(b2sd_state_handle state);
/* Test aid: how many block copies the steps of engine h have issued to bind a state's (or the global) conditioning */
int64_t b2sd_conditioning_binds(b2sd_handle h);
/* How many frames will be in flight on this GPU (lanes / independent streams).  1 (default): launch policy tuned for the
 * latency of a single frame; > 1: policy tuned for throughput (smaller operand rings so CTAs of different frames share an
 * SM; from 4 frames in flight on, contractions are launched as CTA pairs -- tcgen05.mma.cta_group::2 -- without split-K: least
 * SM time per contraction).
 * Takes effect at the next b2sd_prepare. */
int b2sd_set_concurrency(b2sd_handle h, int frames_in_flight);

#ifdef __cplusplus
}
#endif
#endif /* B200SD_H */
