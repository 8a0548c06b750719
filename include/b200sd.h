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
 *   out[row][j] = acc_scale * (sum_seg sum_tap sum_c src[seg](row, tap, c) * w[j][k] + colbias[b][j])
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
} b2sd_igemm_plan_info;
int b2sd_igemm_plan_dry(const b2sd_igemm_desc* d, int autotile, int allow_swap, b2sd_igemm_plan_info* out);

/* Host-only: launch shape of GroupNorm over [ca | cb] channels, hw pixels per image: cluster = CTAs per (image, group) of the
 * cluster kernel (0 = whole-grid cooperative kernel), threads per CTA, pixels per CTA. */
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

/* GroupNorm(+SiLU) over the channel concatenation [xa | xb] (xb may be NULL), NHWC fp16. */
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

/* ------------------------------------------------------------------------------------------------
 * Engine level: one handle == one temporal stream (one StreamDiffusion instance, lib/wrapper.py:168).
 * Replaces StreamDiffusion + UNet2DConditionModelEngine + AutoencoderKLEngine
 * (lib/wrapper.py:445-466, 494-504) for mode="img2img", use_denoising_batch=True, frame_buffer_size=1,
 * cfg_type="self" with guidance_scale <= 1 (the only configuration lib/pipeline.py:23-42 builds).
 * ---------------------------------------------------------------------------------------------- */
typedef struct b2sd_engine* b2sd_handle;

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
                                    A lane inherits its parent's value. */
    int control_processor;       /* with controlnet = 1: B2SD_CONTROL_FRAME (0) or B2SD_CONTROL_HED (1): the control image is the
                                    HED edge map of the frame (controlnet_aux HEDdetector at the engine's size; weights under
                                    "hed." + ControlNetHED.pth keys, e.g. "hed.block1.convs.0.weight", "hed.norm").  Inherited
                                    by lanes. */
    int vae;                     /* B2SD_VAE_TINY (0): TAESD (weights "vae." + AutoencoderTiny keys).  B2SD_VAE_KL (1): the model's
                                    own AutoencoderKL (weights "vae." + diffusers AutoencoderKL keys, e.g.
                                    "vae.encoder.down_blocks.0.resnets.0.conv1.weight", "vae.quant_conv.weight"; mid-block attention
                                    as to_q / to_k / to_v / to_out.0 with q/k/v as [512][512]); the latent is scaling_factor times the
                                    mean of the encoder's distribution (not a sample).  Inherited by lanes. */
    float vae_scaling_factor;    /* with vae = B2SD_VAE_KL: vae/config.json scaling_factor; 0 = 0.18215 */
} b2sd_config;
enum { B2SD_CONTROL_FRAME = 0, B2SD_CONTROL_HED = 1 };
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
 * B2_KEEP_RAW=1 to keep them); loading further tensors into such an engine is an error. */
int b2sd_load_tensor(b2sd_handle h, const char* key, const void* ptr, int dtype, const int64_t* shape, int ndim);

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
/* StreamDiffusion.update_prompt (lib/pipeline.py:44-45): refresh the per-layer cross-attention K/V cache */
int b2sd_set_prompt_embeds(b2sd_handle h, const void* prompt_embeds, void* stream);
/* lib/wrapper.py:389-407 update_t_index_list: only sub_timesteps change (alpha/beta/c_skip/c_out keep the
 * values given to b2sd_prepare -- reference behaviour) */
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
 * "control" (the u8 edge value as fp16, [1][h][w][1]).
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
/* Stage pipelining of ONE stateful stream (stream batch T > 1, where frame n+1 needs frame n's latent buffer and lanes cannot
 * simply alternate): `lane` shares `owner`'s stream-batch state; the frame program of each is cut into TAESD encoder body |
 * last encoder conv + UNet + scheduler step | TAESD decoder, and only the middle stage is serialised between the lanes (one
 * CUDA event), so the encoder of frame n+1 and the decoder of frame n-1 overlap the UNet of frame n.  Both engines must be
 * lanes of one weight store with equal batch / size; call before b2sd_prepare; submit frames alternately, in order. */
int b2sd_share_stream_state(b2sd_handle lane, b2sd_handle owner);
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
