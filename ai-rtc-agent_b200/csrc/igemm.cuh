// Implicit-GEMM convolution / linear layer on wgmma tensor cores (sm_90a).
//
// One kernel covers every contraction of the UNet and TAESD hot path:
//   conv3x3 (stride 1/2, pad 1), conv1x1, Linear, fused "conv3x3 + 1x1 shortcut" (longer K loop),
//   channel-concatenated inputs (several TMA sources, zero-copy torch.cat), split-K.
// Activations are NHWC fp16; a "row" of the GEMM is one output pixel (or token), a K-block is
// 64 channels of one filter tap, fetched by a 4-D tiled TMA box whose (h, w) origin is shifted by
// the tap offset -- out-of-bounds rows are zero-filled by the TMA unit, which is the conv padding.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

constexpr int IG_BM = 128;        // rows (pixels/tokens) per CTA tile == two wgmma M = 64 slabs
constexpr int IG_BK = 64;         // fp16 elements per K-block (128 B = one swizzle row)
constexpr int IG_MAX_SRC = 3;
constexpr int IG_MAX_STAGES = 8;
constexpr int IG_CONS = 256;      // two consumer warpgroups (MMA + epilogue), warps 0-7
constexpr int IG_THREADS = IG_CONS + 32;   // + warp 8: TMA producer
constexpr int IG_SMS = 132;       // H100 SXM streaming multiprocessors (launch-shape policy)

enum : int {
    IG_RELU = 1,    // relu after bias/residual
    IG_GEGLU = 2,   // tile columns [0,BN/2) = value, [BN/2,BN) = gate; out = v * gelu_erf(g)
    IG_SPLITK = 4,  // set by the planner: K is split over a thread-block cluster, partial tiles are reduced through DSMEM
    IG_SILU = 8,    // x * sigmoid(x) after bias/residual (ControlNet conditioning embedding)
    IG_PAD0 = 16,   // 3x3 taps start at the output pixel (input coord = stride * out + tap; zero row/column only at the far edge)
};

struct IgEpilogue {
    __half* out;            // [rows][ldc] fp16
    int ldc;
    const float* colbias;   // fp32 [nb][colbias_bstride]: bias (+ time-embedding projection); may be null
    int colbias_bstride;    // 0 => shared by every batch item
    const __half* res;      // residual / noise, same row indexing as out; may be null
    int ldr;
    float acc_scale;        // out = acc_scale * (acc + bias) + res_scale * res
    float res_scale;
    int flags;
    int n_valid;            // valid output columns (Cout)
    // ---- LayerNorm without a LayerNorm launch (transformer blocks: diffusers attention.py BasicTransformerBlock norm1/2/3) ----
    // producer side: besides storing its fp16 output rows, accumulate their (sum, sum of squares) as 2^20 fixed point in
    // 64-bit integer atomics -- integer addition commutes, so the statistics are bit-reproducible whatever order the N tiles
    // and split-K CTAs arrive in.  [rows][2], zeroed at the start of every frame.
    unsigned long long* rowstat_out;
    // consumer side: y = LN(x) W^T + b  ==  rstd_r * (x W'^T - mean_r * colsum) + bias'  with W' = W diag(gamma) (packed at load
    // time), colsum[n] = sum_k W'[n][k], bias'[n] = sum_k W[n][k] beta[k] + b[n] (passed as colbias).  rowstat_in = the
    // statistics of this GEMM's A rows written by its producer; ln_inv_c = 1 / C, ln_eps = 1e-5.
    const unsigned long long* rowstat_in;
    const float* colsum;
    float ln_inv_c, ln_eps;
    // ---- fused q/k/v projection: output columns >= col2 (the V block) are stored TRANSPOSED, out2[(col - col2) * ld2 + row],
    // which is the K-major V^T operand the attention kernel's P.V MMA reads (was a separate swapped-operand GEMM launch)
    __half* out2;
    int ld2, col2;
};

constexpr float IG_STAT_SCALE = 1048576.f;   // 2^20 fixed point of the row statistics

struct IgemmParams {
    CUtensorMap tmA[IG_MAX_SRC];
    CUtensorMap tmB;
    int seg_ntap[IG_MAX_SRC];     // 1 or 9
    int seg_cblocks[IG_MAX_SRC];  // 64-channel blocks in this segment
    int seg_c0[IG_MAX_SRC];       // first channel inside the source view
    int nseg;
    int total_kb;
    int kb_per_split;
    int tw, th, tn;               // output tile = tn images x th rows x tw cols  (<= 128 pixels)
    int tiles_w, tiles_h, tiles_n;
    int Wo, Ho, Nb;
    int stride;                   // input coord = stride * out + tap - 1 (IG_PAD0: + tap)
    int BN;                       // wgmma N (multiple of 16, <= 256)
    int num_stages;
    int acc_bufs;                 // 1, or 2 when the launch is persistent over M tiles
    uint32_t a_bytes;             // TMA box bytes of one A tile
    uint32_t b_bytes;
    uint32_t tmem_cols;           // accumulator columns of the tile(s) a CTA holds, rounded up to a power of two (plan info)
    unsigned long long* dbg_ts;   // debug: 8 globaltimer stamps per CTA (null = off)
    int n_pad;
    int swap;                     // 1: weights on the M side (128 output channels per CTA), pixels on the N side
    int tw_log2, th_log2;         // swap mode: pixel-tile extents are powers of two
    int dbg_mode;                 // bound study (-DB2_BOUND_STUDY + env B2_DBG_MODE): 1 = TMA loads only for the first ring pass, 2 = no MMAs
    IgEpilogue epi;
};

struct ActView {
    const __half* ptr;
    int N, H, W, C;   // logical NHWC extents visible to the TMA map
    int ld;           // channel pitch in elements (>= C, multiple of 8)
};

struct IgemmDesc {
    ActView src[IG_MAX_SRC];
    int ntap[IG_MAX_SRC];
    int nseg;
    const __half* w;  // packed weights [w_rows][w_ld], K order = segments in sequence, each [tap][c]
    int w_rows;
    int w_ld;
    int stride;
    int Nb, Ho, Wo;
    int BN;           // 0 = auto
    int swap;         // 1 = swapped orientation: D^T = W . X^T, BN pixels (64/128/256) on the N side, transposed store
    int splits;       // 0/1 = none
    int ring_kb;      // operand ring budget in KB, 0 = auto (200, or 100 when two CTAs per SM are resident and needed)
    int max_splits;   // cap of the split-K factor chosen by igemm_autotile, 0 = 8
    int pair_auto;    // igemm_autotile only: 0 = single CTAs, 1 = launch every eligible contraction as CTA pairs, 2 = only K >= 1280
    int pair_splits;  // ... and cap the split-K factor of those paired launches (0 = 4); the N tile of the single-CTA policy is kept
    int pair;         // 1 = CTA pairs (2-CTA cluster): neighbouring M tiles share the weight tile, each CTA loads half of it
                      // and multicasts it to both.  Normal orientation only, BN % 32 == 0, split-K <= 4.
    unsigned long long* dbg_ts;  // optional per-CTA timeline (8 stamps per CTA)
    float* partial;   // unused since split-K moved into a cluster (kept for ABI stability; op-level entry: debug timeline)
    int* tile_counters;  // unused (ABI stability)
    IgEpilogue epi;
};

struct IgemmPlan {
    int mode;       // 0 = single CTAs, 1 = CTA pairs (plan-info ABI)
    IgemmParams p;
    dim3 grid;
    size_t smem;
    int splits;
    long rows_total;
    int pair;       // launched as CTA pairs with cluster dims (2, 1, splits)
};

// Returns 0 on success; fills plan. Encodes TMA descriptors (host side, no launch).
int igemm_plan(const IgemmDesc& d, IgemmPlan* plan);
// Enqueue on stream (one launch; split-K plans launch a thread-block cluster per output tile).
int igemm_launch(const IgemmPlan& plan, cudaStream_t stream);
// dry run (this thread): igemm_plan computes tiling, grid, shared memory, pipeline depth but encodes no TMA descriptor,
// so it works on a machine without a GPU driver (host-logic tests)
void igemm_set_dry_run(bool on);
// one-time function attributes / driver entry points (call outside stream capture)
int igemm_init();
// streaming multiprocessors of the current device (IG_SMS when there is none)
int b2_device_sms();
// legacy: workspace floats of the former global-memory split-K (no workspace is needed any more)
size_t igemm_partial_floats(int splits, long rows_total, int n_valid);
const char* b2_last_error();
void b2_set_error(const char* fmt, ...);

}  // namespace b2

// Tile / split-K policy of the frame program (engine.cu): picks BN, split-K factor and orientation for one contraction and
// fills `plan`.  Host-only logic; combine with igemm_set_dry_run(true) to evaluate it without a GPU.
int igemm_autotile(b2::IgemmDesc d, bool allow_swap, b2::IgemmPlan* plan);
