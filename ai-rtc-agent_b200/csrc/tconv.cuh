// Persistent 3x3 convolution for the TAESD body (64 -> 64 channels, stride 1) on wgmma tensor cores.
//
// TAESD (lib/wrapper.py:445-453: the reference's vae_encoder / vae_decoder engines) is 60 such convolutions over up to
// 512x512 pixels.  With one 64-wide N tile the generic tap-by-tap kernel (igemm.cu) spends its shared-memory port on
// refilling operands: per output tile it re-fetches the activations nine times (once per filter tap) and the 72 KB weight
// matrix once.  Here
//   * the whole weight matrix (9 taps x [64 x 64]) is loaded ONCE per CTA and stays resident in shared memory,
//   * one TMA load brings an (16+2) x (8+2)-pixel halo tile; the nine taps are nine shifted wgmma descriptors over it,
//   * CTAs are persistent (one per SM) with a ring of halo buffers and two consumer warpgroups that take alternate tiles
//     (accumulators in registers), so loads, MMAs and the epilogue of neighbouring tiles overlap,
//   * each warpgroup commits a tile's two 64-pixel slabs as two wgmma groups and runs slab 0's epilogue while slab 1's MMAs
//     are still in the tensor pipe,
//   * the residual arrives by TMA in a per-warpgroup staging tile; the epilogue reads it there, writes the fp16 result in its
//     place and TMA stores it, so no thread of the epilogue waits on a global load.
// Operand fill drops from 216 KB to 23 KB per 128-pixel tile.
//
// Shared memory (227 KB per SM): 72 KB of weights, TC_MAX_ABUF halo slots of 23 KB, two 16 KB residual / staging tiles.
#pragma once
#include "igemm.cuh"

namespace b2 {

constexpr int TC_CONS = 256;           // warps 0-7: two consumer warpgroups (MMA + epilogue)
constexpr int TC_THREADS = TC_CONS + 32;   // + warp 8: TMA producer
constexpr int TC_TW = 8, TC_TH = 16;   // output tile: 16 rows x 8 columns = 128 pixels (= two wgmma M = 64 slabs); 8-pixel rows are the 8-row core groups
constexpr int TC_C = 64;               // input channels == output channels == one 128-byte swizzle row
constexpr int TC_MAX_ABUF = 4;         // halo ring depth: 6 slots and the staging tiles would not fit beside the weights

struct TconvParams {
    CUtensorMap tmA;       // activations NHWC: box (64 ch, TW+2, TH+2, 1), zero fill outside the image = conv padding
    CUtensorMap tmB;       // packed weights [64][9*64] (K order [tap][c]): box (64 k, 64 rows)
    CUtensorMap tmO;       // output NHWC (pitch ldc): box (64 ch, TW, TH/2, 1), one slab per store
    CUtensorMap tmR;       // residual NHWC (pitch ldr): box (64 ch, TW, TH, 1); encoded only when the epilogue has one
    int tiles_w, tiles_h, num_tiles;
    int Wo, Ho, Nb;
    int nbuf;              // halo ring depth
    uint32_t abuf_bytes;   // one halo buffer (1024-aligned)
    IgEpilogue epi;
};

struct TconvPlan {
    TconvParams p;
    dim3 grid;
    size_t smem;
    long rows_total;
};

// stride-1 3x3, one 64-channel source, 64 output channels, epilogue of bias shared by the batch / scale / residual / ReLU
// with 16-byte-aligned pitches
bool tconv_eligible(const IgemmDesc& d);
int tconv_plan(const IgemmDesc& d, TconvPlan* plan);   // honours igemm_set_dry_run()
int tconv_launch(const TconvPlan& plan, cudaStream_t stream);
int tconv_init();

}  // namespace b2
