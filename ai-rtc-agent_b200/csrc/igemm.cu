// wgmma implicit-GEMM kernel + host-side plan builder. See igemm.cuh for the design.
#include "igemm.cuh"

#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "epilogue.cuh"
#include "launch.cuh"
#include "ptx.cuh"

namespace b2 {

// per-CTA timeline stamps (tools/timeline.py): compiled in only with -DB2_TIMELINE, they lengthen the MMA issue loop
#ifdef B2_TIMELINE
#define B2_TS(stmt) stmt
#else
#define B2_TS(stmt)
#endif

// ------------------------------------------------------------------------------------------
// error string shared by the whole library (C-ABI: b2sd_last_error)
static thread_local char g_err[1024] = "";
const char* b2_last_error() { return g_err; }
void b2_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// Swapped orientation: an accumulator row is an output CHANNEL, its columns are the pixels of the tile, so the NHWC store
// needs a transpose.  It goes through a small fp32 shared-memory tile T[pixel][128 channels]: the consumer warpgroups park a
// chunk of <= 32 pixels of their fragments there, then the 256 consumer threads sweep T row-wise: one thread = 8 consecutive
// channels of one pixel (16-byte residual load, 16-byte store), a warp = two complete 256-byte pixel rows.  Bias, scale,
// residual and ReLU are applied in that coalesced sweep.
constexpr int SWAP_CH = 32;                        // pixels per transposition chunk (T = 32 x 128 fp32 = 16 KB)
constexpr int SWAP_ITEMS = SWAP_CH * 16 / IG_CONS;   // (pixel, 8-channel) items per consumer thread and chunk

__device__ __forceinline__ void cons_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(IG_CONS) : "memory"); }

// What one thread needs from global memory for its (pixel, 8-channel) items of a chunk: fetched BEFORE the
// transposition barrier so the latency overlaps the fills of T.
struct SwapPre {
    uint4 res[SWAP_ITEMS];
    float4 b0[SWAP_ITEMS], b1[SWAP_ITEMS];
    long orow[SWAP_ITEMS];      // < 0: nothing to store
};

__device__ __forceinline__ void swap_prefetch(const IgemmParams& p, SwapPre& pre, int npix, int j0, int ntile, int n0, int h0,
                                              int w0, int t) {
    const IgEpilogue& e = p.epi;
    const int tw = 1 << p.tw_log2, th = 1 << p.th_log2;
#pragma unroll
    for (int k = 0; k < SWAP_ITEMS; ++k) {
        const int item = t + IG_CONS * k;
        pre.orow[k] = -1;
        pre.res[k] = make_uint4(0, 0, 0, 0);
        pre.b0[k] = pre.b1[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (item >= npix * 16) continue;
        const int pl = item >> 4, q = item & 15;
        const int j = j0 + pl;
        const int wi = j & (tw - 1);
        const int hi = (j >> p.tw_log2) & (th - 1);
        const int ni = j >> (p.tw_log2 + p.th_log2);
        const int n = n0 + ni, h = h0 + hi, w = w0 + wi;
        const int cout0 = ntile * IG_BM + q * 8;
        if (ni >= p.tn || n >= p.Nb || h >= p.Ho || w >= p.Wo || cout0 >= e.n_valid) continue;
        const long orow = ((long)n * p.Ho + h) * p.Wo + w;
        pre.orow[k] = orow;
        if (e.colbias) {
            const float4* bp = reinterpret_cast<const float4*>(e.colbias + (long)n * e.colbias_bstride + cout0);
            pre.b0[k] = __ldg(bp);
            pre.b1[k] = __ldg(bp + 1);
        }
        if (e.res) pre.res[k] = __ldg(reinterpret_cast<const uint4*>(e.res + orow * e.ldr + cout0));
    }
}

template <bool SILU>
__device__ __forceinline__ void swap_store_chunk(const IgemmParams& p, const SwapPre& pre, const float* T, int ntile, int t) {
    const IgEpilogue& e = p.epi;
#pragma unroll
    for (int k = 0; k < SWAP_ITEMS; ++k) {
        if (pre.orow[k] < 0) continue;
        const int item = t + IG_CONS * k;
        const int pl = item >> 4, q = item & 15;
        const int cout0 = ntile * IG_BM + q * 8;
        const float4 a0 = *reinterpret_cast<const float4*>(T + pl * IG_BM + q * 8);
        const float4 a1 = *reinterpret_cast<const float4*>(T + pl * IG_BM + q * 8 + 4);
        const float4 b0 = pre.b0[k], b1 = pre.b1[k];
        float v[8] = {a0.x + b0.x, a0.y + b0.y, a0.z + b0.z, a0.w + b0.w, a1.x + b1.x, a1.y + b1.y, a1.z + b1.z, a1.w + b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] *= e.acc_scale;
        if (e.res) {
            const __half2* rh = reinterpret_cast<const __half2*>(&pre.res[k]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = __half22float2(rh[i]);
                v[2 * i] += e.res_scale * f.x;
                v[2 * i + 1] += e.res_scale * f.y;
            }
        }
        if (e.flags & IG_RELU) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
        }
        if (SILU && (e.flags & IG_SILU)) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = silu_f(v[i]);
        }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) oh[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        *reinterpret_cast<uint4*>(e.out + pre.orow[k] * e.ldc + cout0) = o;
    }
}

// Cluster split-K: sum one 16-column (4 x float4) strip of accumulator row `row` over the K slices held in the peers'
// shared memory.  All loads of up to four slices are in flight together (a dependent chain of DSMEM round trips was
// the dominant cost of the reduction); the summation order is fixed => bit-reproducible.
// (pair launches: cluster dims (2,1,splits), the K slice s of this CTA's M tile lives in cluster rank 2*s + rank_add)
template <int SPL>
__device__ __forceinline__ void splitk_sum16(uint32_t stg_local, int cc, int row, float (&acc)[16], int rank_mul = 1, int rank_add = 0) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    constexpr int G = SPL < 4 ? SPL : 4;
#pragma unroll
    for (int s0 = 0; s0 < SPL; s0 += G) {
        float4 v[G][4];
#pragma unroll
        for (int s = 0; s < G; ++s) {
            const uint32_t peer = dsmem_map(stg_local, (uint32_t)((s0 + s) * rank_mul + rank_add));
#pragma unroll
            for (int i = 0; i < 4; ++i) v[s][i] = dsmem_ld_f4(peer + (uint32_t)(((cc * 4 + i) * IG_BM + row) * 16));
        }
#pragma unroll
        for (int s = 0; s < G; ++s)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                acc[4 * i] += v[s][i].x; acc[4 * i + 1] += v[s][i].y; acc[4 * i + 2] += v[s][i].z; acc[4 * i + 3] += v[s][i].w;
            }
    }
}

// ------------------------------------------------------------------------------------------
// Warp roles: warps 0-3 and 4-7 are the two consumer warpgroups (accumulator rows [0,64) and [64,128) of the tile, wgmma
// M = 64 each, the fp32 accumulator lives in their registers), warp 8 lane 0 is the TMA producer.  The consumers run the
// epilogue of a tile straight from their registers, so a persistent CTA's next mainloop starts after that epilogue; the
// producer meanwhile fills the ring for the next tile.
//
// PAIR: the CTAs (2j, 2j+1) of grid.x form a cluster pair (cluster dims (2,1,splits)) that computes two neighbouring M tiles
// with the same weight tile: each CTA loads its own 128 pixel rows and HALF of the weight rows, multicast into both CTAs'
// shared memory, so each SM fetches half of the weight bytes from L2.  A ring slot is refilled only when the warps of BOTH
// CTAs have released it (every consumer warp arrives on its own and on the peer's empty barrier).
template <int BN, bool PAIR, bool SILU, bool PAD0 = false>
__device__ __forceinline__ void igemm_body(const IgemmParams& p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                               ~static_cast<uintptr_t>(1023));
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    constexpr uint32_t A_BYTES = IG_BM * IG_BK * 2;
    constexpr uint32_t stage_bytes = A_BYTES + (uint32_t)BN * IG_BK * 2;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.num_stages * stage_bytes);
    uint64_t* empty_bar = full_bar + IG_MAX_STAGES;
    const int cr = PAIR ? (int)(blockIdx.x & 1) : 0;       // rank inside the CTA pair
    const int mt_first = (int)blockIdx.x;                  // first M tile of this CTA ...
    const int mt_step = (int)gridDim.x;                    // ... and the stride of a persistent launch (even for pairs)
    const int mt_guard = PAIR ? cr : 0;                    // pairs iterate together: the loop bound looks at the even CTA's tile

    // Persistent over M tiles: CTA x handles tiles x, x + gridDim.x, ...; the prologue (barriers, descriptors) is paid once.
    const int num_mtiles = p.tiles_w * p.tiles_h * p.tiles_n;
    const int ntile = blockIdx.y;
    const int kb_begin = blockIdx.z * p.kb_per_split;
    const int kb_end = min(p.total_kb, kb_begin + p.kb_per_split);
    [[maybe_unused]] unsigned long long* ts = p.dbg_ts ? p.dbg_ts + ((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 8 : nullptr;
    B2_TS(if (ts && threadIdx.x == 0) ts[0] = globaltimer_ns();)

    if (threadIdx.x == IG_CONS) {
        for (int s = 0; s < p.nseg; ++s) tma_prefetch_desc(&p.tmA[s]);
        tma_prefetch_desc(&p.tmB);
        for (int s = 0; s < p.num_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], (PAIR ? 2 : 1) * (IG_CONS / 32));   // one arrival per consumer warp (of both CTAs)
        }
        fence_mbar_init();
    }
    if (PAIR) {   // the peer's barriers exist before anything arrives on them (execution barrier only: the release/acquire form
        cluster_arrive_relaxed();   // costs a MEMBAR.ALL.GPU + L1 invalidate)
        cluster_wait();
    }
    __syncthreads();

    pdl_launch_dependents();   // the next kernel may start its own prologue now
    pdl_wait();                // ... and everything below reads the previous kernel's output
    B2_TS(if (ts && threadIdx.x == 0) ts[1] = globaltimer_ns();)

    if (warp == IG_CONS / 32) {
        if (lane == 0) {
            // ===== TMA producer =====
            [[maybe_unused]] const uint16_t pair_mask = PAIR ? (uint16_t)(3u << (cluster_ctarank() & ~1u)) : (uint16_t)0;
            int stage = 0;
            uint32_t phase = 0;
            for (int mt = mt_first; mt - mt_guard < num_mtiles; mt += mt_step) {
                const int w0 = (mt % p.tiles_w) * p.tw, h0 = ((mt / p.tiles_w) % p.tiles_h) * p.th;
                const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.tn;   // (odd tile count: the last pair's second tile lies outside, TMA zero-fills)
                int seg = 0, base = 0;
                while (seg < p.nseg - 1 && kb_begin >= base + p.seg_ntap[seg] * p.seg_cblocks[seg]) {
                    base += p.seg_ntap[seg] * p.seg_cblocks[seg];
                    ++seg;
                }
                int tap = (kb_begin - base) / p.seg_cblocks[seg];
                int cb = (kb_begin - base) % p.seg_cblocks[seg];
                for (int kb = kb_begin; kb < kb_end; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
#ifdef B2_BOUND_STUDY
                    if (p.dbg_mode == 1 && kb >= kb_begin + p.num_stages) {   // bound study: operands stay whatever they were
                        mbar_arrive(&full_bar[stage]);
                        if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
                        continue;
                    }
#endif
                    mbar_expect_tx(&full_bar[stage], p.a_bytes + p.b_bytes);
                    uint8_t* sa = smem + (size_t)stage * stage_bytes;
                    uint8_t* sb = sa + A_BYTES;
                    int dy = 0, dx = 0;
                    if (p.seg_ntap[seg] == 9) {   // PAD0: tap origin 0 (input coord = stride * out + tap)
                        dy = tap / 3 - (PAD0 ? 0 : 1);
                        dx = tap % 3 - (PAD0 ? 0 : 1);
                    }
                    // normal: pixels -> A (M side), weights -> B.  swapped: weights (128 output channels) -> A, pixels -> B
                    tma_load_4d(p.swap ? sb : sa, &p.tmA[seg], &full_bar[stage], p.seg_c0[seg] + cb * IG_BK,
                                w0 * p.stride + dx, h0 * p.stride + dy, n0);
                    if (PAIR)
                        tma_load_2d_mc(sb + cr * (BN / 2) * 128, &p.tmB, &full_bar[stage], kb * IG_BK, ntile * BN + cr * (BN / 2), pair_mask);
                    else
                        tma_load_2d(p.swap ? sa : sb, &p.tmB, &full_bar[stage], kb * IG_BK, ntile * (p.swap ? IG_BM : BN));
                    B2_TS(if (ts && mt == (int)blockIdx.x && kb == kb_begin) ts[2] = globaltimer_ns();)
                    if (++cb == p.seg_cblocks[seg]) {
                        cb = 0;
                        if (++tap == p.seg_ntap[seg]) {
                            tap = 0;
                            ++seg;
                        }
                    }
                    if (++stage == p.num_stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroups: wgmma mainloop, then the epilogue from registers =====
        const int wg = warp >> 2;                                   // accumulator rows [64 wg, 64 wg + 64) of the tile
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // this thread's rows: r0 and r0 + 8
        [[maybe_unused]] const uint32_t peer_empty = PAIR ? dsmem_map(smem_u32(empty_bar), cluster_ctarank() ^ 1u) : 0u;
        const IgEpilogue& e = p.epi;
        const bool ln_fma = e.colsum && !p.swap && !(e.flags & IG_SPLITK) && (e.ldc & 7) == 0 && (e.n_valid & 15) == 0;
        const uint32_t smem_base = smem_u32(smem);
        auto release = [&](int s) {   // this warp's reads of ring slot s have retired
            if (lane == 0) {
                mbar_arrive(&empty_bar[s]);
                if (PAIR) mbar_arrive_remote(peer_empty + (uint32_t)s * 8u);
            }
        };
        int stage = 0;
        uint32_t phase = 0;
        int it = 0;
        for (int mt = mt_first; mt - mt_guard < num_mtiles; mt += mt_step, ++it) {
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev = -1;
            for (int kb = kb_begin; kb < kb_end; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                B2_TS(if (ts && it == 0 && kb == kb_begin && threadIdx.x == 0) ts[3] = globaltimer_ns();)
                const uint32_t sa = smem_base + (uint32_t)stage * stage_bytes;
                const uint64_t da = make_kmajor_sw128_desc(sa + (uint32_t)wg * (64 * 128));
                const uint64_t db = make_kmajor_sw128_desc(sa + A_BYTES);
#ifdef B2_BOUND_STUDY
                if (p.dbg_mode != 2)
#endif
                {
                    wgmma_fence_regs(acc);
                    wgmma_fence();
                    // +32 B per K = 16 step inside the 128 B swizzle row => +2 in the (addr >> 4) field
#pragma unroll
                    for (int k = 0; k < 4; ++k) Wgmma<BN>::ss(acc, da + 2 * k, db + 2 * k, 1u);
                    wgmma_commit();
                    wgmma_wait<1>();   // the previous K-block's MMAs have retired: its slot may be refilled
                    wgmma_fence_regs(acc);
                }
                if (prev >= 0) release(prev);
                prev = stage;
                if (++stage == p.num_stages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            if (prev >= 0) release(prev);
            B2_TS(if (ts && it == 0 && threadIdx.x == 0) ts[4] = globaltimer_ns();)

            const int w0 = (mt % p.tiles_w) * p.tw, h0 = ((mt / p.tiles_w) % p.tiles_h) * p.th;
            const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.tn;
            if (p.swap || (e.flags & IG_SPLITK)) {
                // one tile per CTA (swapped and split-K plans are never persistent): once both warpgroups have retired their
                // MMAs the operand ring is idle and its head holds the fp32 tile
                float* stg = reinterpret_cast<float*>(smem);
                cons_bar_sync();
                if (e.flags & IG_SPLITK) {
                    // Split-K inside a thread-block cluster (one CTA per K slice): every CTA parks its fp32 partial tile in its
                    // own shared memory, laid out [4-column group][row]; the reduction happens after the cluster barrier below.
                    frag_to_smem<BN>(stg, acc, r0, lane, 0, BN, false);
                } else {
                    for (int c = 0; c < BN; c += SWAP_CH) {
                        SwapPre pre;
                        swap_prefetch(p, pre, SWAP_CH, c, ntile, n0, h0, w0, threadIdx.x);
                        frag_to_smem<BN>(stg, acc, r0, lane, c, SWAP_CH, true);
                        cons_bar_sync();
                        swap_store_chunk<SILU>(p, pre, stg, ntile, threadIdx.x);
                        cons_bar_sync();
                    }
                }
            } else {
                EpiRow rw[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const int wi = r % p.tw, hi = (r / p.tw) % p.th, ni = r / (p.tw * p.th);
                    const int n = n0 + ni, hh = h0 + hi, ww = w0 + wi;
                    rw[h].ok = (ni < p.tn) && (n < p.Nb) && (hh < p.Ho) && (ww < p.Wo);
                    rw[h].orow = ((long)n * p.Ho + hh) * p.Wo + ww;
                    rw[h].b = n;
                    ln_row_stats(e, rw[h].orow, rw[h].ok, rw[h].mu, rw[h].rstd);
                }
                epi_frag<BN, SILU>(e, acc, rw, ntile, ln_fma, lane);
            }
            B2_TS(if (ts && it == 0 && threadIdx.x == 0) ts[5] = globaltimer_ns();)
        }
    }
    if (p.epi.flags & IG_SPLITK) {
        // ---- cluster-wide deterministic reduction over the K slices through distributed shared memory ----
        const int mt = blockIdx.x;
        const int w0 = (mt % p.tiles_w) * p.tw, h0 = ((mt / p.tiles_w) % p.tiles_h) * p.th;
        const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.tn;
        const int splits = (int)gridDim.z;
        const int rk_mul = PAIR ? 2 : 1, rk_add = cr;   // cluster rank of K slice s (same M tile) = s * rk_mul + rk_add
        cluster_sync_all();  // all partial tiles are in place (release/acquire over the cluster)
        B2_TS(if (ts && threadIdx.x == 0) ts[6] = globaltimer_ns();)   // split launches: [6] cluster barrier passed, [7] reduced
        if (warp < IG_CONS / 32 && p.swap) {
            // swapped orientation: this CTA finalises the pixel columns [rank*cols_per, (rank+1)*cols_per) of the tile; the two
            // halves of the consumer threads take alternate 16-pixel strips (8 pixels: one float4 group each) of one channel row
            const int rank = (int)cluster_ctarank();
            const int cols_per = BN / splits;
            const int ch = cols_per < SWAP_CH ? cols_per : SWAP_CH;
            const int t = threadIdx.x & (IG_BM - 1);     // accumulator row == output channel of the tile
            const int half = threadIdx.x >> 7;
            const uint32_t stg_local = smem_u32(smem);
            float* T = reinterpret_cast<float*>(smem + (size_t)BN * IG_BM * 4);   // right after the staging tile
            for (int c = rank * cols_per; c < (rank + 1) * cols_per; c += ch) {
                SwapPre pre;
                swap_prefetch(p, pre, ch, c, ntile, n0, h0, w0, threadIdx.x);
                if (ch >= 16) {
                    for (int g = 4 * half; g < (ch >> 2); g += 8) {     // 16 pixel columns per pass (ch is 16 or 32)
                        float acc[16];
                        const int cc = ((c >> 2) + g) >> 2;      // 16-column strip index
                        switch (splits) {
                            case 2: splitk_sum16<2>(stg_local, cc, t, acc); break;
                            case 4: splitk_sum16<4>(stg_local, cc, t, acc); break;
                            default: splitk_sum16<8>(stg_local, cc, t, acc); break;
                        }
#pragma unroll
                        for (int i = 0; i < 16; ++i) T[(4 * g + i) * IG_BM + t] = acc[i];
                    }
                } else {
                    // 8 pixel columns per CTA (BN 64 over 8 slices): two float4 groups, one per half
                    const int gg = half;
                    float4 v[8];
#pragma unroll
                    for (int sidx = 0; sidx < 8; ++sidx)
                        v[sidx] = dsmem_ld_f4(dsmem_map(stg_local, (uint32_t)sidx) + (uint32_t)((((c >> 2) + gg) * IG_BM + t) * 16));
                    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int sidx = 0; sidx < 8; ++sidx) { a.x += v[sidx].x; a.y += v[sidx].y; a.z += v[sidx].z; a.w += v[sidx].w; }
                    T[(4 * gg + 0) * IG_BM + t] = a.x;
                    T[(4 * gg + 1) * IG_BM + t] = a.y;
                    T[(4 * gg + 2) * IG_BM + t] = a.z;
                    T[(4 * gg + 3) * IG_BM + t] = a.w;
                }
                cons_bar_sync();
                swap_store_chunk<SILU>(p, pre, T, ntile, threadIdx.x);
                cons_bar_sync();
            }
        } else if (warp < IG_CONS / 32) {
            const int rank = (int)cluster_ctarank() / rk_mul;
            const int rows_per = IG_BM / splits;          // splits in {2,4,8}
            const int t = threadIdx.x;
            const int chunks = BN >> 4;
            const uint32_t stg_local = smem_u32(smem);
            for (int item = t; item < rows_per * chunks; item += IG_CONS) {
                const int rl = item % rows_per;
                const int cc = item / rows_per;
                const int r = rank * rows_per + rl;       // row of the tile this CTA finalises
                const int wi = r % p.tw, hi = (r / p.tw) % p.th, ni = r / (p.tw * p.th);
                const int n = n0 + ni, h = h0 + hi, w = w0 + wi;
                const bool ok = (ni < p.tn) && (n < p.Nb) && (h < p.Ho) && (w < p.Wo);
                float acc[16];
                switch (splits) {
                    case 2: splitk_sum16<2>(stg_local, cc, r, acc, rk_mul, rk_add); break;
                    case 4: splitk_sum16<4>(stg_local, cc, r, acc, rk_mul, rk_add); break;
                    default: splitk_sum16<8>(stg_local, cc, r, acc, rk_mul, rk_add); break;
                }
                if (ok) {
                    const long orow = ((long)n * p.Ho + h) * p.Wo + w;
                    float mu, rstd;
                    ln_row_stats(p.epi, orow, true, mu, rstd);
                    epi_store16<0, 16, float, SILU>(p.epi, acc, n, orow, ntile * BN + cc * 16, mu, rstd);
                }
            }
        }
        B2_TS(if (ts && threadIdx.x == 0) ts[7] = globaltimer_ns();)
        cluster_sync_all();  // nobody may exit while a peer still reads its shared memory
    }
    if (PAIR) {   // nobody exits while the peer may still multicast into it or arrive on its barriers
        cluster_arrive_relaxed();
        cluster_wait();
    }
}

template <int BN, bool PAIR, bool SILU = false>
__global__ void __launch_bounds__(IG_THREADS, 1) igemm_kernel(const __grid_constant__ IgemmParams p) { igemm_body<BN, PAIR, SILU>(p); }
// IG_PAD0: 3x3 taps read input (stride * out + tap), i.e. F.pad(x, (0, 1, 0, 1)) before an unpadded conv -- the AutoencoderKL
// Downsample2D(padding=0).  Its own instantiations (single CTAs, N tiles 64 / 128 / 256), so every other kernel is unchanged.
template <int BN>
__global__ void __launch_bounds__(IG_THREADS, 1) igemm_pad0_kernel(const __grid_constant__ IgemmParams p) { igemm_body<BN, false, false, true>(p); }

using IgemmFn = void (*)(IgemmParams);
// every N tile the planner can produce (multiples of 16 up to 256); CTA pairs need BN % 32 == 0.  At 168 registers the widest
// tiles (BN >= 192: 96+ accumulator registers per thread) spill a few hundred bytes to local memory; the frame program's
// autotile picks 256 only for the K-heavy split-K launches, its usual tiles are 64 / 128 / 160.
template <bool PAIR>
static IgemmFn igemm_fn(int bn) {
    switch (bn) {
#define B2_IG_CASE(N) case N: if constexpr (PAIR && (N % 32)) return nullptr; else return igemm_kernel<N, PAIR>;
        B2_IG_CASE(16) B2_IG_CASE(32) B2_IG_CASE(48) B2_IG_CASE(64) B2_IG_CASE(80) B2_IG_CASE(96) B2_IG_CASE(112) B2_IG_CASE(128)
        B2_IG_CASE(144) B2_IG_CASE(160) B2_IG_CASE(176) B2_IG_CASE(192) B2_IG_CASE(208) B2_IG_CASE(224) B2_IG_CASE(240) B2_IG_CASE(256)
#undef B2_IG_CASE
        default: return nullptr;
    }
}
// IG_SILU epilogues (the ControlNet conditioning embedding: N = 16 / 32 / 96 / 256, single CTAs, N tiles <= 128) are separate
// instantiations, so the SiLU code costs the other kernels no registers (a 256-wide SiLU tile would spill)
static IgemmFn igemm_select(int bn, bool pair, bool silu, bool pad0 = false) {
    if (pad0) {
        if (pair || silu) return nullptr;
        switch (bn) {
            case 64: return igemm_pad0_kernel<64>;
            case 128: return igemm_pad0_kernel<128>;
            case 256: return igemm_pad0_kernel<256>;
            default: return nullptr;
        }
    }
    if (!silu) return pair ? igemm_fn<true>(bn) : igemm_fn<false>(bn);
    if (pair) return nullptr;
    switch (bn) {
        case 16: return igemm_kernel<16, false, true>;
        case 32: return igemm_kernel<32, false, true>;
        case 64: return igemm_kernel<64, false, true>;
        case 128: return igemm_kernel<128, false, true>;
        default: return nullptr;
    }
}

// ------------------------------------------------------------------------------------------
// host side
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (err != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
        b2_set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s",
                     cudaGetErrorString(err));
        return nullptr;
    }
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    return fn;
}

// Planning without a GPU (tests of the host logic, b2sd_igemm_plan_dry): the tensor maps are left zeroed.
static thread_local bool g_plan_dry = false;
void igemm_set_dry_run(bool on) { g_plan_dry = on; }

static int encode_act_map(CUtensorMap* m, const ActView& a, int box_c, int box_w, int box_h, int box_n,
                          int estride) {
    if (g_plan_dry) return 0;
    auto enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[4] = {(cuuint64_t)a.C, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.N};
    cuuint64_t strides[3] = {(cuuint64_t)a.ld * 2, (cuuint64_t)a.W * a.ld * 2,
                             (cuuint64_t)a.H * a.W * a.ld * 2};
    cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_n};
    cuuint32_t es[4] = {1, (cuuint32_t)estride, (cuuint32_t)estride, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(a.ptr), dims, strides,
                     box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        b2_set_error("cuTensorMapEncodeTiled(act) failed: %d (ptr %p dims %d,%d,%d,%d ld %d box "
                     "%d,%d,%d,%d es %d)",
                     (int)r, a.ptr, a.C, a.W, a.H, a.N, a.ld, box_c, box_w, box_h, box_n, estride);
        return -1;
    }
    return 0;
}

static int encode_w_map(CUtensorMap* m, const __half* w, int rows, int ld, int box_rows) {
    if (g_plan_dry) return 0;
    auto enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[2] = {(cuuint64_t)ld, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {IG_BK, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(w), dims, strides, box,
                     es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        b2_set_error("cuTensorMapEncodeTiled(weights) failed: %d (rows %d ld %d box %d)", (int)r, rows,
                     ld, box_rows);
        return -1;
    }
    return 0;
}

size_t igemm_partial_floats(int splits, long rows_total, int n_valid) {
    // worst case n_pad = n_tiles * BN < n_valid + 256
    long n_pad = ((n_valid + 255) / 256 + 1) * 256;
    return (size_t)splits * rows_total * n_pad;
}

// Swapped orientation plan: output channels on the M side (128 per CTA), a tile of BN pixels on the N side.
static int plan_swap(const IgemmDesc& d, IgemmPlan* plan) {
    IgemmParams& p = plan->p;
    if ((d.epi.flags & (IG_GEGLU | IG_PAD0)) || d.nseg < 1 || d.nseg > IG_MAX_SRC || d.epi.rowstat_out || d.epi.colsum || d.epi.out2) {
        b2_set_error("igemm(swap): unsupported (GEGLU / tap origin 0 / LayerNorm fold / row statistics / transposed V / nseg %d)", d.nseg);
        return -1;
    }
    int BN = d.BN;
    const long rows_total = (long)d.Nb * d.Ho * d.Wo;
    if (BN <= 0) BN = rows_total >= 256 ? 256 : (rows_total >= 128 ? 128 : 64);
    if (BN != 64 && BN != 128 && BN != 256) {
        b2_set_error("igemm(swap): BN %d must be 64, 128 or 256", BN);
        return -1;
    }
    p.swap = 1;
    { static const char* dm = getenv("B2_DBG_MODE"); p.dbg_mode = dm ? atoi(dm) : 0; }
    p.acc_bufs = 1;
    p.BN = BN;
    auto lg = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
    int tw, th, tn;
    if (d.Ho == 1 && d.Nb == 1) { tw = BN; th = 1; tn = 1; }
    else if (d.Wo >= 16) { tw = 16; th = BN / 16; tn = 1; }
    else { tw = 8; th = 8; tn = BN / 64; }
    p.tw = tw; p.th = th; p.tn = tn;
    p.tw_log2 = lg(tw); p.th_log2 = lg(th);
    p.tiles_w = (d.Wo + tw - 1) / tw;
    p.tiles_h = (d.Ho + th - 1) / th;
    p.tiles_n = (d.Nb + tn - 1) / tn;
    p.Wo = d.Wo; p.Ho = d.Ho; p.Nb = d.Nb;
    p.stride = d.stride < 1 ? 1 : d.stride;
    p.nseg = d.nseg;
    int total_kb = 0;
    for (int s = 0; s < d.nseg; ++s) {
        const ActView& a = d.src[s];
        if (a.C % IG_BK != 0 || (a.ld % 8) != 0 || (reinterpret_cast<uintptr_t>(a.ptr) & 15) || (d.ntap[s] != 1 && d.ntap[s] != 9)) {
            b2_set_error("igemm(swap): bad source %d", s);
            return -1;
        }
        p.seg_ntap[s] = d.ntap[s];
        p.seg_cblocks[s] = a.C / IG_BK;
        p.seg_c0[s] = 0;
        total_kb += d.ntap[s] * p.seg_cblocks[s];
        if (encode_act_map(&p.tmA[s], a, IG_BK, tw * p.stride, th * p.stride, tn, p.stride)) return -1;
    }
    p.total_kb = total_kb;
    if (d.w_ld < total_kb * IG_BK || (d.w_ld % 8) != 0 || (reinterpret_cast<uintptr_t>(d.w) & 15)) {
        b2_set_error("igemm(swap): weight ld %d < K %d or misaligned", d.w_ld, total_kb * IG_BK);
        return -1;
    }
    if (encode_w_map(&p.tmB, d.w, d.w_rows, d.w_ld, IG_BM)) return -1;
    p.a_bytes = IG_BM * IG_BK * 2;            // weight tile (lands in the A region)
    p.b_bytes = (uint32_t)BN * IG_BK * 2;     // pixel tile
    int splits = d.splits < 1 ? 1 : d.splits;
    if (splits > total_kb) splits = total_kb;
    if (splits >= 8) splits = 8; else if (splits >= 4) splits = 4; else if (splits >= 2) splits = 2;
    p.kb_per_split = (total_kb + splits - 1) / splits;
    while (splits > 1 && (total_kb + p.kb_per_split - 1) / p.kb_per_split != splits) {
        splits >>= 1;
        p.kb_per_split = (total_kb + splits - 1) / splits;
    }
    plan->splits = splits;
    plan->rows_total = rows_total;
    p.epi = d.epi;
    p.dbg_ts = d.dbg_ts;
    if (splits > 1) p.epi.flags |= IG_SPLITK;
    const int c_tiles = (d.epi.n_valid + IG_BM - 1) / IG_BM;
    p.n_pad = c_tiles * IG_BM;
    if ((d.epi.n_valid & 7) || (d.epi.ldc & 7) || (d.epi.res && (d.epi.ldr & 7)) || (d.epi.colbias && (d.epi.colbias_bstride & 3)) ||
        (reinterpret_cast<uintptr_t>(d.epi.out) & 15) || (reinterpret_cast<uintptr_t>(d.epi.res) & 15) ||
        (reinterpret_cast<uintptr_t>(d.epi.colbias) & 15)) {
        b2_set_error("igemm(swap): epilogue needs n_valid/ldc/ldr multiples of 8 and 16-byte aligned pointers");
        return -1;
    }
    const size_t stage_bytes = (size_t)IG_BM * IG_BK * 2 + (size_t)BN * IG_BK * 2;
    // swapped launches are small grids (<= ~1 CTA per SM): give the ring most of the shared memory
    static const char* sw_stage_env = getenv("B2_SWAP_STAGE_KB");
    int stages = (int)(((size_t)(sw_stage_env ? atoi(sw_stage_env) : (d.ring_kb > 0 ? d.ring_kb : 200)) * 1024) / stage_bytes);
    if (stages < 2) stages = 2;
    if (stages > IG_MAX_STAGES) stages = IG_MAX_STAGES;
    if (stages > p.kb_per_split) stages = p.kb_per_split < 2 ? 2 : p.kb_per_split;
    size_t pipe_bytes = stages * stage_bytes;
    {
        // epilogue scratch carved out of the ring: [split-K staging tile BN x 128 fp32] + transposition tile (<= 32 x 128 fp32)
        const int cols_per = BN / splits;
        const size_t need = (splits > 1 ? (size_t)BN * IG_BM * 4 : 0) + (size_t)(cols_per < SWAP_CH ? cols_per : SWAP_CH) * IG_BM * 4;
        if (need > pipe_bytes) {
            stages = (int)((need + stage_bytes - 1) / stage_bytes);
            if (stages > IG_MAX_STAGES) {
                b2_set_error("igemm(swap): split-K staging does not fit (BN %d)", BN);
                return -1;
            }
            pipe_bytes = stages * stage_bytes;
        }
    }
    p.num_stages = stages;
    plan->smem = pipe_bytes + 1024 + 512;
    uint32_t cols = 32;
    while (cols < (uint32_t)BN) cols <<= 1;
    p.tmem_cols = cols;
    plan->grid = dim3(p.tiles_w * p.tiles_h * p.tiles_n, c_tiles, splits);
    plan->mode = 0;
    return 0;
}

int b2_device_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            sms = n;
        else
            sms = IG_SMS;
        cudaGetLastError();   // no device (planning on a CPU-only machine) is not an error of the next call
    }
    return sms;
}

// CTAs of the kernel for this tile that one SM holds at once as far as registers and threads allow (the plan sizes the
// shared memory).  Dry runs do not touch the device: they assume the one CTA per SM that 288 threads at 168 registers allow.
static int igemm_ctas_per_sm(int bn, bool pair, bool silu, bool pad0) {
    if (g_plan_dry) return 1;
    IgemmFn fn = igemm_select(bn, pair, silu, pad0);
    int n = 0;
    if (fn && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, IG_THREADS, 0) == cudaSuccess && n > 0) return n;
    cudaGetLastError();
    return 1;
}

int igemm_plan(const IgemmDesc& d, IgemmPlan* plan) {
    *plan = IgemmPlan{};
    if (d.swap) return plan_swap(d, plan);
    IgemmParams& p = plan->p;
    if (d.nseg < 1 || d.nseg > IG_MAX_SRC) {
        b2_set_error("igemm: bad nseg %d", d.nseg);
        return -1;
    }
    const bool geglu = (d.epi.flags & IG_GEGLU) != 0;
    const int n_gemm = geglu ? d.epi.n_valid * 2 : d.epi.n_valid;  // GEMM N (packed weight rows used)
    // ---- N tile
    int BN = d.BN;
    if (BN <= 0) {
        if (n_gemm <= 256 && n_gemm % 16 == 0) BN = n_gemm;
        else if (n_gemm < 16) BN = 16;
        else if (n_gemm % 128 == 0) BN = 128;
        else if (n_gemm % 160 == 0) BN = 160;
        else if (n_gemm % 64 == 0) BN = 64;
        else BN = 128;
    }
    if (BN % 16 != 0 || BN < 16 || BN > 256 || (geglu && (BN % 32 != 0 || n_gemm % BN != 0))) {
        b2_set_error("igemm: unsupported BN %d (n %d)", BN, n_gemm);
        return -1;
    }
    const bool pair = d.pair != 0;
    if ((d.epi.flags & IG_SILU) && !igemm_select(BN, pair, true)) {
        b2_set_error("igemm: no SiLU-epilogue kernel for BN %d%s (16/32/64/128, single CTAs)", BN, pair ? " (CTA pair)" : "");
        return -1;
    }
    if ((d.epi.flags & IG_PAD0) && !igemm_select(BN, pair, (d.epi.flags & IG_SILU) != 0, true)) {
        b2_set_error("igemm: no tap-origin-0 kernel for BN %d%s (64/128/256, single CTAs, no SiLU)", BN, pair ? " (CTA pair)" : "");
        return -1;
    }
    if (pair && BN % 32 != 0) {
        b2_set_error("igemm(pair): BN %d must be a multiple of 32", BN);
        return -1;
    }
    p.BN = BN;
    { static const char* dm = getenv("B2_DBG_MODE"); p.dbg_mode = dm ? atoi(dm) : 0; }
    const int n_tiles = (n_gemm + BN - 1) / BN;
    if (d.w_rows < n_gemm) {
        // TMA zero-fills rows beyond w_rows; allowed (padded N) but flag obviously wrong descs
        if (d.w_rows <= 0) {
            b2_set_error("igemm: w_rows %d", d.w_rows);
            return -1;
        }
    }
    // ---- spatial tile
    int tw, th, tn;
    if (d.Ho == 1 && d.Nb == 1) {
        tw = IG_BM; th = 1; tn = 1;
    } else {
        if (d.Wo <= 16) tw = d.Wo;
        else if (d.Wo % 16 == 0) tw = 16;
        else if (d.Wo % 8 == 0) tw = 8;
        else tw = 16;
        th = IG_BM / tw;
        if (th > d.Ho) th = d.Ho;
        tn = IG_BM / (tw * th);
        if (tn > d.Nb) tn = d.Nb;
        if (tn < 1) tn = 1;
    }
    p.tw = tw; p.th = th; p.tn = tn;
    p.tiles_w = (d.Wo + tw - 1) / tw;
    p.tiles_h = (d.Ho + th - 1) / th;
    p.tiles_n = (d.Nb + tn - 1) / tn;
    p.Wo = d.Wo; p.Ho = d.Ho; p.Nb = d.Nb;
    p.stride = d.stride < 1 ? 1 : d.stride;
    if (p.stride > 2) {
        b2_set_error("igemm: stride %d", p.stride);
        return -1;
    }
    // ---- K segments + TMA maps
    p.nseg = d.nseg;
    int total_kb = 0;
    for (int s = 0; s < d.nseg; ++s) {
        const ActView& a = d.src[s];
        if (a.C % IG_BK != 0 || (a.ld % 8) != 0 || (reinterpret_cast<uintptr_t>(a.ptr) & 15)) {
            b2_set_error("igemm: source %d: C=%d must be a multiple of 64, ld=%d multiple of 8, ptr "
                         "16B aligned",
                         s, a.C, a.ld);
            return -1;
        }
        if (d.ntap[s] != 1 && d.ntap[s] != 9) {
            b2_set_error("igemm: ntap %d", d.ntap[s]);
            return -1;
        }
        p.seg_ntap[s] = d.ntap[s];
        p.seg_cblocks[s] = a.C / IG_BK;
        p.seg_c0[s] = 0;
        total_kb += d.ntap[s] * p.seg_cblocks[s];
        if (encode_act_map(&p.tmA[s], a, IG_BK, tw * p.stride, th * p.stride, tn, p.stride)) return -1;
    }
    p.total_kb = total_kb;
    if (d.w_ld < total_kb * IG_BK || (d.w_ld % 8) != 0 || (reinterpret_cast<uintptr_t>(d.w) & 15)) {
        b2_set_error("igemm: weight ld %d < K %d or misaligned", d.w_ld, total_kb * IG_BK);
        return -1;
    }
    const int b_rows = pair ? BN / 2 : BN;   // weight rows one CTA loads per K-block (pairs: multicast to both CTAs)
    if (encode_w_map(&p.tmB, d.w, d.w_rows, d.w_ld, b_rows)) return -1;
    p.a_bytes = (uint32_t)(tw * th * tn) * IG_BK * 2;
    p.b_bytes = (uint32_t)BN * IG_BK * 2;    // weight bytes landing in each CTA per K-block
    // ---- split-K
    int splits = d.splits < 1 ? 1 : d.splits;
    if (splits > total_kb) splits = total_kb;
    if (pair && splits > 4) splits = 4;   // cluster = 2 x splits CTAs, portable limit 8
    if (splits >= 8) splits = 8;        // portable cluster size; power of two so rows divide evenly
    else if (splits >= 4) splits = 4;
    else if (splits >= 2) splits = 2;
    p.kb_per_split = (total_kb + splits - 1) / splits;
    while (splits > 1 && (total_kb + p.kb_per_split - 1) / p.kb_per_split != splits) {  // keep every slice non-empty
        splits >>= 1;
        p.kb_per_split = (total_kb + splits - 1) / splits;
    }
    plan->splits = splits;
    plan->rows_total = (long)d.Nb * d.Ho * d.Wo;
    p.epi = d.epi;
    p.dbg_ts = d.dbg_ts;
    p.n_pad = n_tiles * BN;
    if (splits > 1) {
        if (geglu) {
            b2_set_error("igemm: split-K cannot be combined with GEGLU");
            return -1;
        }
        p.epi.flags |= IG_SPLITK;
    }
    // ---- pipeline depth / smem
    // one K-block (64 channels of one tap) per pipeline stage: packing several per stage was measured slower (shallower
    // prefetch, longer MMA issue code)
    const size_t stage_bytes = (size_t)IG_BM * IG_BK * 2 + (size_t)BN * IG_BK * 2;
    // The mainloop is TMA-latency bound: throughput per SM = bytes in flight / latency.  When registers admit only one CTA per
    // SM (the case of this kernel: 288 threads at up to 168 registers) the ring takes (nearly) all the shared memory; only
    // when two could be resident AND the launch needs them is the ring halved so that they fit.
    const int per_sm = igemm_ctas_per_sm(BN, pair, (d.epi.flags & IG_SILU) != 0, (d.epi.flags & IG_PAD0) != 0);
    const long resident = (long)per_sm * b2_device_sms();   // CTAs the GPU runs at once
    static const char* pc_env = getenv("B2_PERSIST_CTAS");   // tuning: CTAs of a persistent launch (default: one resident wave)
    const long persist_ctas = pc_env ? atoi(pc_env) : resident;
    const long all_tiles = (long)p.tiles_w * p.tiles_h * p.tiles_n * n_tiles;
    static const bool no_persist_e = getenv("B2_NO_PERSIST") != nullptr;
    const bool will_persist = !no_persist_e && splits == 1 && all_tiles > resident && 2 * BN <= 512;
    const long total_ctas = will_persist ? persist_ctas : all_tiles * splits;
    static const char* stage_env = getenv("B2_STAGE_KB");
    const size_t ring_budget = stage_env ? (size_t)atoi(stage_env) * 1024
                                         : (d.ring_kb > 0 ? (size_t)d.ring_kb * 1024
                                                          : (size_t)((per_sm >= 2 && total_ctas > b2_device_sms() ? 100 : 200) * 1024));
    int stages = (int)(ring_budget / stage_bytes);
    if (stages < 2) stages = 2;
    if (stages > IG_MAX_STAGES) stages = IG_MAX_STAGES;
    if (stages > p.kb_per_split) stages = p.kb_per_split < 2 ? 2 : p.kb_per_split;
    p.num_stages = stages;
    size_t pipe_bytes = stages * stage_bytes;
    if (splits > 1) {
        // the split-K staging tile [BN/4][128] float4 reuses the pipeline buffers
        const size_t stg = (size_t)BN * IG_BM * 4;
        if (stg > pipe_bytes) {
            // grow the ring rather than carving a second region (barriers live right after the ring)
            stages = (int)((stg + stage_bytes - 1) / stage_bytes);
            if (stages > IG_MAX_STAGES) {
                b2_set_error("igemm: split-K staging does not fit (BN %d)", BN);
                return -1;
            }
            p.num_stages = stages;
            pipe_bytes = stages * stage_bytes;
        }
    }
    plan->smem = pipe_bytes + 1024 /*align slack*/ + 512 /*barriers*/;
    // persistent over M tiles when the launch would need more than one resident wave
    const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
    int grid_x = m_tiles;
    p.acc_bufs = 1;
    if (will_persist) {
        grid_x = (int)(persist_ctas / n_tiles);
        if (grid_x < 1) grid_x = 1;
        if (grid_x > m_tiles) grid_x = m_tiles;
        p.acc_bufs = 2;
    }
    if (pair) {   // CTAs (2j, 2j+1) of x are a pair: an odd tile count leaves one masked tile; a persistent launch stays within
        // the resident wave (round down)
        grid_x = (p.acc_bufs == 2 && grid_x > 2) ? (grid_x & ~1) : ((grid_x + 1) & ~1);
    }
    uint32_t cols = 32;
    while (cols < (uint32_t)(BN * p.acc_bufs)) cols <<= 1;
    p.tmem_cols = cols;
    plan->grid = dim3(grid_x, n_tiles, splits);
    plan->mode = pair ? 1 : 0;
    plan->pair = pair ? 1 : 0;
    return 0;
}

int igemm_encode_act_map(CUtensorMap* m, const ActView& a, int box_c, int box_w, int box_h, int box_n, int estride) {
    return encode_act_map(m, a, box_c, box_w, box_h, box_n, estride);
}
int igemm_encode_w_map(CUtensorMap* m, const __half* w, int rows, int ld, int box_rows) { return encode_w_map(m, w, rows, ld, box_rows); }

int igemm_init() {
    static bool attr_set = false;
    if (!attr_set) {
        for (int bn = 16; bn <= 256; bn += 16) {
            for (int pair = 0; pair < 4; ++pair) {   // single CTAs, CTA pairs, single CTAs with the SiLU epilogue, tap origin 0
                IgemmFn fn = igemm_select(bn, pair == 1, pair == 2, pair == 3);
                if (!fn) continue;
                cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
                if (e != cudaSuccess) {
                    b2_set_error("cudaFuncSetAttribute(igemm BN %d%s): %s", bn, pair ? " pair" : "", cudaGetErrorString(e));
                    return -1;
                }
            }
        }
        if (!get_encode()) return -1;
        attr_set = true;
    }
    return 0;
}

int igemm_launch(const IgemmPlan& plan, cudaStream_t stream) {
    if (igemm_init()) return -1;
    const int cz = plan.splits > 1 ? plan.splits : 1;
    IgemmFn fn = igemm_select(plan.p.BN, plan.pair, (plan.p.epi.flags & IG_SILU) != 0, (plan.p.epi.flags & IG_PAD0) != 0);
    if (!fn) {
        b2_set_error("igemm launch: no kernel for BN %d%s%s%s", plan.p.BN, plan.pair ? " (CTA pair)" : "",
                     (plan.p.epi.flags & IG_SILU) ? " with the SiLU epilogue" : "", (plan.p.epi.flags & IG_PAD0) ? " with tap origin 0" : "");
        return -1;
    }
    cudaError_t e = plan.pair ? launch_kc(fn, plan.grid, dim3(IG_THREADS), plan.smem, stream, 2, cz, plan.p)
                              : launch_k(fn, plan.grid, dim3(IG_THREADS), plan.smem, stream, cz, plan.p);
    if (e != cudaSuccess) {
        b2_set_error("igemm launch: %s", cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

}  // namespace b2
