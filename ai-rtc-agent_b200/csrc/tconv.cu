// Persistent halo-tile 3x3 convolution with resident weights (see tconv.cuh).
#include "tconv.cuh"

#include <cudaTypedefs.h>
#include <stdlib.h>

#include "launch.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b2 {

constexpr uint32_t TC_WTILE = TC_C * TC_C * 2;                               // one tap's [64 x 64] fp16 weight tile
constexpr uint32_t TC_HALO_BYTES = (TC_TW + 2) * (TC_TH + 2) * TC_C * 2;     // 10 x 18 pixels x 128 B
constexpr uint32_t TC_SLAB_BYTES = 64 * TC_C * 2;                            // one 64-pixel slab of the output tile
constexpr uint32_t TC_STG_BYTES = 2 * TC_SLAB_BYTES;                         // residual / staging tile: 128 pixels x 128 B

__global__ void __launch_bounds__(TC_THREADS, 1) tconv_kernel(const __grid_constant__ TconvParams p) {
    extern __shared__ uint8_t smem_raw[];
    // aligned by an offset from smem_raw, so that the compiler still sees shared-memory pointers (LDS / STS in the epilogue)
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint8_t* sW = smem;                       // nine weight tiles, tap-major, each the canonical K-major SWIZZLE_128B tile
    uint8_t* sA = smem + 9 * TC_WTILE;        // halo ring
    uint8_t* sS = sA + (size_t)p.nbuf * p.abuf_bytes;   // one residual / staging tile per consumer warpgroup
    uint64_t* w_full = reinterpret_cast<uint64_t*>(sS + 2 * TC_STG_BYTES);
    uint64_t* a_full = w_full + 1;
    uint64_t* a_empty = a_full + TC_MAX_ABUF;
    uint64_t* r_full = a_empty + TC_MAX_ABUF;   // per warpgroup: its staging tile holds the residual (or is free, without one)

    if (threadIdx.x == TC_CONS) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        tma_prefetch_desc(&p.tmO);
        if (p.epi.res) tma_prefetch_desc(&p.tmR);
        mbar_init(w_full, 1);
        for (int s = 0; s < p.nbuf; ++s) {
            mbar_init(&a_full[s], 1);
            mbar_init(&a_empty[s], 4);   // the four warps of the warpgroup that consumed the halo
        }
        mbar_init(&r_full[0], 1);
        mbar_init(&r_full[1], 1);
        fence_mbar_init();
    }
    __syncthreads();
    // the weights are constants of the stream: request them before the programmatic-dependency wait
    if (threadIdx.x == TC_CONS) {
        mbar_expect_tx(w_full, 9 * TC_WTILE);
        for (int tap = 0; tap < 9; ++tap) tma_load_2d(sW + tap * TC_WTILE, &p.tmB, w_full, tap * TC_C, 0);
    }
    pdl_launch_dependents();
    pdl_wait();

    const int tiles_per_img = p.tiles_w * p.tiles_h;
    if (warp == TC_CONS / 32) {
        if (lane == 0) {
            // ===== halo producer: one (TH+2) x (TW+2) pixel tile per output tile =====
            int slot = 0;
            uint32_t phase = 0;
            for (int mt = blockIdx.x; mt < p.num_tiles; mt += gridDim.x) {
                const int tiw = mt % p.tiles_w, tih = (mt / p.tiles_w) % p.tiles_h, n0 = mt / tiles_per_img;
                mbar_wait(&a_empty[slot], phase ^ 1);
                mbar_expect_tx(&a_full[slot], TC_HALO_BYTES);
                tma_load_4d(sA + (size_t)slot * p.abuf_bytes, &p.tmA, &a_full[slot], 0, tiw * TC_TW - 1, tih * TC_TH - 1, n0);
                if (++slot == p.nbuf) {
                    slot = 0;
                    phase ^= 1;
                }
            }
        }
    } else {
        // ===== consumer warpgroup wg: the CTA's tiles it = wg, wg + 2, ... (all 128 pixels of each, as two M = 64 slabs, two
        // wgmma groups), so one warpgroup's epilogue overlaps the other's MMAs, and slab 0's epilogue its own slab 1 MMAs =====
        const int wg = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;   // issues this warpgroup's residual loads and output stores
        const uint32_t sa_base = smem_u32(sA);
        const uint64_t db0 = make_kmajor_sw128_desc(smem_u32(sW));
        constexpr int pitch = TC_TW + 2;   // pixels per halo row: the 8-row core groups of the A operand are `pitch` pixels apart
        const int rq = (warp & 3) * 16 + (lane >> 2);   // this thread's first row inside a 64-row slab
        const IgEpilogue& e = p.epi;
        const bool has_bias = e.colbias != nullptr, has_res = e.res != nullptr, relu = (e.flags & IG_RELU) != 0;
        // fragment columns 8j + 2 (lane % 4) + {0,1}: the same for every row, so the bias is read once
        float bias[TC_C / 4];
#pragma unroll
        for (int j = 0; j < TC_C / 8; ++j) {
            const float2 b = has_bias ? *reinterpret_cast<const float2*>(e.colbias + 8 * j + 2 * (lane & 3)) : make_float2(0.f, 0.f);
            bias[2 * j] = b.x;
            bias[2 * j + 1] = b.y;
        }
        // The staging tile is the residual box as TMA lays it out with SWIZZLE_128B: tile row r (pixel (r / 8, r % 8)) at
        // r * 128 B, its 16-byte chunk j at position j ^ (r % 8).  This thread's rows are rq + 8h (+ 64 per slab), all with
        // r % 8 == lane / 4; it reads its residual values and writes its outputs in the same place.
        uint8_t* stg = sS + wg * TC_STG_BYTES;
        uint8_t* stg_t = stg + rq * 128 + 4 * (lane & 3);
        mbar_wait(w_full, 0);
        for (int it = wg, mt = blockIdx.x + wg * gridDim.x; mt < p.num_tiles; it += 2, mt += 2 * gridDim.x) {
            const int tiw = mt % p.tiles_w, tih = (mt / p.tiles_w) % p.tiles_h, n0 = mt / tiles_per_img;
            const int slot = it % p.nbuf;
            mbar_wait(&a_full[slot], (uint32_t)(it / p.nbuf) & 1u);
            float acc[2][TC_C / 2];
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int i = 0; i < TC_C / 2; ++i) acc[m][i] = 0.f;
            wgmma_fence_regs(acc[0]);
            wgmma_fence_regs(acc[1]);
            wgmma_fence();
            // A descriptor of tap (0,0): rows r = 8*hi + wi -> halo pixel hi*pitch + wi (+ tap shift); slab m starts at hi = 8m.
            // The swizzle follows the absolute shared-memory address bits, so the 128-byte-granular tap shifts need no base offset.
            const uint32_t a0 = sa_base + (uint32_t)slot * p.abuf_bytes;
#pragma unroll
            for (int m = 0; m < 2; ++m) {
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
                    const uint64_t db = db0 + (uint64_t)(tap * (TC_WTILE >> 4));
                    const uint32_t sa = a0 + (uint32_t)((8 * m + tap / 3) * pitch + tap % 3) * 128u;   // 128 B per pixel
                    const uint64_t da = make_kmajor_sw128_desc(sa, pitch * 128);
#pragma unroll
                    for (int k = 0; k < 4; ++k) Wgmma<TC_C>::ss(acc[m], da + 2 * k, db + 2 * k, 1u);
                }
                wgmma_commit();
            }
            // while the MMAs run: once the previous tile's stores have read the staging tile, refill it with this tile's residual
            if (leader) {
                bulk_wait_group_read<0>();
                if (has_res) {
                    mbar_expect_tx(&r_full[wg], TC_STG_BYTES);
                    tma_load_4d(stg, &p.tmR, &r_full[wg], 0, tiw * TC_TW, tih * TC_TH, n0);
                } else {
                    mbar_arrive(&r_full[wg]);
                }
            }
            // ===== epilogue, slab by slab: registers (+ bias) (* acc_scale) (+ res_scale * residual) (ReLU) -> fp16 in the
            // staging tile -> TMA store (clipped at the image edge).  The fp32 operations and their order are epi_frag's. =====
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                if (m == 0) {
                    wgmma_wait<1>();
                    wgmma_fence_regs(acc[0]);
                    mbar_wait(&r_full[wg], (uint32_t)(it >> 1) & 1u);
                } else {
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc[1]);
                    if (lane == 0) mbar_arrive(&a_empty[slot]);   // the halo buffer may be refilled
                }
#pragma unroll
                for (int j = 0; j < TC_C / 8; ++j) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        __half2* sp = reinterpret_cast<__half2*>(stg_t + (64 * m + 8 * h) * 128 + ((j ^ (lane >> 2)) << 4));
                        float x0 = acc[m][4 * j + 2 * h], x1 = acc[m][4 * j + 2 * h + 1];
                        if (has_bias) {
                            x0 += bias[2 * j];
                            x1 += bias[2 * j + 1];
                        }
                        if (e.acc_scale != 1.0f) {
                            x0 *= e.acc_scale;
                            x1 *= e.acc_scale;
                        }
                        if (has_res) {
                            const float2 f = __half22float2(*sp);
                            x0 = fmaf(e.res_scale, f.x, x0);
                            x1 = fmaf(e.res_scale, f.y, x1);
                        }
                        if (relu) {
                            x0 = fmaxf(x0, 0.f);
                            x1 = fmaxf(x1, 0.f);
                        }
                        *sp = __floats2half2_rn(x0, x1);
                    }
                }
                fence_proxy_async_smem();
                named_bar_sync(1 + wg, 128);
                if (leader) {
                    tma_store_4d(&p.tmO, stg + m * TC_SLAB_BYTES, 0, tiw * TC_TW, tih * TC_TH + 8 * m, n0);
                    bulk_commit_group();
                }
            }
        }
        // the stores must be complete before the CTA retires: a programmatic dependent's wait then sees the output
        if (leader) bulk_wait_group<0>();
    }
}

// ------------------------------------------------------------------------------------------ host side
bool tconv_eligible(const IgemmDesc& d) {
    const IgEpilogue& e = d.epi;
    return d.nseg == 1 && d.ntap[0] == 9 && d.stride <= 1 && !d.swap && d.src[0].C == TC_C && e.n_valid == TC_C &&
           d.w_rows >= TC_C && d.w_ld == 9 * TC_C && d.src[0].H == d.Ho && d.src[0].W == d.Wo && d.src[0].N == d.Nb &&
           !(e.flags & (IG_GEGLU | IG_SPLITK | IG_SILU)) && !e.colsum && !e.rowstat_out && !e.out2 && !e.acc_scale_b && (e.ldc & 7) == 0 &&
           (!e.res || (e.ldr & 7) == 0) && e.colbias_bstride == 0 &&
           (d.src[0].ld & 7) == 0 && !(reinterpret_cast<uintptr_t>(d.src[0].ptr) & 15) && !(reinterpret_cast<uintptr_t>(d.w) & 15) &&
           !(reinterpret_cast<uintptr_t>(e.out) & 15) && !(reinterpret_cast<uintptr_t>(e.res) & 15) &&
           !(reinterpret_cast<uintptr_t>(e.colbias) & 15);
}

int igemm_encode_act_map(CUtensorMap* m, const ActView& a, int box_c, int box_w, int box_h, int box_n, int estride);
int igemm_encode_w_map(CUtensorMap* m, const __half* w, int rows, int ld, int box_rows);

int tconv_plan(const IgemmDesc& d, TconvPlan* plan) {
    *plan = TconvPlan{};
    if (!tconv_eligible(d)) {
        b2_set_error("tconv: needs a stride-1 3x3 convolution with 64 input and 64 output channels, 16-byte-aligned pitches and an "
                     "epilogue of a batch-shared bias / scale / residual / ReLU (no per-item scale)");
        return -1;
    }
    TconvParams& p = plan->p;
    p.tiles_w = (d.Wo + TC_TW - 1) / TC_TW;
    p.tiles_h = (d.Ho + TC_TH - 1) / TC_TH;
    p.num_tiles = p.tiles_w * p.tiles_h * d.Nb;
    p.Wo = d.Wo; p.Ho = d.Ho; p.Nb = d.Nb;
    static const char* nb_env = getenv("B2_TCONV_NBUF");
    p.nbuf = nb_env ? atoi(nb_env) : TC_MAX_ABUF;
    if (p.nbuf < 2) p.nbuf = 2;
    if (p.nbuf > TC_MAX_ABUF) p.nbuf = TC_MAX_ABUF;
    // even depth: the two warpgroups take alternate tiles, so every halo slot then belongs to one warpgroup and its phase
    // parity wait cannot be satisfied by the other warpgroup's earlier use of the slot
    p.nbuf &= ~1;
    p.abuf_bytes = (TC_HALO_BYTES + 1023u) & ~1023u;
    p.epi = d.epi;
    if (igemm_encode_act_map(&p.tmA, d.src[0], TC_C, TC_TW + 2, TC_TH + 2, 1, 1)) return -1;
    if (igemm_encode_w_map(&p.tmB, d.w, d.w_rows, d.w_ld, TC_C)) return -1;
    // output and residual: the tile's pixels without halo, in the same SWIZZLE_128B layout; stored one 8-row slab at a time
    const ActView out{d.epi.out, d.Nb, d.Ho, d.Wo, TC_C, d.epi.ldc};
    if (igemm_encode_act_map(&p.tmO, out, TC_C, TC_TW, TC_TH / 2, 1, 1)) return -1;
    if (d.epi.res) {
        const ActView res{d.epi.res, d.Nb, d.Ho, d.Wo, TC_C, d.epi.ldr};
        if (igemm_encode_act_map(&p.tmR, res, TC_C, TC_TW, TC_TH, 1, 1)) return -1;
    }
    const int sms = b2_device_sms();
    plan->grid = dim3(p.num_tiles < sms ? p.num_tiles : sms, 1, 1);
    plan->smem = 9 * (size_t)TC_WTILE + (size_t)p.nbuf * p.abuf_bytes + 2 * (size_t)TC_STG_BYTES + 1024 /*align slack*/ +
                 512 /*barriers*/;
    plan->rows_total = (long)d.Nb * d.Ho * d.Wo;
    return 0;
}

int tconv_init() {
    static bool done = false;
    if (!done) {
        cudaError_t e = cudaFuncSetAttribute(tconv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) {
            b2_set_error("cudaFuncSetAttribute(tconv): %s", cudaGetErrorString(e));
            return -1;
        }
        done = true;
    }
    return 0;
}

int tconv_launch(const TconvPlan& plan, cudaStream_t stream) {
    if (tconv_init()) return -1;
    cudaError_t e = launch_k(tconv_kernel, plan.grid, dim3(TC_THREADS), plan.smem, stream, 1, plan.p);
    if (e != cudaSuccess) {
        b2_set_error("tconv launch: %s", cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

}  // namespace b2
