// wgmma flash attention (see attention.cuh).
#include "attention.cuh"

#include <cudaTypedefs.h>
#include <math.h>
#include <string.h>

#include "igemm.cuh"  // b2_set_error
#include "launch.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b2 {

constexpr int AT_BQ = 128;      // query rows per CTA: two consumer warpgroups of 64 rows (wgmma M)
constexpr int AT_STAGES = 3;    // K/V ring depth
constexpr int AT_CONS = 256;    // warps 0-7: consumer warpgroups (MMAs, online softmax, epilogue)
constexpr int AT_THREADS = AT_CONS + 32;   // + warp 8: TMA producer
// Each consumer thread holds two query rows of its warpgroup's S = Q K^T fragment and of the O accumulator (registers).  The
// softmax numerators P are rounded to fp16 and repacked in registers as the A operand of the P.V wgmma: the m64nNk16 D
// fragment of S columns [16k, 16k+16) is exactly the A fragment of K step k, so P never touches shared memory.  Row maxima and
// sums are reduced over the 4 lanes that share a row.

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

struct AttnParams {
    CUtensorMap tmq, tmk, tmv;
    __half* out;
    int ldo;
    int sq, skv, heads, d_real;
    long k_bstride, vt_bstride;
    float scale_log2;
};

template <int DA, int BKV>
__global__ void __launch_bounds__(AT_THREADS, 1) attn_kernel(const __grid_constant__ AttnParams p) {
    constexpr int DP = DA * 64;
    constexpr int NST = AT_STAGES;
    constexpr int KVA = BKV / 64;                       // kv atoms per block (V^T tiles)
    constexpr uint32_t Q_BYTES = DA * AT_BQ * 128;      // DA atoms of [128 rows][128 B]
    constexpr uint32_t K_BYTES = DA * BKV * 128;        // DA atoms of [BKV rows][128 B]
    constexpr uint32_t V_BYTES = KVA * DP * 128;        // KVA atoms of [DP rows][128 B]
    constexpr uint32_t STAGE_BYTES = K_BYTES + V_BYTES;

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sQ = smem;
    uint8_t* sKV = sQ + Q_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + NST * STAGE_BYTES);
    uint64_t* q_full = bars;
    uint64_t* k_full = bars + 1;          // [NST]  K and V^T tiles travel through separate rings: a K slot is free as soon
    uint64_t* k_empty = k_full + NST;     // [NST]  as QK^T(j) retires, before the softmax of block j, so K(j+NST) is
    uint64_t* v_full = k_empty + NST;     // [NST]  requested a softmax earlier than the V slot of the same stage
    uint64_t* v_empty = v_full + NST;     // [NST]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ;
    const int h = blockIdx.y, b = blockIdx.z;
    const int nblk = (p.skv + BKV - 1) / BKV;

    if (threadIdx.x == AT_CONS) {
        if (smem_u32(smem) & 1023u) {
            printf("b2 attn: dynamic smem base not 1024-aligned\n");
            __trap();
        }
        tma_prefetch_desc(&p.tmq);
        tma_prefetch_desc(&p.tmk);
        tma_prefetch_desc(&p.tmv);
        mbar_init(q_full, 1);
        for (int s = 0; s < NST; ++s) {
            mbar_init(&k_full[s], 1);
            mbar_init(&k_empty[s], AT_CONS / 32);   // one arrival per consumer warp
            mbar_init(&v_full[s], 1);
            mbar_init(&v_empty[s], AT_CONS / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_launch_dependents();   // the next kernel may start its own prologue now
    pdl_wait();                // ... and everything below reads the previous kernel's output

    if (warp == AT_CONS / 32) {
        if (lane == 0) {
            // ===== TMA producer =====
            mbar_expect_tx(q_full, Q_BYTES);
#pragma unroll
            for (int a = 0; a < DA; ++a)
                tma_load_2d(sQ + a * (AT_BQ * 128), &p.tmq, q_full, h * DP + a * 64, b * p.sq + q0);
            auto load_k = [&](int j) {
                const int st = j % NST;
                mbar_wait(&k_empty[st], ((j / NST) & 1) ^ 1);
                uint8_t* sk = sKV + st * STAGE_BYTES;
                mbar_expect_tx(&k_full[st], K_BYTES);
#pragma unroll
                for (int a = 0; a < DA; ++a)
                    tma_load_2d(sk + a * (BKV * 128), &p.tmk, &k_full[st], h * DP + a * 64, (int)(b * p.k_bstride) + j * BKV);
            };
            auto load_v = [&](int j) {
                const int st = j % NST;
                mbar_wait(&v_empty[st], ((j / NST) & 1) ^ 1);
                uint8_t* sv = sKV + st * STAGE_BYTES + K_BYTES;
                mbar_expect_tx(&v_full[st], V_BYTES);
#pragma unroll
                for (int a = 0; a < KVA; ++a)
                    tma_load_2d(sv + a * (DP * 128), &p.tmv, &v_full[st], (int)(b * p.vt_bstride) + j * BKV + a * 64, h * DP);
            };
            // issue order = the order in which slots become free: K(j+1) [after QK(j+1-NST)] before V(j) [after PV(j-NST)]
            load_k(0);
            for (int j = 0; j < nblk; ++j) {
                if (j + 1 < nblk) load_k(j + 1);
                load_v(j);
            }
        }
    } else {
        // ===== consumer warpgroup wg: query rows [64 wg, 64 wg + 64) of the tile; this thread: rows rq and rq + 8 =====
        const int wg = warp >> 2;
        const int rq = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q2 = 2 * (lane & 3);
        const uint32_t sq_addr = smem_u32(sQ) + (uint32_t)wg * (64 * 128), skv_addr = smem_u32(sKV);
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        float o[DP / 2];
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
        mbar_wait(q_full, 0);
        for (int j = 0; j < nblk; ++j) {
            const int st = j % NST;
            const uint32_t ph = (uint32_t)(j / NST) & 1u;
            const uint32_t sk = skv_addr + st * STAGE_BYTES;
            // S = Q K^T
            float s[BKV / 2];
#pragma unroll
            for (int i = 0; i < BKV / 2; ++i) s[i] = 0.f;
            mbar_wait(&k_full[st], ph);
            wgmma_fence_regs(s);
            wgmma_fence();
#pragma unroll
            for (int a = 0; a < DA; ++a) {
                const uint64_t dq = make_kmajor_sw128_desc(sq_addr + a * (AT_BQ * 128));
                const uint64_t dk = make_kmajor_sw128_desc(sk + a * (BKV * 128));
#pragma unroll
                for (int k = 0; k < 4; ++k) Wgmma<BKV>::ss(s, dq + 2 * k, dk + 2 * k, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(s);
            if (lane == 0) mbar_arrive(&k_empty[st]);   // S is in registers: the K slot may be refilled
            // online softmax: block maximum, P = exp2(s*scale - m) packed as fp16 A fragments, row sums
            const int kv_valid = p.skv - j * BKV;  // columns >= kv_valid are masked
            float alpha[2], m_new[2];
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                float mx = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
                    for (int u = 0; u < 2; ++u)
                        if (8 * jj + q2 + u < kv_valid) mx = fmaxf(mx, s[4 * jj + 2 * hr + u]);
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                m_new[hr] = fmaxf(m_run[hr], mx * p.scale_log2);
                alpha[hr] = ex2_approx(m_run[hr] - m_new[hr]);
            }
            uint32_t pa[BKV / 16][4];
            float rs[2] = {0.f, 0.f};
#pragma unroll
            for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    float p0 = ex2_approx(s[4 * jj + 2 * hr] * p.scale_log2 - m_new[hr]);
                    float p1 = ex2_approx(s[4 * jj + 2 * hr + 1] * p.scale_log2 - m_new[hr]);
                    if (8 * jj + q2 >= kv_valid) p0 = 0.f;
                    if (8 * jj + q2 + 1 >= kv_valid) p1 = 0.f;
                    rs[hr] += p0 + p1;
                    pa[jj >> 1][(jj & 1) * 2 + hr] = pack_half2(p0, p1);
                }
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                l_run[hr] = l_run[hr] * alpha[hr] + rs[hr];
                m_run[hr] = m_new[hr];
            }
#pragma unroll
            for (int jj = 0; jj < DP / 8; ++jj)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    o[4 * jj + 2 * hr] *= alpha[hr];
                    o[4 * jj + 2 * hr + 1] *= alpha[hr];
                }
            // O += P V  (B = V^T tile, K-major over the kv index)
            const uint32_t sv = sk + K_BYTES;
            mbar_wait(&v_full[st], ph);
            wgmma_fence_regs(o);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < BKV / 16; ++kk) {
                const uint64_t dv = make_kmajor_sw128_desc(sv + (kk >> 2) * (DP * 128)) + 2 * (kk & 3);
                Wgmma<DP>::rs(o, pa[kk], dv, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            if (lane == 0) mbar_arrive(&v_empty[st]);
        }
        // epilogue: O / l -> fp16 -> global
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            float l = l_run[hr];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv_l = 1.0f / l;
            const int r = rq + 8 * hr;
            if (q0 + r >= p.sq) continue;
            __half* orow = p.out + ((long)b * p.sq + q0 + r) * p.ldo + h * p.d_real;
#pragma unroll
            for (int jj = 0; jj < DP / 8; ++jj) {
                const int col = 8 * jj + q2;
                if (col < p.d_real)
                    *reinterpret_cast<uint32_t*>(orow + col) = pack_half2(o[4 * jj + 2 * hr] * inv_l, o[4 * jj + 2 * hr + 1] * inv_l);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ host
static int encode_2d(CUtensorMap* m, const __half* ptr, long cols, long rows, long ld, int box_cols, int box_rows,
                     const char* what) {
    static PFN_cuTensorMapEncodeTiled_v12000 enc = nullptr;
    if (!enc) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres);
        if (err != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fp) {
            b2_set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed");
            return -1;
        }
        enc = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fp);
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(ptr), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        b2_set_error("attn: cuTensorMapEncodeTiled(%s) failed: %d (cols %ld rows %ld ld %ld box %d,%d)", what, (int)r,
                     cols, rows, ld, box_cols, box_rows);
        return -1;
    }
    return 0;
}

static size_t attn_smem_bytes(int da, int bkv) {
    const size_t q = (size_t)da * AT_BQ * 128;
    const size_t k = (size_t)da * bkv * 128;
    const size_t v = (size_t)(bkv / 64) * da * 64 * 128;
    return q + AT_STAGES * (k + v) + 256;   // + barriers
}

int attn_plan(const AttnDesc& d, AttnPlan* plan) {
    *plan = AttnPlan{};
    if (d.dp != 64 && d.dp != 128 && d.dp != 192) {
        b2_set_error("attn: padded head dim %d unsupported", d.dp);
        return -1;
    }
    if (d.d_real > d.dp || (d.d_real & 7) || (d.ldo & 7) || (d.ldq & 7) || (d.ldk & 7) || (d.ldvt & 7)) {
        b2_set_error("attn: bad dims d_real %d dp %d", d.d_real, d.dp);
        return -1;
    }
    plan->d = d;
    const int bkv = (d.dp == 192) ? 64 : 128;
    if (encode_2d(&plan->tmq, d.q, (long)d.heads * d.dp, (long)d.nb * d.sq, d.ldq, 64, AT_BQ, "q")) return -1;
    if (encode_2d(&plan->tmk, d.k, (long)d.heads * d.dp, d.k_rows, d.ldk, 64, bkv, "k")) return -1;
    if (encode_2d(&plan->tmv, d.vt, d.vt_cols, (long)d.heads * d.dp, d.ldvt, 64, d.dp, "vt")) return -1;
    plan->grid = dim3((d.sq + AT_BQ - 1) / AT_BQ, d.heads, d.nb);
    plan->smem = attn_smem_bytes(d.dp / 64, bkv);
    return 0;
}

int attn_init() {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e1 = cudaFuncSetAttribute(attn_kernel<1, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        cudaError_t e2 = cudaFuncSetAttribute(attn_kernel<2, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        cudaError_t e3 = cudaFuncSetAttribute(attn_kernel<3, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) {
            b2_set_error("cudaFuncSetAttribute(attn) failed");
            return -1;
        }
        attr_set = true;
    }
    return 0;
}

int attn_launch(const AttnPlan& plan, cudaStream_t s) {
    if (attn_init()) return -1;
    const AttnDesc& d = plan.d;
    AttnParams p;
    p.tmq = plan.tmq; p.tmk = plan.tmk; p.tmv = plan.tmv;
    p.out = d.out; p.ldo = d.ldo;
    p.sq = d.sq; p.skv = d.skv; p.heads = d.heads; p.d_real = d.d_real;
    p.k_bstride = d.k_bstride; p.vt_bstride = d.vt_bstride;
    p.scale_log2 = (float)(1.4426950408889634 / sqrt((double)d.d_real));
    cudaError_t e;
    if (d.dp == 64) e = launch_k(attn_kernel<1, 128>, plan.grid, dim3(AT_THREADS), plan.smem, s, 1, p);
    else if (d.dp == 128) e = launch_k(attn_kernel<2, 128>, plan.grid, dim3(AT_THREADS), plan.smem, s, 1, p);
    else e = launch_k(attn_kernel<3, 64>, plan.grid, dim3(AT_THREADS), plan.smem, s, 1, p);
    if (e != cudaSuccess) {
        b2_set_error("attn launch: %s", cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

}  // namespace b2
