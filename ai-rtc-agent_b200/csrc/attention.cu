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

// ------------------------------------------------------------------------------------------ head dim 512
// Single-head attention of the AutoencoderKL mid blocks (diffusers Attention(heads=1, dim_head=512)).  A 64-row warpgroup cannot
// hold a 512-wide fp32 O accumulator, so the output columns are split over CTAs: blockIdx.y = head * A5_SLICES + slice, and each
// CTA computes the full S = Q K^T (32 k16 steps), keeps its own online-softmax statistics and accumulates P V only for its
// 128-column slice of V^T.  S is recomputed once per slice (4x the Q K^T work, 3 x 17 GFLOP extra at 4096 tokens).  S stays in
// fp32 registers (upcast softmax); P is rounded to fp16 as the A operand of the P.V MMA, as in attn_kernel.  Warp-level
// mma.sync m16n8k16 with ldmatrix operands, cp.async double-buffered K / V^T blocks.  Every summation order is fixed, so the
// output is bit-reproducible.
constexpr int A5_D = 512;
constexpr int A5_DS = 128;                 // output columns per CTA
constexpr int A5_SLICES = A5_D / A5_DS;
constexpr int A5_BQ = 128;                 // query rows per CTA: 8 warps x 16
constexpr int A5_BKV = 32;                 // keys per block
constexpr int A5_THREADS = 256;
constexpr int A5_QP = A5_D + 8;            // smem row pitches in halves (+16 B: ldmatrix rows fall in different banks)
constexpr int A5_VP = A5_BKV + 8;
constexpr size_t A5_Q_ELEMS = (size_t)A5_BQ * A5_QP;
constexpr size_t A5_K_ELEMS = (size_t)A5_BKV * A5_QP;
constexpr size_t A5_V_ELEMS = (size_t)A5_DS * A5_VP;
constexpr size_t A5_SMEM = (A5_Q_ELEMS + 2 * (A5_K_ELEMS + A5_V_ELEMS)) * 2;

struct Attn512Params {
    const __half* q; const __half* k; const __half* vt;
    __half* out;
    int ldq, ldk, ldvt, ldo;
    int sq, skv;
    long k_bstride, vt_bstride;
    float scale_log2;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(A5_THREADS, 1) attn_d512_kernel(const __grid_constant__ Attn512Params p) {
    extern __shared__ __align__(128) __half sm5[];
    __half* sQ = sm5;
    __half* sK = sQ + A5_Q_ELEMS;                 // [2][A5_BKV][A5_QP]
    __half* sV = sK + 2 * A5_K_ELEMS;             // [2][A5_DS][A5_VP]: V^T rows (output columns) x keys
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * A5_BQ;
    const int head = blockIdx.y / A5_SLICES, slice = blockIdx.y % A5_SLICES;
    const int b = blockIdx.z;
    const int col0 = head * A5_D;
    const int nblk = (p.skv + A5_BKV - 1) / A5_BKV;
    const __half* qb = p.q + (long)b * p.sq * p.ldq + col0;
    const __half* kb = p.k + b * p.k_bstride * p.ldk + col0;
    const __half* vb = p.vt + (long)(col0 + slice * A5_DS) * p.ldvt + b * p.vt_bstride;

    pdl_launch_dependents();
    pdl_wait();

    // rows / keys past the end are zero-filled (cp.async src-size 0), so no value outside the operands enters an MMA
    for (int i = tid; i < A5_BQ * (A5_D / 8); i += A5_THREADS) {
        const int r = i / (A5_D / 8), c = (i % (A5_D / 8)) * 8;
        const bool ok = q0 + r < p.sq;
        cp_async16(smem_u32(sQ + r * A5_QP + c), ok ? qb + (long)(q0 + r) * p.ldq + c : qb, ok ? 16 : 0);
    }
    auto load_kv = [&](int j, int buf) {
        __half* sk = sK + buf * A5_K_ELEMS;
        __half* sv = sV + buf * A5_V_ELEMS;
        const int kv0 = j * A5_BKV;
        for (int i = tid; i < A5_BKV * (A5_D / 8); i += A5_THREADS) {
            const int r = i / (A5_D / 8), c = (i % (A5_D / 8)) * 8;
            const bool ok = kv0 + r < p.skv;
            cp_async16(smem_u32(sk + r * A5_QP + c), ok ? kb + (long)(kv0 + r) * p.ldk + c : kb, ok ? 16 : 0);
        }
        for (int i = tid; i < A5_DS * (A5_BKV / 8); i += A5_THREADS) {
            const int r = i / (A5_BKV / 8), c = (i % (A5_BKV / 8)) * 8;
            const int valid = p.skv - (kv0 + c);
            const int bytes = valid >= 8 ? 16 : (valid > 0 ? 2 * valid : 0);
            cp_async16(smem_u32(sv + r * A5_VP + c), bytes ? vb + (long)r * p.ldvt + kv0 + c : vb, bytes);
        }
    };
    load_kv(0, 0);
    cp_async_commit();

    const int r_lo = lane >> 2, q2 = 2 * (lane & 3);
    float o[A5_DS / 8][4];
#pragma unroll
    for (int n = 0; n < A5_DS / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    // ldmatrix lane addresses: A (16x16, row-major Q) and B (two n8 tiles x k16 from [n][k] rows: K, V^T)
    const uint32_t a_base = smem_u32(sQ + (warp * 16 + (lane & 15)) * A5_QP + (lane >> 4) * 8);
    const int b_row = (lane & 7) + ((lane >> 4) << 3), b_col = ((lane >> 3) & 1) * 8;

    for (int j = 0; j < nblk; ++j) {
        const int buf = j & 1;
        if (j + 1 < nblk) {
            load_kv(j + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        // S = Q K^T for this warp's 16 rows x A5_BKV keys
        float s[A5_BKV / 8][4];
#pragma unroll
        for (int n = 0; n < A5_BKV / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
        const uint32_t k_base = smem_u32(sK + buf * A5_K_ELEMS + b_row * A5_QP + b_col);
#pragma unroll 4
        for (int kk = 0; kk < A5_D / 16; ++kk) {
            uint32_t a[4];
            ldsm_x4(a_base + kk * 32, a[0], a[1], a[2], a[3]);
#pragma unroll
            for (int np = 0; np < A5_BKV / 16; ++np) {
                uint32_t b0, b1, b2, b3;
                ldsm_x4(k_base + (np * 16 * A5_QP) * 2 + kk * 32, b0, b1, b2, b3);
                mma16816(s[2 * np], a, b0, b1);
                mma16816(s[2 * np + 1], a, b2, b3);
            }
        }
        // online softmax over the valid keys (columns >= kv_valid are masked)
        const int kv_valid = p.skv - j * A5_BKV;
        float alpha[2], m_new[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            float mx = -INFINITY;
#pragma unroll
            for (int n = 0; n < A5_BKV / 8; ++n)
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (8 * n + q2 + u < kv_valid) mx = fmaxf(mx, s[n][2 * hr + u]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            m_new[hr] = fmaxf(m_run[hr], mx * p.scale_log2);
            alpha[hr] = ex2_approx(m_run[hr] - m_new[hr]);
        }
        uint32_t pa[A5_BKV / 16][4];
        float rs[2] = {0.f, 0.f};
#pragma unroll
        for (int n = 0; n < A5_BKV / 8; ++n)
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                float p0 = ex2_approx(s[n][2 * hr] * p.scale_log2 - m_new[hr]);
                float p1 = ex2_approx(s[n][2 * hr + 1] * p.scale_log2 - m_new[hr]);
                if (8 * n + q2 >= kv_valid) p0 = 0.f;
                if (8 * n + q2 + 1 >= kv_valid) p1 = 0.f;
                rs[hr] += p0 + p1;
                pa[n >> 1][(n & 1) * 2 + hr] = pack_half2(p0, p1);
            }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            l_run[hr] = l_run[hr] * alpha[hr] + rs[hr];
            m_run[hr] = m_new[hr];
        }
#pragma unroll
        for (int n = 0; n < A5_DS / 8; ++n) {
            o[n][0] *= alpha[0]; o[n][1] *= alpha[0];
            o[n][2] *= alpha[1]; o[n][3] *= alpha[1];
        }
        // O += P V over this CTA's column slice (B = V^T rows, keys contiguous)
        const uint32_t v_base = smem_u32(sV + buf * A5_V_ELEMS + b_row * A5_VP + b_col);
#pragma unroll
        for (int t = 0; t < A5_BKV / 16; ++t)
#pragma unroll
            for (int np = 0; np < A5_DS / 16; ++np) {
                uint32_t b0, b1, b2, b3;
                ldsm_x4(v_base + (np * 16 * A5_VP) * 2 + t * 32, b0, b1, b2, b3);
                mma16816(o[2 * np], pa[t], b0, b1);
                mma16816(o[2 * np + 1], pa[t], b2, b3);
            }
        __syncthreads();   // every warp is done with this buffer before the next iteration refills it
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        float l = l_run[hr];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv_l = 1.0f / l;
        const int r = q0 + warp * 16 + r_lo + 8 * hr;
        if (r >= p.sq) continue;
        __half* orow = p.out + ((long)b * p.sq + r) * p.ldo + col0 + slice * A5_DS;
#pragma unroll
        for (int n = 0; n < A5_DS / 8; ++n)
            *reinterpret_cast<uint32_t*>(orow + 8 * n + q2) = pack_half2(o[n][2 * hr] * inv_l, o[n][2 * hr + 1] * inv_l);
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
    if (d.dp == A5_D) {   // attn_d512_kernel: plain pointers (cp.async), no tensor maps
        const auto misaligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) != 0; };
        if (d.d_real != A5_D || (d.ldq & 7) || (d.ldk & 7) || (d.ldvt & 7) || (d.ldo & 7) || (d.vt_bstride & 7) ||
            misaligned(d.q) || misaligned(d.k) || misaligned(d.vt) || misaligned(d.out) || d.sq < 1 || d.skv < 1) {
            b2_set_error("attn(d512): needs d_real 512, row pitches and the V^T batch stride multiples of 8, 16-byte aligned "
                         "pointers (d_real %d ldq %d ldk %d ldvt %d ldo %d vt_bstride %ld)", d.d_real, d.ldq, d.ldk, d.ldvt, d.ldo,
                         d.vt_bstride);
            return -1;
        }
        plan->d = d;
        plan->grid = dim3((d.sq + A5_BQ - 1) / A5_BQ, d.heads * A5_SLICES, d.nb);
        plan->smem = A5_SMEM;
        return 0;
    }
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
        cudaError_t e4 = cudaFuncSetAttribute(attn_d512_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)A5_SMEM);
        if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess || e4 != cudaSuccess) {
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
    if (d.dp == A5_D) {
        Attn512Params q5;
        q5.q = d.q; q5.k = d.k; q5.vt = d.vt; q5.out = d.out;
        q5.ldq = d.ldq; q5.ldk = d.ldk; q5.ldvt = d.ldvt; q5.ldo = d.ldo;
        q5.sq = d.sq; q5.skv = d.skv; q5.k_bstride = d.k_bstride; q5.vt_bstride = d.vt_bstride;
        q5.scale_log2 = (float)(1.4426950408889634 / sqrt((double)d.d_real));
        const cudaError_t e5 = launch_k(attn_d512_kernel, plan.grid, dim3(A5_THREADS), plan.smem, s, 1, q5);
        if (e5 != cudaSuccess) {
            b2_set_error("attn(d512) launch: %s", cudaGetErrorString(e5));
            return -1;
        }
        return 0;
    }
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
