// Epilogue helpers shared by the wgmma contraction kernels (igemm.cu, tconv.cu): accumulator fragment (registers) or staged
// fp32 row -> bias / scale / residual / ReLU / GEGLU -> fp16 NHWC stores.
#pragma once
#include "igemm.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b2 {

__device__ __forceinline__ float gelu_erf(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

__device__ __forceinline__ void store_half16(__half* dst, const float* v, int nv, bool vec_ok) {
    if (nv == 16 && vec_ok) {
        uint4 u[2];
        __half2* h = reinterpret_cast<__half2*>(u);
#pragma unroll
        for (int i = 0; i < 8; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        reinterpret_cast<uint4*>(dst)[0] = u[0];
        reinterpret_cast<uint4*>(dst)[1] = u[1];
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i)
            if (i < nv) dst[i] = __float2half_rn(v[i]);
    }
}

// LayerNorm statistics of row `orow` from the fixed-point sums its producer accumulated (see IgEpilogue)
__device__ __forceinline__ void ln_row_stats(const IgEpilogue& e, long orow, bool row_ok, float& mu, float& rstd) {
    mu = 0.f;
    rstd = 1.f;
    if (!e.rowstat_in || !row_ok) return;
    const ulonglong2 st = *reinterpret_cast<const ulonglong2*>(e.rowstat_in + 2 * orow);
    const float s1 = (float)((double)(long long)st.x * (1.0 / IG_STAT_SCALE));
    const float s2 = (float)((double)(long long)st.y * (1.0 / IG_STAT_SCALE));
    mu = s1 * e.ln_inv_c;
    const float var = fmaxf(s2 * e.ln_inv_c - mu * mu, 0.f);
    rstd = rsqrtf(var + e.ln_eps);
}
__device__ __forceinline__ void rowstat_add(const IgEpilogue& e, long orow, float s1, float s2) {
    atomicAdd(e.rowstat_out + 2 * orow, (unsigned long long)__float2ll_rn(s1 * IG_STAT_SCALE));
    atomicAdd(e.rowstat_out + 2 * orow + 1, (unsigned long long)__float2ll_rn(s2 * IG_STAT_SCALE));
}

// 16 accumulator columns [col0, col0+16) of output row `orow` (batch item b); the accumulators are
// acc[OFF .. OFF+16) of a register array (compile-time indices only: nothing may spill to local memory).
// SILU: compile the IG_SILU branch in (kernels that never see the flag leave it out: it costs registers in the wide tiles).
template <int OFF, int N, typename T, bool SILU = false>
__device__ __forceinline__ void epi_store16(const IgEpilogue& e, const T (&acc)[N], int b, long orow, int col0, float mu = 0.f,
                                            float rstd = 1.f) {
    int nv = e.n_valid - col0;
    if (nv <= 0) return;
    if (nv > 16) nv = 16;
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if constexpr (sizeof(T) == 4 && !__is_same(T, float)) v[i] = __uint_as_float(acc[OFF + i]);
        else v[i] = acc[OFF + i];
    }
    if (e.colsum) {   // folded LayerNorm of the A rows
        const float* cs = e.colsum + col0;
#pragma unroll
        for (int i = 0; i < 16; ++i)
            if (i < nv) v[i] = rstd * (v[i] - mu * cs[i]);
    }
    if (e.colbias) {
        const float* bp = e.colbias + (long)b * e.colbias_bstride + col0;
        if (nv == 16 && (e.colbias_bstride & 3) == 0) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float4 t = reinterpret_cast<const float4*>(bp)[i];
                v[4 * i + 0] += t.x; v[4 * i + 1] += t.y; v[4 * i + 2] += t.z; v[4 * i + 3] += t.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i)
                if (i < nv) v[i] += bp[i];
        }
    }
    if (e.acc_scale != 1.0f) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] *= e.acc_scale;
    }
    if (e.res) {
        const __half* rp = e.res + orow * e.ldr + col0;
        if (nv == 16 && (e.ldr & 7) == 0) {
            uint4 u[2];
            u[0] = reinterpret_cast<const uint4*>(rp)[0];
            u[1] = reinterpret_cast<const uint4*>(rp)[1];
            const __half2* h = reinterpret_cast<const __half2*>(u);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float2 f = __half22float2(h[i]);
                v[2 * i] += e.res_scale * f.x;
                v[2 * i + 1] += e.res_scale * f.y;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i)
                if (i < nv) v[i] += e.res_scale * __half2float(rp[i]);
        }
    }
    if (e.flags & IG_RELU) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.0f);
    }
    if (SILU && (e.flags & IG_SILU)) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = silu_f(v[i]);
    }
    if (e.out2 && col0 >= e.col2) {   // V block of the fused q/k/v projection: transposed store (32 lanes = 32 consecutive tokens)
        __half* tp = e.out2 + (long)(col0 - e.col2) * e.ld2 + orow;
#pragma unroll
        for (int i = 0; i < 16; ++i)
            if (i < nv) tp[(long)i * e.ld2] = __float2half_rn(v[i]);
        return;
    }
    if (e.rowstat_out) {   // statistics of the values as stored (fp16-rounded), like a LayerNorm reading them back
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i)
            if (i < nv) {
                const float x = __half2float(__float2half_rn(v[i]));
                s1 += x;
                s2 += x * x;
            }
        rowstat_add(e, orow, s1, s2);
    }
    store_half16(e.out + orow * e.ldc + col0, v, nv, (e.ldc & 7) == 0);
}

// Output row of the accumulator fragment (see wgmma.cuh): each thread holds two rows of its warpgroup's 64-row slab.
struct EpiRow {
    long orow;      // output row (pixel / token)
    int b;          // batch item (per-item bias)
    bool ok;        // inside the output
    float mu, rstd; // folded LayerNorm statistics of the A row (0 / 1 when unused)
};

__device__ __forceinline__ void store_half2(__half* dst, float x0, float x1, bool two, bool vec_ok) {
    if (two && vec_ok) {
        *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(x0, x1);
    } else {
        dst[0] = __float2half_rn(x0);
        if (two) dst[1] = __float2half_rn(x1);
    }
}

// Sum of this row's per-thread partial statistics over the 4 lanes that share it, then one fixed-point add per row.
__device__ __forceinline__ void rowstat_quad(const IgEpilogue& e, const EpiRow& rw, float s1, float s2, int lane) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
    if ((lane & 3) == 0 && rw.ok) rowstat_add(e, rw.orow, s1, s2);
}

// Epilogue of one warpgroup accumulator fragment of BN columns, straight from registers (no split-K, normal orientation):
// acc[4j + 2h + {0,1}] is row rw[h], columns gcol0 + 8j + 2 (lane % 4) + {0,1}.
//   ln_fma: LayerNorm-folded launch with vectorisable pitches: x = rstd * acc - rstd * mu * colsum + bias'
//   GEGLU: tile columns [0, BN/2) are values, [BN/2, BN) gates; out = v * gelu_erf(g)
//   otherwise: bias / scale / residual / ReLU, optional row statistics and transposed V block
template <int BN, bool SILU = false>
__device__ __forceinline__ void epi_frag(const IgEpilogue& e, const float (&acc)[BN / 2], const EpiRow (&rw)[2], int ntile,
                                         bool ln_fma, int lane) {
    const int q2 = 2 * (lane & 3);
    const bool vec_out = (e.ldc & 1) == 0;
    if (e.flags & IG_GEGLU) {
        constexpr int HALF = BN / 2;
        const int pv0 = ntile * BN, oc0 = ntile * HALF;
#pragma unroll
        for (int j = 0; j < HALF / 8; ++j) {
            const int c = 8 * j + q2;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!rw[h].ok) continue;
                float v[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    float a = acc[4 * j + 2 * h + u], g = acc[4 * (j + HALF / 8) + 2 * h + u];
                    const int pv = pv0 + c + u, pg = pv0 + HALF + c + u;
                    if (ln_fma) {
                        const float nmr = -rw[h].mu * rw[h].rstd;
                        a = fmaf(rw[h].rstd, a, fmaf(nmr, e.colsum[pv], e.colbias ? e.colbias[pv] : 0.f));
                        g = fmaf(rw[h].rstd, g, fmaf(nmr, e.colsum[pg], e.colbias ? e.colbias[pg] : 0.f));
                    } else {
                        if (e.colsum) {
                            a = rw[h].rstd * (a - rw[h].mu * e.colsum[pv]);
                            g = rw[h].rstd * (g - rw[h].mu * e.colsum[pg]);
                        }
                        if (e.colbias) {
                            a += e.colbias[pv];
                            g += e.colbias[pg];
                        }
                    }
                    v[u] = a * gelu_erf(g);
                }
                store_half2(e.out + rw[h].orow * e.ldc + oc0 + c, v[0], v[1], true, vec_out);
            }
        }
        return;
    }
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = ntile * BN + 8 * j + q2;
        if (col >= e.n_valid) continue;
        const bool two = col + 1 < e.n_valid;
        const bool transposed = e.out2 && col >= e.col2;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (!rw[h].ok) continue;
            float x[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};
            const float* bp = e.colbias ? e.colbias + (long)rw[h].b * e.colbias_bstride + col : nullptr;
            if (ln_fma) {
                const float nmr = -rw[h].mu * rw[h].rstd;
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    x[u] = fmaf(rw[h].rstd, x[u], fmaf(nmr, e.colsum[col + u], bp && (u == 0 || two) ? bp[u] : 0.f));
            } else {
                if (e.colsum) {
#pragma unroll
                    for (int u = 0; u < 2; ++u)
                        if (u == 0 || two) x[u] = rw[h].rstd * (x[u] - rw[h].mu * e.colsum[col + u]);
                }
                if (bp) {
                    x[0] += bp[0];
                    if (two) x[1] += bp[1];
                }
                if (e.acc_scale != 1.0f) {
                    x[0] *= e.acc_scale;
                    x[1] *= e.acc_scale;
                }
                if (e.res) {
                    const __half* rp = e.res + rw[h].orow * e.ldr + col;
                    if (two && (e.ldr & 1) == 0) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(rp));
                        x[0] += e.res_scale * f.x;
                        x[1] += e.res_scale * f.y;
                    } else {
                        x[0] += e.res_scale * __half2float(rp[0]);
                        if (two) x[1] += e.res_scale * __half2float(rp[1]);
                    }
                }
                if (e.flags & IG_RELU) {
                    x[0] = fmaxf(x[0], 0.f);
                    x[1] = fmaxf(x[1], 0.f);
                }
                if (SILU && (e.flags & IG_SILU)) {
                    x[0] = silu_f(x[0]);
                    x[1] = silu_f(x[1]);
                }
            }
            if (transposed) {   // V block of the fused q/k/v projection -> V^T
                __half* tp = e.out2 + (long)(col - e.col2) * e.ld2 + rw[h].orow;
                tp[0] = __float2half_rn(x[0]);
                if (two) tp[e.ld2] = __float2half_rn(x[1]);
                continue;
            }
            if (e.rowstat_out && !ln_fma) {   // statistics of the values as stored (fp16-rounded)
                const float r0 = __half2float(__float2half_rn(x[0]));
                const float r1 = two ? __half2float(__float2half_rn(x[1])) : 0.f;
                s1[h] += r0 + r1;
                s2[h] += r0 * r0 + r1 * r1;
            }
            store_half2(e.out + rw[h].orow * e.ldc + col, x[0], x[1], two, vec_out);
        }
    }
    if (e.rowstat_out && !ln_fma) {
        rowstat_quad(e, rw[0], s1[0], s2[0], lane);
        rowstat_quad(e, rw[1], s1[1], s2[1], lane);
    }
}

// Fragment -> fp32 tile in shared memory laid out [4-column group][128 rows] float4 (split-K partials: conflict-free for the
// peers' DSMEM reads), or [column][128 rows] when `colmajor` (swapped orientation: rows are output channels, columns pixels).
// r0 = this thread's first row inside the 128-row tile; only columns [c0, c0 + NC) of the fragment are written, at c - c0.
template <int BN>
__device__ __forceinline__ void frag_to_smem(float* dst, const float (&acc)[BN / 2], int r0, int lane, int c0, int nc, bool colmajor) {
    const int q2 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + q2 - c0;
        if (c < 0 || c >= nc) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            if (colmajor) {
                dst[c * 128 + r] = acc[4 * j + 2 * h];
                dst[(c + 1) * 128 + r] = acc[4 * j + 2 * h + 1];
            } else {
                *reinterpret_cast<float2*>(dst + (((c >> 2) * 128 + r) << 2) + (c & 3)) =
                    make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
}

}  // namespace b2
