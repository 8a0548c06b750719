// Flash-style attention on wgmma: S = Q K^T and O += P V as warpgroup MMAs with the accumulators in
// registers, online softmax on the S fragment, P kept in registers as the A operand of the P.V MMA.
// Self-attention (seq 64..9216) and
// cross-attention against the cached prompt K/V (77 keys) use the same kernel.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace b2 {

struct AttnDesc {
    const __half* q;    // [nb*sq][ldq], head h occupies columns [h*dp, h*dp+dp)
    int ldq;
    const __half* k;    // [rows][ldk], same head layout; batch b starts at row b*k_bstride
    int ldk;
    long k_bstride;     // rows; 0 => K/V shared by every batch item (prompt cache)
    long k_rows;        // total rows addressable
    const __half* vt;   // V^T: [heads*dp][ldvt], kv index contiguous; batch b starts at column b*vt_bstride
    int ldvt;
    long vt_bstride;
    long vt_cols;       // total valid columns
    __half* out;        // [nb*sq][ldo], head h occupies columns [h*d_real, (h+1)*d_real)
    int ldo;
    int nb, heads, sq, skv;
    int d_real;         // true head dim (softmax scale = d_real^-0.5)
    int dp;             // padded head dim: 64, 128 or 192 (zero-padded columns)
    // Decoupled image segment (IP-Adapter), all null = none: out = softmax(Q K^T) V + softmax(Q Kip^T) Vip, the second
    // softmax over the first *n_ip keys (device int, 0..64; 0 skips the segment).  Shared by every batch item.  The caller
    // allocates full 64-key blocks with zeroed padding: k_ip [64][ldk] (head layout of k), vt_ip [heads*dp][64].  An image
    // scale is folded into vt_ip.
    const __half* k_ip;
    const __half* vt_ip;
    const int* n_ip;
};

constexpr int ATTN_IP_KEYS = 64;   // keys of the image segment's block (the most n_ip may be)

struct AttnPlan {
    CUtensorMap tmq, tmk, tmv;
    CUtensorMap tmk_ip, tmv_ip;   // the image segment's (AttnDesc::n_ip set)
    AttnDesc d;
    dim3 grid;
    size_t smem;
};

int attn_plan(const AttnDesc& d, AttnPlan* plan);
int attn_launch(const AttnPlan& plan, cudaStream_t s);
int attn_init();

}  // namespace b2
