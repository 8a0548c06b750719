// Canny edge detector kernels (see canny.cuh)
#include "canny.cuh"

#include <math.h>

#include "elementwise.cuh"   // SC_IN_*
#include "igemm.cuh"         // b2_set_error
#include "launch.cuh"

namespace b2 {

namespace {

constexpr int CY_TW = 32, CY_TH = 16;   // pixel tile of every Canny kernel: one thread per pixel, 512 threads

__device__ __forceinline__ void canny_pdl_entry() {
    pdl_launch_dependents();
    pdl_wait();
}

// one channel of the frame at engine pixel (y, x), already clamped into the image, as u8: torch's nearest index rule (as
// smallconv_kernel), and rint(clamp(v, 0, 1) * 255) for float frames, so a frame that came from u8 v / 255 gives back v
__device__ __forceinline__ void load_rgb(const CannyHeadArgs& a, int y, int x, float sy_scale, float sx_scale, uint8_t* rgb) {
    int sy = y, sx = x;
    if (a.in_h != a.h || a.in_w != a.w) {
        sy = min((int)floorf((float)y * sy_scale), a.in_h - 1);
        sx = min((int)floorf((float)x * sx_scale), a.in_w - 1);
    }
    if (a.in_flags & SC_IN_U8) {
        const uint8_t* p = static_cast<const uint8_t*>(a.x) + ((long)sy * a.in_w + sx) * 3;
        rgb[0] = p[0]; rgb[1] = p[1]; rgb[2] = p[2];
        return;
    }
    const long plane = (long)a.in_h * a.in_w, idx = (long)sy * a.in_w + sx;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = (a.in_flags & SC_IN_F32_NCHW) ? static_cast<const float*>(a.x)[c * plane + idx]
                                                      : __half2float(static_cast<const __half*>(a.x)[c * plane + idx]);
        rgb[c] = (uint8_t)__float2int_rn(fminf(fmaxf(v, 0.f), 1.f) * 255.f);   // fmaxf: NaN -> 0
    }
}

__global__ void __launch_bounds__(CY_TW * CY_TH) canny_head_kernel(CannyHeadArgs a) {
    canny_pdl_entry();
    constexpr int PW = CY_TW + 4, PH = CY_TH + 4;   // pixels: the tile with a 2-pixel halo
    constexpr int MW = CY_TW + 2, MH = CY_TH + 2;   // magnitudes: the tile with a 1-pixel halo
    __shared__ uint8_t px[PH][PW][3];
    __shared__ int mag[MH][MW];
    __shared__ short gdx[CY_TH][CY_TW], gdy[CY_TH][CY_TW];
    const int x0 = blockIdx.x * CY_TW, y0 = blockIdx.y * CY_TH;
    const int t = threadIdx.y * CY_TW + threadIdx.x;
    const float sy_scale = (float)a.in_h / (float)a.h, sx_scale = (float)a.in_w / (float)a.w;
    // replicated border (cv2.BORDER_REPLICATE): a halo pixel outside the image is its nearest pixel inside
    for (int i = t; i < PH * PW; i += CY_TW * CY_TH) {
        const int r = i / PW, c = i - r * PW;
        const int y = min(max(y0 - 2 + r, 0), a.h - 1), x = min(max(x0 - 2 + c, 0), a.w - 1);
        load_rgb(a, y, x, sy_scale, sx_scale, px[r][c]);
    }
    __syncthreads();
    // 3x3 Sobels of every channel; the channel of largest |dx| + |dy| (the first on ties, as cv::Canny on 3 channels).
    // Positions outside the image have magnitude 0 (cv::Canny's zero border of the magnitude buffer).
    for (int i = t; i < MH * MW; i += CY_TW * CY_TH) {
        const int r = i / MW, c = i - r * MW;
        const int y = y0 - 1 + r, x = x0 - 1 + c;
        int best = 0, bdx = 0, bdy = 0;
        if (y >= 0 && y < a.h && x >= 0 && x < a.w) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                // px[r + 1][c + 1] is pixel (y, x)
                const int dx = ((int)px[r][c + 2][ch] - px[r][c][ch]) + 2 * ((int)px[r + 1][c + 2][ch] - px[r + 1][c][ch]) +
                               ((int)px[r + 2][c + 2][ch] - px[r + 2][c][ch]);
                const int dy = ((int)px[r + 2][c][ch] + 2 * px[r + 2][c + 1][ch] + px[r + 2][c + 2][ch]) -
                               ((int)px[r][c][ch] + 2 * px[r][c + 1][ch] + px[r][c + 2][ch]);
                const int m = abs(dx) + abs(dy);
                if (ch == 0 || m > best) { best = m; bdx = dx; bdy = dy; }
            }
        }
        mag[r][c] = best;
        if (r >= 1 && r <= CY_TH && c >= 1 && c <= CY_TW) {
            gdx[r - 1][c - 1] = (short)bdx;
            gdy[r - 1][c - 1] = (short)bdy;
        }
    }
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int x = x0 + tx, y = y0 + ty;
    if (x >= a.w || y >= a.h) return;
    // cv::Canny's non-maximum suppression (CANNY_SHIFT 15, TG22 = round(tan 22.5deg * 2^15)): '>' against one neighbour and
    // '>=' against the other across horizontal and vertical gradients, '>' against both across diagonal ones
    constexpr int CANNY_SHIFT = 15, TG22 = 13573;
    const int r = ty + 1, c = tx + 1;
    const int m = mag[r][c];
    uint8_t cls = 0;
    if (m > a.low) {
        const int xs = gdx[ty][tx], ys = gdy[ty][tx];
        const int ax = abs(xs), ay = abs(ys) << CANNY_SHIFT;
        const int tg22x = ax * TG22;
        bool keep;
        if (ay < tg22x) {
            keep = m > mag[r][c - 1] && m >= mag[r][c + 1];
        } else {
            const int tg67x = tg22x + (ax << (CANNY_SHIFT + 1));
            if (ay > tg67x) {
                keep = m > mag[r - 1][c] && m >= mag[r + 1][c];
            } else {
                const int sgn = (xs ^ ys) < 0 ? -1 : 1;
                keep = m > mag[r - 1][c - sgn] && m > mag[r + 1][c + sgn];
            }
        }
        if (keep) cls = m > a.high ? 2 : 1;
    }
    a.cls[(long)y * a.w + x] = cls;
}

__device__ __forceinline__ int ld_parent(const int* p, int i) { return *reinterpret_cast<const volatile int*>(p + i); }

__device__ __forceinline__ int find_root(const int* parent, int i) {
    int p;
    while ((p = ld_parent(parent, i)) != i) i = p;
    return i;
}

// union of the trees of a and b: the larger root is linked below the smaller with atomicMin, retried from whatever an
// earlier link left there (every parent is <= its child, so the forest has no cycle)
__device__ __forceinline__ void unite(int* parent, int a, int b) {
    while (true) {
        a = find_root(parent, a);
        b = find_root(parent, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(parent + b, a);
        if (old == b) return;
        b = old;
    }
}

// stage 0: each tile's candidates are labelled in shared memory; every pixel's parent is its local root (global index),
// every flag cleared
__global__ void __launch_bounds__(CY_TW * CY_TH) canny_ccl_local_kernel(CannyCclArgs a) {
    canny_pdl_entry();
    __shared__ int lab[CY_TH * CY_TW];
    __shared__ uint8_t cs[CY_TH * CY_TW];
    const int tx = threadIdx.x, ty = threadIdx.y, p = ty * CY_TW + tx;
    const int x0 = blockIdx.x * CY_TW, y0 = blockIdx.y * CY_TH, x = x0 + tx, y = y0 + ty;
    const bool in = x < a.w && y < a.h;
    const long g = (long)y * a.w + x;
    const uint8_t c = in ? a.cls[g] : 0;
    lab[p] = p;
    cs[p] = c;
    __syncthreads();
    if (c) {
        // the backward half of the 8-neighbourhood inside the tile: each adjacent pair once
        if (tx > 0 && cs[p - 1]) unite(lab, p, p - 1);
        if (ty > 0) {
            if (tx > 0 && cs[p - CY_TW - 1]) unite(lab, p, p - CY_TW - 1);
            if (cs[p - CY_TW]) unite(lab, p, p - CY_TW);
            if (tx < CY_TW - 1 && cs[p - CY_TW + 1]) unite(lab, p, p - CY_TW + 1);
        }
    }
    __syncthreads();
    if (!in) return;
    const int root = find_root(lab, p);
    // local and global row-major orders agree, so parent <= child holds globally
    a.parent[g] = (y0 + root / CY_TW) * a.w + x0 + root % CY_TW;
    a.flag[g] = 0;
}

// stage 1: candidates adjacent across a tile border are united in the global forest.  Each pixel on a tile's top row,
// left or right column unites with the candidates of its backward neighbours (left, up-left, up, up-right) in other tiles.
__global__ void canny_ccl_merge_kernel(CannyCclArgs a) {
    canny_pdl_entry();
    const int x0 = blockIdx.x * CY_TW, y0 = blockIdx.y * CY_TH;
    constexpr int PERIM = CY_TW + 2 * (CY_TH - 1);
    for (int i = threadIdx.x; i < PERIM; i += blockDim.x) {
        int x, y;
        if (i < CY_TW) { x = x0 + i; y = y0; }
        else if (i < CY_TW + CY_TH - 1) { x = x0; y = y0 + 1 + (i - CY_TW); }
        else { x = x0 + CY_TW - 1; y = y0 + 1 + (i - CY_TW - (CY_TH - 1)); }
        if (x >= a.w || y >= a.h) continue;
        const int g = y * a.w + x;
        if (!a.cls[g]) continue;
        const int nx[4] = {x - 1, x - 1, x, x + 1}, ny[4] = {y, y - 1, y - 1, y - 1};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int qx = nx[k], qy = ny[k];
            if (qx < 0 || qy < 0 || qx >= a.w) continue;
            if (qx / CY_TW == x / CY_TW && qy / CY_TH == y / CY_TH) continue;   // same tile: stage 0 did it
            const int q = qy * a.w + qx;
            if (a.cls[q]) unite(a.parent, g, q);
        }
    }
}

// stage 2: every candidate points at its root directly (the forest is final: only roots are written), and a strong pixel
// flags its root
__global__ void __launch_bounds__(CY_TW * CY_TH) canny_ccl_flag_kernel(CannyCclArgs a) {
    canny_pdl_entry();
    const int x = blockIdx.x * CY_TW + threadIdx.x, y = blockIdx.y * CY_TH + threadIdx.y;
    if (x >= a.w || y >= a.h) return;
    const int g = y * a.w + x;
    const uint8_t c = a.cls[g];
    if (!c) return;
    const int root = find_root(a.parent, g);
    *reinterpret_cast<volatile int*>(a.parent + g) = root;
    if (c == 2) a.flag[root] = 1;
}

// stage 3: 255 on the candidates whose component holds a strong pixel, 0 elsewhere, replicated to 3 channels (HWC3)
__global__ void __launch_bounds__(CY_TW * CY_TH) canny_ccl_out_kernel(CannyCclArgs a) {
    canny_pdl_entry();
    const int x = blockIdx.x * CY_TW + threadIdx.x, y = blockIdx.y * CY_TH + threadIdx.y;
    if (x >= a.w || y >= a.h) return;
    const long g = (long)y * a.w + x;
    const uint8_t v = (a.cls[g] && a.flag[a.parent[g]]) ? 255 : 0;
    a.out[3 * g] = v;
    a.out[3 * g + 1] = v;
    a.out[3 * g + 2] = v;
}

}  // namespace

void canny_thresholds(double low, double high, int* lo, int* hi) {
    if (low > high) { const double t = low; low = high; high = t; }
    auto fl = [](double v) { return (int)fmin(fmax(floor(v), -1.0), 2041.0); };
    *lo = fl(low);
    *hi = fl(high);
}

int canny_head_launch(const CannyHeadArgs& a, cudaStream_t s) {
    if (!a.x || !a.cls || a.h < 1 || a.w < 1 || a.in_h < 1 || a.in_w < 1 ||
        !(a.in_flags & (SC_IN_U8 | SC_IN_F32_NCHW | SC_IN_F16_NCHW))) {
        b2_set_error("canny_head: bad arguments");
        return -1;
    }
    const dim3 grid((a.w + CY_TW - 1) / CY_TW, (a.h + CY_TH - 1) / CY_TH);
    const cudaError_t e = launch_k(canny_head_kernel, grid, dim3(CY_TW, CY_TH), 0, s, 1, a);
    if (e != cudaSuccess) {
        b2_set_error("canny_head launch: %s", cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

int canny_ccl_launch(const CannyCclArgs& a, int stage, cudaStream_t s) {
    if (!a.cls || !a.parent || !a.flag || !a.out || a.h < 1 || a.w < 1 || (long)a.h * a.w >= (1l << 31) ||
        stage < 0 || stage >= CANNY_CCL_STAGES) {
        b2_set_error("canny_ccl: bad arguments");
        return -1;
    }
    const dim3 grid((a.w + CY_TW - 1) / CY_TW, (a.h + CY_TH - 1) / CY_TH);
    cudaError_t e;
    switch (stage) {
        case CANNY_CCL_LOCAL: e = launch_k(canny_ccl_local_kernel, grid, dim3(CY_TW, CY_TH), 0, s, 1, a); break;
        case CANNY_CCL_MERGE: e = launch_k(canny_ccl_merge_kernel, grid, dim3(64), 0, s, 1, a); break;
        case CANNY_CCL_FLAG: e = launch_k(canny_ccl_flag_kernel, grid, dim3(CY_TW, CY_TH), 0, s, 1, a); break;
        default: e = launch_k(canny_ccl_out_kernel, grid, dim3(CY_TW, CY_TH), 0, s, 1, a); break;
    }
    if (e != cudaSuccess) {
        b2_set_error("canny_ccl stage %d launch: %s", stage, cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

}  // namespace b2
