// Canny edge detector (ControlNet processor "canny"): controlnet_aux's CannyDetector, i.e. cv2.Canny(img, low, high) with
// aperture 3 and the L1 gradient, bit for bit.  Two parts:
//   canny_head  reads the caller's frame (nearest-resized to h x w, as every input head), takes OpenCV's 3x3 Sobels of each
//               channel with replicated borders, keeps the channel of largest |dx| + |dy| (the first on ties), applies
//               OpenCV's non-maximum suppression and writes a class map: 0 none, 1 candidate (m > low), 2 strong (m > high);
//   canny_ccl   hysteresis as connected-component labelling of the candidates (8-connected), with a fixed number of launches:
//               union-find inside each tile in shared memory, union across tile borders with atomics on a global parent
//               array, each strong pixel flags its root, then each candidate reads its root's flag: 255 or 0, on 3 channels.
// The result is a set, not an order: whichever order the atomics resolve in, the same pixels are 255.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

struct CannyHeadArgs {
    const void* x;    // the caller's frame: u8 NHWC [in_h][in_w][3], or fp32 / fp16 NCHW [3][in_h][in_w] in [0, 1]
    int in_flags;     // SC_IN_U8, SC_IN_F32_NCHW or SC_IN_F16_NCHW (elementwise.cuh)
    int in_h, in_w;
    int h, w;         // the engine's size
    int low, high;    // integer thresholds (canny_thresholds)
    uint8_t* cls;     // [h][w] class map
};
int canny_head_launch(const CannyHeadArgs& a, cudaStream_t s);

struct CannyCclArgs {
    const uint8_t* cls;   // [h][w] class map of canny_head
    int* parent;          // [h][w] union-find forest (scratch)
    uint8_t* flag;        // [h][w] "the component rooted here has a strong pixel" (scratch)
    uint8_t* out;         // [h][w][3] edge image, 0 / 255
    int h, w;
};
// the four hysteresis launches in order: stage 0 local labels, 1 border merges, 2 root flags, 3 output
enum { CANNY_CCL_LOCAL = 0, CANNY_CCL_MERGE = 1, CANNY_CCL_FLAG = 2, CANNY_CCL_OUT = 3, CANNY_CCL_STAGES = 4 };
int canny_ccl_launch(const CannyCclArgs& a, int stage, cudaStream_t s);

// cv::Canny's thresholds as the kernels take them: swapped when low > high, floored, and clamped to [-1, 2041] (the L1
// magnitude of 3x3 Sobels of u8 data is at most 2040, so the clamp changes no comparison).  Finite inputs only.
void canny_thresholds(double low, double high, int* lo, int* hi);

}  // namespace b2
