// Video codec boundary of the frame path (SURVEY.md 8f-1): the aiortc fork of the reference decodes with NVDEC and encodes with
// NVENC (requirements.txt:12-13, env NVDEC / NVENC*, docs/environment.md:17-25) and hands lib/pipeline.py RGB tensors in HBM
// (lib/pipeline.py:50-51, 83, 96).  The fixed-function engines work on NV12 surfaces, so both directions need a colour
// conversion next to them:
//   nv12_to_rgb_u8   NVDEC surface (Y plane + interleaved UV plane, pitch-linear) -> u8 NHWC RGB, the frame format of b2sd_step
//   rgb_u8_to_nv12   u8 NCHW RGB (what b2sd_step writes)                          -> NV12 surface for NVENC
// BT.709 or BT.601, limited ("video") or full range, 2x2 chroma sub-sampling: the co-sited-left MPEG-2 / H.264 default is
// approximated by the box average of the four RGB-derived chroma samples (what NPP / CV-CUDA do).
// b2_codec_probe() dlopen()s libnvcuvid / libnvidia-encode; where neither is installed the session wrappers stop at
// "codec unavailable" and the synthetic feeder is the source.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

enum : int { CSC_BT709 = 0, CSC_BT601 = 1, CSC_FULL_RANGE = 2 };

int nv12_to_rgb_u8_launch(const uint8_t* y, int y_pitch, const uint8_t* uv, int uv_pitch, uint8_t* rgb_nhwc, int h, int w,
                          int flags, cudaStream_t s);
int rgb_u8_to_nv12_launch(const uint8_t* rgb_nchw, uint8_t* y, int y_pitch, uint8_t* uv, int uv_pitch, int h, int w, int flags,
                          cudaStream_t s);
// bit 0: libnvcuvid (NVDEC) loadable, bit 1: libnvidia-encode (NVENC) loadable
int codec_probe();

}  // namespace b2
