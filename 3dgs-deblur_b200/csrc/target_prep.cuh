// Splatfacto's ground-truth preparation, shared by the loss kernels (loss.cu) and the evaluation metrics (ssim.cu) so
// that both prepare the same float target bit for bit: get_gt_img's uint8 -> float (splatfacto.py:900-910,
// `image.float() / 255.0`) and composite_with_background (:912-923, `alpha * rgb + (1 - alpha) * background`).  The
// products and the sum are the separate torch kernels of the reference, so they stay unfused (__fmul_rn / __fadd_rn).
#pragma once
#include <stdint.h>

namespace b200 {

#ifdef __CUDACC__

__device__ __forceinline__ float unit_u8(uint8_t k) { return (float)k / 255.0f; }

// the three colour channels t of an RGBA pixel with alpha `al`, composited over the background bg in place
__device__ __forceinline__ void composite_over_bg(float (&t)[3], float al, const float (&bg)[3]) {
    const float om = __fsub_rn(1.0f, al);
    t[0] = __fadd_rn(__fmul_rn(al, t[0]), __fmul_rn(om, bg[0]));
    t[1] = __fadd_rn(__fmul_rn(al, t[1]), __fmul_rn(om, bg[1]));
    t[2] = __fadd_rn(__fmul_rn(al, t[2]), __fmul_rn(om, bg[2]));
}

#endif  // __CUDACC__

}  // namespace b200
