// Source-index arithmetic of the bilinear resizes (csrc/resample.cu, csrc/eval_views.cu): ATen's
// area_pixel_compute_source_index, so results agree with F.interpolate to fp32 round-off.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float src_index(float scale, int dst, bool align_corners) {
    if (align_corners) return scale * (float)dst;
    float s = scale * ((float)dst + 0.5f) - 0.5f;
    return s < 0.f ? 0.f : s;
}

static inline float resize_scale(int in, int out, int align_corners) {
    if (align_corners) return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
    return (float)in / (float)out;
}
