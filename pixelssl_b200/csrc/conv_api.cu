// The FFMA convolution entry points of include/pixelssl_b200.h; the wgmma kernels have entry points of their own.
#include "common.cuh"

extern "C" int pxl_conv_fp32_impl(const pxl_conv_geom*, const int*, const float*, const float*, const float*, float*, void*);
extern "C" int pxl_conv_wgrad_fp32_impl(const pxl_conv_geom*, const int*, const float*, const float*, float*, void*);

extern "C" int pxl_conv_nhwc(const pxl_conv_geom* geom, const int* taps, const float* in, const float* w,
                             const float* bias, float* out, void* stream) {
    if (!geom || geom->precision != 0) return PXL_ERR_BAD_ARG;
    return pxl_conv_fp32_impl(geom, taps, in, w, bias, out, stream);
}

extern "C" int pxl_conv_wgrad_nhwc(const pxl_conv_geom* geom, const int* taps, const float* in,
                                   const float* dy, float* dw, void* stream) {
    if (!geom || geom->precision != 0) return PXL_ERR_BAD_ARG;
    return pxl_conv_wgrad_fp32_impl(geom, taps, in, dy, dw, stream);
}

// Scratch buffers of the kernels that store per-block partials and sum them in a fixed order, one per (purpose,
// stream): launches on different streams may run at the same time and must not share one.  A buffer grows on demand;
// cudaFree synchronises the device, so a buffer is never released under a kernel that still uses it.
extern "C" void* pxl_workspace_(int purpose, void* stream, size_t bytes, int* rc) {
    struct Ent { void* stream; void* buf; size_t bytes; bool used; };
    static Ent ents[PXL_WS_PURPOSES][PXL_WS_STREAMS];
    *rc = 0;
    if (purpose < 0 || purpose >= PXL_WS_PURPOSES) { *rc = PXL_ERR_BAD_ARG; return nullptr; }
    Ent* e = nullptr;
    for (int i = 0; i < PXL_WS_STREAMS && !e; ++i)
        if (ents[purpose][i].used && ents[purpose][i].stream == stream) e = &ents[purpose][i];
    for (int i = 0; i < PXL_WS_STREAMS && !e; ++i)
        if (!ents[purpose][i].used) { e = &ents[purpose][i]; e->used = true; e->stream = stream; }
    if (!e) { *rc = PXL_ERR_UNSUPPORTED; return nullptr; }
    if (bytes > e->bytes) {
        if (e->buf) {
            cudaError_t f = cudaFree(e->buf);
            e->buf = nullptr; e->bytes = 0;
            if (f != cudaSuccess) { *rc = (int)f; return nullptr; }
        }
        cudaError_t m = cudaMalloc(&e->buf, bytes);
        if (m != cudaSuccess) { e->buf = nullptr; *rc = (int)m; return nullptr; }
        e->bytes = bytes;
    }
    return e->buf;
}
