// Shared helpers for the pixelssl_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/pixelssl_b200.h"

#define PXL_NUM_SMS 132

extern "C" void pxl_count_launch_(int n);

// per-(purpose, stream) scratch buffer (conv_api.cu); *rc != 0 on failure
#define PXL_WS_WGRAD 0
#define PXL_WS_BIAS 1
#define PXL_WS_CE 2
#define PXL_WS_CPS 3
#define PXL_WS_UNIMATCH 4
#define PXL_WS_STRONG_AUG 5
#define PXL_WS_OHEM 6
#define PXL_WS_DEPTHWISE 7
#define PXL_WS_PURPOSES 8
#define PXL_WS_STREAMS 8
extern "C" void* pxl_workspace_(int purpose, void* stream, size_t bytes, int* rc);

#define PXL_CHECK_LAUNCH()                                   \
    do {                                                     \
        pxl_count_launch_(1);                                \
        cudaError_t e__ = cudaPeekAtLastError();             \
        if (e__ != cudaSuccess) return (int)e__;             \
    } while (0)

static inline int64_t pxl_cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Programmatic dependent launch (PDL): a kernel launched through pxl_launch_pdl may become resident while its
// predecessor in the stream is still running (as SM resources free up); it must execute PXL_PDL_SYNC() before it
// touches global memory - the predecessor's results are complete and visible after it.  What overlaps is the launch
// latency, CTA scheduling and the part of the kernel before PXL_PDL_SYNC (barrier init, shared
// memory clearing of the wgmma kernels).  PXL_PDL=0 launches everything with plain stream order.
#define PXL_PDL_SYNC()                                                   \
    do {                                                                 \
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  \
        asm volatile("griddepcontrol.wait;" ::: "memory");               \
    } while (0)

extern "C" int pxl_pdl_enabled_(void);

template <typename... KArgs, typename... Args>
static inline cudaError_t pxl_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                         Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pxl_pdl_enabled_() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// streaming (read-once / write-once) 128-bit accesses that do not pollute L1
__device__ __forceinline__ float4 ld_stream4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream4(float* p, float4 v) {
    asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// power-of-two scale s = 2^(target_log2 - e) with amax <= 2^e: amax * s lands in (2^(target-1), 2^target]
// (fp16 pairs of gradient tensors, csrc/h16_prep.cu); 1 for a zero / non-finite absmax
__device__ __forceinline__ float pxl_pow2_scale(float amax, int target_log2) {
    if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
    int e;
    frexpf(amax, &e);
    int k = target_log2 - e;
    if (k > 126) k = 126;
    if (k < -126) k = -126;
    return ldexpf(1.f, k);
}
