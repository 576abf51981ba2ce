// fp16 "pairs": the operand format of the wgmma f16 convolutions (conv_tc.cu, precision 3 / 4).
//
//   t  = x * s                 s = a power of two (exact), per tensor
//   hi = fp16_rn(t)            11 significant bits
//   lo = fp16_rn(t - hi)       the next 11 bits (t - hi is exact in fp32)
//
// so x*s = hi + lo up to max(2^-22 |t|, 2^-25): with hi*hi + lo*hi + hi*lo accumulated in fp32 a product
// carries a relative error of ~2^-21, the level of the 3xTF32 path, at twice its MMA rate and with no in-kernel
// operand transform; hi alone has the 11-bit significand of TF32.  fp16's narrow exponent is what the scale is
// for: activations and weights use fixed powers of two chosen by the caller, gradients a per-tensor scale derived
// on the device from the tensor's absmax (pxl_h16_absmax + the DYN path below).  Values that still leave the fp16
// range saturate at +-65504 and are counted: pxl_h16_status() != 0 means some operand lost information.
#include "common.cuh"
#include <cuda_fp16.h>

// saturation events per producer site: [0] pxl_h16_split fixed scale, [1] pxl_h16_split dynamic scale,
// [2] BatchNorm apply (activations), [3] BatchNorm backward dx (gradients)
static int* g_sat_counter = nullptr;

extern "C" int* pxl_h16_sat_counter(void) {
    if (!g_sat_counter) {
        if (cudaMalloc(&g_sat_counter, 4 * sizeof(int)) != cudaSuccess) return nullptr;
        cudaMemset(g_sat_counter, 0, 4 * sizeof(int));
    }
    return g_sat_counter;
}

extern "C" int pxl_h16_status_sites(int* out4_host) {
    for (int i = 0; i < 4; ++i) out4_host[i] = 0;
    if (!g_sat_counter) return 0;
    return cudaMemcpy(out4_host, g_sat_counter, 4 * sizeof(int), cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

extern "C" int pxl_h16_status(void) {
    int v[4];
    if (pxl_h16_status_sites(v) != 0) return -1;
    long long t = (long long)v[0] + v[1] + v[2] + v[3];
    return t > 0x7fffffff ? 0x7fffffff : (int)t;
}

extern "C" int pxl_h16_reset_status(void) {
    if (g_sat_counter) cudaMemset(g_sat_counter, 0, 4 * sizeof(int));
    return 0;
}

// slot layout (4 floats): [0] s, [1] 1/s, [2] absmax as uint bits (atomicMax target), [3] unused
// s = pxl_pow2_scale(absmax, target_log2): absmax * s lands in (2^(target-1), 2^target]
template <bool DYN>
__global__ void __launch_bounds__(256)
h16_split_kernel(const float4* __restrict__ x, uint2* __restrict__ hi, uint2* __restrict__ lo, int64_t n4,
                 float scale, float* __restrict__ slot, int target_log2, int* __restrict__ sat) {
    float s = scale;
    if (DYN) {
        s = pxl_pow2_scale(__uint_as_float(((const unsigned*)slot)[2]), target_log2);
        if (blockIdx.x == 0 && threadIdx.x == 0) { slot[0] = s; slot[1] = 1.f / s; }
    }
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    bool clipped = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 v = __ldcs(x + i);
        const float t[4] = {v.x * s, v.y * s, v.z * s, v.w * s};
        __half h[4], l[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float c = fminf(fmaxf(t[k], -65504.f), 65504.f);
            clipped |= (c != t[k]) && (t[k] == t[k]);
            h[k] = __float2half_rn(c);
            l[k] = __float2half_rn(c - __half2float(h[k]));
        }
        uint2 ph, pl;
        ph.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
        ph.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
        hi[i] = ph;
        if (lo) {
            pl.x = (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16);
            pl.y = (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16);
            lo[i] = pl;
        }
    }
    if (clipped && sat) atomicAdd(sat, 1);
}

// x -> (hi, lo) with a fixed scale (slot == NULL) or with the scale derived from slot[2] = absmax bits
// (pxl_h16_absmax must have run on the same stream); lo nullable (precision 4 only reads hi); n % 4 == 0.
extern "C" int pxl_h16_split(const float* x, void* hi, void* lo, int64_t n, float scale, float* slot, int target_log2,
                             void* stream) {
    if (!x || !hi || n <= 0 || (n & 3)) return PXL_ERR_BAD_ARG;
    if (!slot && !(scale > 0.f)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = n / 4;
    int blocks = (int)(pxl_cdiv(n4, 256 * 2) < PXL_NUM_SMS * 8 ? pxl_cdiv(n4, 256 * 2) : PXL_NUM_SMS * 8);
    int* sat = pxl_h16_sat_counter();
    if (slot) h16_split_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (uint2*)hi, (uint2*)lo, n4, 1.f, slot, target_log2, sat ? sat + 1 : sat);
    else h16_split_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (uint2*)hi, (uint2*)lo, n4, scale, nullptr, 0, sat);
    PXL_CHECK_LAUNCH();
    return 0;
}

__global__ void __launch_bounds__(256)
h16_absmax_kernel(const float4* __restrict__ x, int64_t n4, float* __restrict__ slot) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 v = __ldg(x + i);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    m = warp_max(m);
    __shared__ float sm[8];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = threadIdx.x < 8 ? sm[threadIdx.x] : 0.f;
        m = warp_max(m);
        if (threadIdx.x == 0 && m > 0.f) atomicMax((unsigned*)slot + 2, __float_as_uint(m));   // non-negative floats order like uints
    }
}

// slot[2] = max(slot[2], absmax(x)) (bit pattern); the slot must have been zeroed by the caller
extern "C" int pxl_h16_absmax(const float* x, int64_t n, float* slot, void* stream) {
    if (!x || !slot || n <= 0 || (n & 3)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = n / 4;
    int blocks = (int)(pxl_cdiv(n4, 256 * 4) < PXL_NUM_SMS * 4 ? pxl_cdiv(n4, 256 * 4) : PXL_NUM_SMS * 4);
    h16_absmax_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)x, n4, slot);
    PXL_CHECK_LAUNCH();
    return 0;
}
