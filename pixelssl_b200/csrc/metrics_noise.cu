// Validation metrics (confusion matrix) and the Mean-Teacher input-noise layer.
//
//   pxl_confusion_matrix  <- SemanticSegmentationFunc.metrics, task/sseg/func.py:36-48
//   pxl_gaussian_noise    <- GaussianNoiseLayer.forward, pixelssl/nn/module/gaussian_noise.py:18-41
//
// Both are HBM-bound streaming kernels; the confusion matrix is exact integer work (bit-exact
// against numpy), the noise layer uses non-contracted fp32 ops in the reference's order so that it
// is bit-exact against torch CPU fp32 for the same noise tensor.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include "common.cuh"
#include "../../include/pixelssl_b200.h"

// ------------------------------------------------------------------------------------------
// confusion matrix: cmat[gt * C + argmax_c pred] += 1 over pixels with 0 <= gt < C
// ------------------------------------------------------------------------------------------
#define CM_MAX_CLASSES 64

__global__ void __launch_bounds__(256)
confusion_kernel(const float* __restrict__ pred, const float* __restrict__ gt, int C, int64_t HW,
                 unsigned long long* __restrict__ cmat) {
    extern __shared__ unsigned int hist[];          // [C*C] per-CTA counts (< 2^32 per CTA by construction)
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    const float* pp = pred + (int64_t)b * C * HW;
    const float* gp = gt + (int64_t)b * HW;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (int64_t)gridDim.x * blockDim.x) {
        const float g = __ldg(gp + p);
        // numpy: mask = (gt >= 0) & (gt < C) on the float labels, then astype('int') truncates
        if (!(g >= 0.f && g < (float)C)) continue;
        float best = __ldg(pp + p);
        int arg = 0;
        bool nan_seen = best != best;               // np.argmax returns the first NaN
        for (int c = 1; c < C; ++c) {
            const float v = __ldg(pp + (int64_t)c * HW + p);
            if (!nan_seen && (v > best || v != v)) { best = v; arg = c; nan_seen = v != v; }
        }
        atomicAdd(hist + (int)g * C + arg, 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += blockDim.x)
        if (hist[i]) atomicAdd(cmat + i, (unsigned long long)hist[i]);
}

extern "C" int pxl_confusion_matrix(const float* pred, const float* gt, int n, int C, int64_t HW,
                                    int64_t* cmat, void* stream) {
    if (!pred || !gt || !cmat || n <= 0 || C <= 0 || HW <= 0) return PXL_ERR_BAD_ARG;
    if (C > CM_MAX_CLASSES || n > 65535) return PXL_ERR_UNSUPPORTED;
    int bx = (int)pxl_cdiv(HW, 256 * 4);
    const int cap = pxl_cdiv(PXL_NUM_SMS * 8, n) > 1 ? (int)pxl_cdiv(PXL_NUM_SMS * 8, n) : 1;
    if (bx > cap) bx = cap;
    dim3 grid((unsigned)bx, (unsigned)n);
    confusion_kernel<<<grid, 256, (size_t)C * C * sizeof(unsigned int), (cudaStream_t)stream>>>(
        pred, gt, C, HW, reinterpret_cast<unsigned long long*>(cmat));
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// Gaussian input noise: per-sample min/max -> normalise -> add noise -> clip -> de-normalise
// ------------------------------------------------------------------------------------------
#define GN_CHUNKS 64

__global__ void __launch_bounds__(256)
gn_minmax_kernel(const float* __restrict__ x, int64_t CHW, float* __restrict__ part) {
    const int b = blockIdx.y;
    const float* xp = x + (int64_t)b * CHW;
    float mn = CUDART_INF_F, mx = -CUDART_INF_F;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < CHW; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = __ldg(xp + i);
        mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
    __shared__ float smn[8], smx[8];
    mn = -warp_max(-mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 1; i < 8; ++i) { mn = fminf(mn, smn[i]); mx = fmaxf(mx, smx[i]); }
        part[((int64_t)b * GN_CHUNKS + blockIdx.x) * 2 + 0] = mn;
        part[((int64_t)b * GN_CHUNKS + blockIdx.x) * 2 + 1] = mx;
    }
}

__global__ void __launch_bounds__(256)
gn_apply_kernel(float* __restrict__ x, const float* __restrict__ noise, int64_t CHW,
                const float* __restrict__ part, int chunks) {
    const int b = blockIdx.y;
    float mn = CUDART_INF_F, mx = -CUDART_INF_F;
    for (int i = 0; i < chunks; ++i) {
        mn = fminf(mn, __ldg(part + ((int64_t)b * GN_CHUNKS + i) * 2));
        mx = fmaxf(mx, __ldg(part + ((int64_t)b * GN_CHUNKS + i) * 2 + 1));
    }
    // (imax - imin + 1e-9) evaluated in fp32 like the reference's tensor arithmetic
    const float range = __fadd_rn(__fsub_rn(mx, mn), 1e-9f);
    float* xp = x + (int64_t)b * CHW;
    const float* np_ = noise + (int64_t)b * CHW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < CHW; i += (int64_t)gridDim.x * blockDim.x) {
        float v = __fdiv_rn(__fsub_rn(xp[i], mn), range);          // inp.sub_(imin).div_(range)
        v = __fadd_rn(v, __ldg(np_ + i));                            // inp.add_(noise)
        const float ub = v > 1.f ? 1.f : 0.f;                       // upper_bound = (inp > 1).float()
        const float lb = v < 0.f ? 1.f : 0.f;                       // lower_bound from the un-clipped value
        v = __fadd_rn(__fmul_rn(v, __fsub_rn(1.f, ub)), ub);        // inp.mul_(1 - ub).add_(ub)
        v = __fmul_rn(v, __fsub_rn(1.f, lb));                       // inp.mul_(1 - lb)
        xp[i] = __fadd_rn(__fmul_rn(v, range), mn);                 // inp.mul_(range).add_(imin)
    }
}

extern "C" int64_t pxl_gaussian_noise_workspace_bytes(int n) { return (int64_t)n * GN_CHUNKS * 2 * sizeof(float); }

extern "C" int pxl_gaussian_noise(float* inp, const float* noise, int n, int64_t CHW, float* workspace,
                                  void* stream) {
    if (!inp || !noise || !workspace || n <= 0 || CHW <= 0) return PXL_ERR_BAD_ARG;
    if (n > 65535) return PXL_ERR_UNSUPPORTED;
    int chunks = (int)pxl_cdiv(CHW, 256 * 8);
    if (chunks > GN_CHUNKS) chunks = GN_CHUNKS;
    cudaStream_t st = (cudaStream_t)stream;
    gn_minmax_kernel<<<dim3((unsigned)chunks, (unsigned)n), 256, 0, st>>>(inp, CHW, workspace);
    PXL_CHECK_LAUNCH();
    int bx = (int)pxl_cdiv(CHW, 256 * 4);
    const int cap = pxl_cdiv(PXL_NUM_SMS * 8, n) > 1 ? (int)pxl_cdiv(PXL_NUM_SMS * 8, n) : 1;
    if (bx > cap) bx = cap;
    gn_apply_kernel<<<dim3((unsigned)bx, (unsigned)n), 256, 0, st>>>(inp, noise, CHW, workspace, chunks);
    PXL_CHECK_LAUNCH();
    return 0;
}
