// ASPP head (Classifier_Module.forward, task/sseg/module/deeplab_v2.py:81-85: the sum of four dilated 3x3
// convolutions 2048 -> C) as ONE dense GEMM plus a gather.
//
// A 36-tap convolution with C = 21 output channels re-reads the 2048-channel latent once per tap and feeds the tensor
// core N = 32 wide tiles: traffic-bound at a few percent of the MMA rate.  Convolution is linear, so the taps can be
// applied AFTER the channel contraction:
//     Z[p, t, co] = sum_ci W_t[co, ci] * x[p, ci]            one 1x1 GEMM, N = 36*C (756 -> 768), x read once
//     out[p, co]  = bias[co] + sum_t Z[p + off_t, t, co]     this file: a 36-term gather over a 53 MB tensor
// and backwards with dZ[q, t, co] = dY[q - off_t, co]:  dX = dZ * W'^T (K = 768) and dW' = dZ^T * X (plain 1x1 wgrad).
// The two kernels here are the gather (forward) and the scatter of dY into the fp16 pair of dZ (backward); both are
// tiny next to the GEMMs.
#include "common.cuh"
#include <cuda_fp16.h>

struct AsppTaps { int n; short dy[PXL_MAX_TAPS], dx[PXL_MAX_TAPS]; };

__global__ void __launch_bounds__(256)
aspp_gather_kernel(const float* __restrict__ Z, const float* __restrict__ bias, float* __restrict__ out,
                   int N, int H, int W, int C, int ldz, int ldo, AsppTaps taps) {
    const int64_t total = (int64_t)N * H * W * ldo;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int co = (int)(i % ldo);
        const int64_t p = i / ldo;
        if (co >= C) { out[i] = 0.f; continue; }
        const int px = (int)(p % W), py = (int)((p / W) % H);
        const int64_t nbase = (p / ((int64_t)W * H)) * H;
        float acc = bias ? __ldg(bias + co) : 0.f;
        for (int t = 0; t < taps.n; ++t) {
            const int y = py + taps.dy[t], x = px + taps.dx[t];
            if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W)
                acc += __ldg(Z + ((nbase + y) * W + x) * ldz + t * C + co);
        }
        out[i] = acc;
    }
}

// out [N,H,W,ldo] (lanes >= C zero) = bias + sum over taps of Z [N,H,W,ldz] at channel t*C + co, zero padding
extern "C" int pxl_aspp_gather(const float* Z, const float* bias, float* out, int N, int H, int W, int C, int ldz, int ldo,
                               const int* taps_dydx_host, int ntaps, void* stream) {
    if (!Z || !out || !taps_dydx_host || N <= 0 || H <= 0 || W <= 0 || C <= 0 || ntaps <= 0 || ntaps > PXL_MAX_TAPS ||
        ntaps * C > ldz || C > ldo)
        return PXL_ERR_BAD_ARG;
    AsppTaps t;
    t.n = ntaps;
    for (int k = 0; k < ntaps; ++k) { t.dy[k] = (short)taps_dydx_host[2 * k]; t.dx[k] = (short)taps_dydx_host[2 * k + 1]; }
    const int64_t total = (int64_t)N * H * W * ldo;
    int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 16 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 16);
    aspp_gather_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(Z, bias, out, N, H, W, C, ldz, ldo, t);
    PXL_CHECK_LAUNCH();
    return 0;
}

__global__ void __launch_bounds__(256)
aspp_scatter_h16_kernel(const float* __restrict__ dy, __half* __restrict__ hi, __half* __restrict__ lo,
                        float* __restrict__ slot, int target_log2, int N, int H, int W, int C, int ldy, int ldz,
                        AsppTaps taps, int* __restrict__ sat) {
    const float s = pxl_pow2_scale(__uint_as_float(((const unsigned*)slot)[2]), target_log2);
    if (blockIdx.x == 0 && threadIdx.x == 0) { slot[0] = s; slot[1] = 1.f / s; }
    const int64_t total = (int64_t)N * H * W * ldz;
    bool clipped = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int zc = (int)(i % ldz);
        const int64_t q = i / ldz;
        float v = 0.f;
        if (zc < taps.n * C) {
            const int t = zc / C, co = zc - t * C;
            const int qx = (int)(q % W), qy = (int)((q / W) % H);
            const int y = qy - taps.dy[t], x = qx - taps.dx[t];
            if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W)
                v = __ldg(dy + (((q / ((int64_t)W * H)) * H + y) * W + x) * ldy + co) * s;
        }
        const float c = fminf(fmaxf(v, -65504.f), 65504.f);
        clipped |= (c != v) && (v == v);
        const __half h = __float2half_rn(c);
        hi[i] = h;
        if (lo) lo[i] = __float2half_rn(c - __half2float(h));
    }
    if (clipped && sat) atomicAdd(sat, 1);
}

// dZ [N,H,W,ldz] as an fp16 pair (lo nullable): dZ[q, t*C + co] = dy[q - off_t, co] (zero outside the image and for
// channels >= ntaps*C); scale from slot[2] = absmax(dy) bits (pxl_h16_absmax), s / 1/s stored in slot[0..1]
extern "C" int pxl_aspp_scatter_h16(const float* dy, void* hi, void* lo, float* slot, int target_log2, int N, int H, int W,
                                    int C, int ldy, int ldz, const int* taps_dydx_host, int ntaps, void* stream) {
    if (!dy || !hi || !slot || !taps_dydx_host || N <= 0 || H <= 0 || W <= 0 || C <= 0 || ntaps <= 0 || ntaps > PXL_MAX_TAPS ||
        ntaps * C > ldz || C > ldy)
        return PXL_ERR_BAD_ARG;
    AsppTaps t;
    t.n = ntaps;
    for (int k = 0; k < ntaps; ++k) { t.dy[k] = (short)taps_dydx_host[2 * k]; t.dx[k] = (short)taps_dydx_host[2 * k + 1]; }
    const int64_t total = (int64_t)N * H * W * ldz;
    int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 16 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 16);
    int* sat = pxl_h16_sat_counter();
    aspp_scatter_h16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dy, (__half*)hi, (__half*)lo, slot, target_log2, N, H, W, C,
                                                                       ldy, ldz, t, sat ? sat + 1 : sat);
    PXL_CHECK_LAUNCH();
    return 0;
}
