// Depthwise 3x3 convolution (groups = C, bias-free) on NHWC fp32 activations with ld lanes: the per-channel half of
// Xception's separable convolutions.  Stride 1 with dilation d >= 1, or stride 2 with dilation 1; padding d on every
// side, so OH = (H - 1) / stride + 1.  Lanes c >= C of every output are written as exact zeros, and no kernel reads
// outside its tensors.
//
// The work is ~9 FMAs per 8 bytes moved, so it is bandwidth-bound: plain FFMA fp32 in every precision mode, channels
// vectorised as float4 across lanes (a warp reads 512 contiguous bytes of one pixel per tap), the 9 weights of a
// thread's 4 channels in registers for a run of DW_PIX output pixels.  The input window is not staged through shared
// memory: neighbouring threads' taps hit the same lines, which L1 / L2 serve.
//
// forward: y[n,oy,ox,c] = sum_t w[c,t] x[n, oy*s + (r-1)*d, ox*s + (u-1)*d, c]   (t = r*3 + u, taps in order)
// dgrad:   dx[n,iy,ix,c] = sum_t w[c,t] dy[n, (iy + d - r*d) / s, ...]  - a gather over the output pixels a tap of
//          the input pixel reaches; at stride 2 only the taps whose offset has the pixel's parity contribute (the
//          parity classes of the dense convolutions' stride-2 dgrad), checked per pixel, so nothing is scattered.
// wgrad:   dw[c,t] = sum_pixels x * dy: each block accumulates a chunk of output pixels in fp32 per thread, reduces its
//          threads in a fixed order in fp64 into its own slot of a per-stream workspace (PXL_WS_DEPTHWISE), and a
//          second launch adds the chunks in chunk order.  No floating-point atomics: repeated calls are bit-identical.
#include "common.cuh"

#define DW_THREADS 256
#define DW_PIX 4              // output pixels per thread of the gather kernels
#define DW_WG_QB 32           // wgrad: channel quads per block (x), DW_THREADS / DW_WG_QB pixel lanes (y)
#define DW_WG_BLOCKS (4 * PXL_NUM_SMS)

__device__ __forceinline__ float4 dw_fma4(float4 w, float4 v, float4 a) {
    a.x = fmaf(w.x, v.x, a.x); a.y = fmaf(w.y, v.y, a.y); a.z = fmaf(w.z, v.z, a.z); a.w = fmaf(w.w, v.w, a.w);
    return a;
}

// forward (DGRAD false): out = y over [N,OH,OW], in = x over [N,IH,IW] with IH = H.
// dgrad (DGRAD true): out = dx over [N,OH,OW] = [N,H,W], in = dy over [N,IH,IW] = the forward's output size.
template <int S, bool DGRAD>
__global__ void __launch_bounds__(DW_THREADS) dw_gather_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                               float* __restrict__ out, int N, int IH, int IW, int OH,
                                                               int OW, int C, int ld, int d, int64_t nruns) {
    const int Q = ld >> 2;
    const int64_t idx = (int64_t)blockIdx.x * DW_THREADS + threadIdx.x;
    if (idx >= nruns * Q) return;
    const int q = (int)(idx % Q);
    const int64_t run = idx / Q;
    const int64_t P = (int64_t)N * OH * OW;
    const int c0 = q * 4;
    if (c0 >= C) {
        for (int k = 0; k < DW_PIX; ++k) {
            const int64_t p = run * DW_PIX + k;
            if (p < P) *reinterpret_cast<float4*>(out + p * ld + c0) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        return;
    }
    float4 wv[9];
#pragma unroll
    for (int t = 0; t < 9; ++t)
        wv[t] = make_float4(__ldg(w + (int64_t)c0 * 9 + t), __ldg(w + (int64_t)(c0 + 1) * 9 + t),
                            __ldg(w + (int64_t)(c0 + 2) * 9 + t), __ldg(w + (int64_t)(c0 + 3) * 9 + t));
    for (int k = 0; k < DW_PIX; ++k) {
        const int64_t p = run * DW_PIX + k;
        if (p >= P) break;
        const int ox = (int)(p % OW);
        const int64_t rest = p / OW;
        const int oy = (int)(rest % OH);
        const int n = (int)(rest / OH);
        const float* base = in + (int64_t)n * IH * IW * ld + c0;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            int iy;
            if (DGRAD) {
                const int num = oy + d - r * d;
                if (num < 0 || (S == 2 && (num & 1))) continue;
                iy = num / S;
            } else {
                iy = oy * S + (r - 1) * d;
                if (iy < 0) continue;
            }
            if (iy >= IH) continue;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                int ix;
                if (DGRAD) {
                    const int num = ox + d - s * d;
                    if (num < 0 || (S == 2 && (num & 1))) continue;
                    ix = num / S;
                } else {
                    ix = ox * S + (s - 1) * d;
                    if (ix < 0) continue;
                }
                if (ix >= IW) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((int64_t)iy * IW + ix) * ld));
                acc = dw_fma4(wv[r * 3 + s], v, acc);
            }
        }
        *reinterpret_cast<float4*>(out + p * ld + c0) = acc;
    }
}

// part[chunk][t][ld] (fp64) = this block's sum over its output pixels of x(tap t) * dy, for its DW_WG_QB channel quads
template <int S>
__global__ void __launch_bounds__(DW_THREADS) dw_wgrad_partial_kernel(const float* __restrict__ x,
                                                                      const float* __restrict__ dy,
                                                                      double* __restrict__ part, int N, int H, int W,
                                                                      int OH, int OW, int C, int ld, int d, int64_t chunk) {
    __shared__ float4 red[DW_THREADS / DW_WG_QB][9][DW_WG_QB];
    const int PY = DW_THREADS / DW_WG_QB;
    const int tx = threadIdx.x % DW_WG_QB, ty = threadIdx.x / DW_WG_QB;
    const int q = blockIdx.y * DW_WG_QB + tx;
    const int c0 = q * 4;
    const int64_t P = (int64_t)N * OH * OW;
    float4 acc[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c0 < C) {
        const int64_t p_end = min(P, ((int64_t)blockIdx.x + 1) * chunk);
        for (int64_t p = (int64_t)blockIdx.x * chunk + ty; p < p_end; p += PY) {
            const int ox = (int)(p % OW);
            const int64_t rest = p / OW;
            const int oy = (int)(rest % OH);
            const int n = (int)(rest / OH);
            const float4 g = __ldg(reinterpret_cast<const float4*>(dy + p * ld + c0));
            const float* base = x + (int64_t)n * H * W * ld + c0;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const int iy = oy * S + (r - 1) * d;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int s = 0; s < 3; ++s) {
                    const int ix = ox * S + (s - 1) * d;
                    if (ix < 0 || ix >= W) continue;
                    const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((int64_t)iy * W + ix) * ld));
                    acc[r * 3 + s] = dw_fma4(v, g, acc[r * 3 + s]);
                }
            }
        }
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) red[ty][t][tx] = acc[t];
    __syncthreads();
    const int Q = ld >> 2;
    for (int e = threadIdx.x; e < 9 * DW_WG_QB; e += DW_THREADS) {
        const int t = e / DW_WG_QB, qx = e % DW_WG_QB;
        const int qq = blockIdx.y * DW_WG_QB + qx;
        if (qq >= Q) continue;
        double sx = 0.0, sy = 0.0, sz = 0.0, sw = 0.0;
        for (int y = 0; y < PY; ++y) {
            const float4 v = red[y][t][qx];
            sx += v.x; sy += v.y; sz += v.z; sw += v.w;
        }
        double* o = part + ((int64_t)blockIdx.x * 9 + t) * ld + qq * 4;
        o[0] = sx; o[1] = sy; o[2] = sz; o[3] = sw;
    }
}

// dw[c*9 + t] (accumulate: +=) = sum over the chunks, in chunk order, of part[chunk][t][c]
__global__ void __launch_bounds__(DW_THREADS) dw_wgrad_sum_kernel(const double* __restrict__ part, float* __restrict__ dw,
                                                                  int C, int ld, int nchunks, int accumulate) {
    const int i = blockIdx.x * DW_THREADS + threadIdx.x;
    if (i >= 9 * C) return;
    const int t = i / C, c = i % C;
    double s = 0.0;
    for (int b = 0; b < nchunks; ++b) s += part[((int64_t)b * 9 + t) * ld + c];
    float* o = dw + (int64_t)c * 9 + t;
    *o = accumulate ? (float)((double)*o + s) : (float)s;
}

// act1, act2: the two activation tensors (float4 accesses), w: the other pointer
static int dw_check(const void* act1, const void* act2, const void* w, int N, int H, int W, int C, int ld, int OH, int OW,
                    int stride, int dilation) {
    if (!act1 || !act2 || !w) return PXL_ERR_BAD_ARG;
    if (((uintptr_t)act1 | (uintptr_t)act2) & 15) return PXL_ERR_BAD_ARG;
    if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || C > ld || (C & 3) || (ld & 3) || dilation < 1) return PXL_ERR_BAD_ARG;
    if (!(stride == 1 || (stride == 2 && dilation == 1))) return PXL_ERR_UNSUPPORTED;
    if (OH != (H - 1) / stride + 1 || OW != (W - 1) / stride + 1) return PXL_ERR_BAD_ARG;
    return 0;
}

template <bool DGRAD>
static int dw_gather(const float* in, const float* w, float* out, int N, int IH, int IW, int OH, int OW, int C, int ld,
                     int stride, int dilation, void* stream) {
    const int64_t nruns = pxl_cdiv((int64_t)N * OH * OW, DW_PIX);
    const int64_t threads = nruns * (ld >> 2);
    const int64_t blocks = pxl_cdiv(threads, DW_THREADS);
    if (blocks > 0x7fffffff) return PXL_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    if (stride == 1)
        dw_gather_kernel<1, DGRAD><<<(unsigned)blocks, DW_THREADS, 0, st>>>(in, w, out, N, IH, IW, OH, OW, C, ld, dilation, nruns);
    else
        dw_gather_kernel<2, DGRAD><<<(unsigned)blocks, DW_THREADS, 0, st>>>(in, w, out, N, IH, IW, OH, OW, C, ld, dilation, nruns);
    PXL_CHECK_LAUNCH();
    return 0;
}

extern "C" int pxl_dw_conv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int C, int ld, int OH,
                               int OW, int stride, int dilation, void* stream) {
    int rc = dw_check(x, y, w, N, H, W, C, ld, OH, OW, stride, dilation);
    if (rc) return rc;
    return dw_gather<false>(x, w, y, N, H, W, OH, OW, C, ld, stride, dilation, stream);
}

extern "C" int pxl_dw_conv_dgrad(const float* dy, const float* w, float* dx, int N, int H, int W, int C, int ld, int OH,
                                 int OW, int stride, int dilation, void* stream) {
    int rc = dw_check(dy, dx, w, N, H, W, C, ld, OH, OW, stride, dilation);
    if (rc) return rc;
    return dw_gather<true>(dy, w, dx, N, OH, OW, H, W, C, ld, stride, dilation, stream);
}

extern "C" int pxl_dw_conv_wgrad(const float* x, const float* dy, float* dw, int N, int H, int W, int C, int ld, int OH,
                                 int OW, int stride, int dilation, int accumulate, void* stream) {
    int rc = dw_check(x, dy, dw, N, H, W, C, ld, OH, OW, stride, dilation);
    if (rc) return rc;
    const int64_t P = (int64_t)N * OH * OW;
    const int gy = (int)pxl_cdiv(ld >> 2, DW_WG_QB);
    // the chunking depends on the shape only, so the summation order (and the result) is the same on every call
    int64_t nchunks = pxl_cdiv(DW_WG_BLOCKS, gy);
    nchunks = max((int64_t)1, min(nchunks, pxl_cdiv(P, (DW_THREADS / DW_WG_QB) * 4)));
    const int64_t chunk = pxl_cdiv(P, nchunks);
    nchunks = pxl_cdiv(P, chunk);
    double* part = (double*)pxl_workspace_(PXL_WS_DEPTHWISE, stream, (size_t)nchunks * 9 * ld * sizeof(double), &rc);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((unsigned)nchunks, (unsigned)gy);
    if (stride == 1)
        dw_wgrad_partial_kernel<1><<<grid, DW_THREADS, 0, st>>>(x, dy, part, N, H, W, OH, OW, C, ld, dilation, chunk);
    else
        dw_wgrad_partial_kernel<2><<<grid, DW_THREADS, 0, st>>>(x, dy, part, N, H, W, OH, OW, C, ld, dilation, chunk);
    PXL_CHECK_LAUNCH();
    dw_wgrad_sum_kernel<<<(unsigned)pxl_cdiv(9 * C, DW_THREADS), DW_THREADS, 0, st>>>(part, dw, C, ld, (int)nchunks,
                                                                                     accumulate);
    PXL_CHECK_LAUNCH();
    return 0;
}
