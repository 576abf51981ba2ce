// Tail kernels of the adversarial / GCT / CCT algorithms: layout changes between the planar class
// maps and the NHWC convolution inputs, LeakyReLU, masked BCE-with-logits, one-hot of the labels,
// Adam on a flat arena, separable reflect-padded Gaussian blur, 3x3 dilation, per-sample min-max
// normalisation.  All HBM-bound, one pass per tensor.
#include "common.cuh"
#include <math_constants.h>

// ------------------------------------------------------------------------------------------
// planar [n, C, HW]  <->  NHWC [n, HW, ldc] (lanes >= C zero-filled).  32 x 32 smem transpose tiles.
//   feeds FCDiscriminator / FlawDetector inputs (ssl_adv.py:148, ssl_gct.py:566-570)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
planar_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int ldc, int coff) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int64_t p0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {          // r: channel, tx: pixel (coalesced planar read)
        const int c = c0 + r;
        const int64_t p = p0 + tx;
        tile[r][tx] = (c < C && p < HW) ? __ldg(in + ((int64_t)n * C + c) * HW + p) : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {          // r: pixel, tx: channel (coalesced NHWC write)
        const int64_t p = p0 + r;
        const int c = c0 + tx;
        if (p < HW && c < C) out[((int64_t)n * HW + p) * ldc + coff + c] = tile[tx][r];
    }
}

// coff: first destination lane (lets two planar tensors be concatenated along channels)
extern "C" int pxl_planar_to_nhwc(const float* in, float* out, int n, int C, int64_t HW, int ldc, int coff, void* stream) {
    if (!in || !out || n <= 0 || C <= 0 || HW <= 0 || coff < 0 || coff + C > ldc || n > 65535) return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(HW, 32), (unsigned)pxl_cdiv(C, 32), (unsigned)n);
    planar_to_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, C, HW, ldc, coff);
    PXL_CHECK_LAUNCH();
    return 0;
}

__global__ void __launch_bounds__(256)
nhwc_to_planar_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int ldc, int coff) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int64_t p0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {          // r: pixel, tx: channel
        const int64_t p = p0 + r;
        const int c = c0 + tx;
        tile[r][tx] = (p < HW && c < C) ? __ldg(in + ((int64_t)n * HW + p) * ldc + coff + c) : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {          // r: channel, tx: pixel
        const int c = c0 + r;
        const int64_t p = p0 + tx;
        if (c < C && p < HW) out[((int64_t)n * C + c) * HW + p] = tile[tx][r];
    }
}

extern "C" int pxl_nhwc_to_planar(const float* in, float* out, int n, int C, int64_t HW, int ldc, int coff, void* stream) {
    if (!in || !out || n <= 0 || C <= 0 || HW <= 0 || coff < 0 || coff + C > ldc || n > 65535) return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(HW, 32), (unsigned)pxl_cdiv(C, 32), (unsigned)n);
    nhwc_to_planar_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, C, HW, ldc, coff);
    PXL_CHECK_LAUNCH();
    return 0;
}

// one-hot of float labels into NHWC lanes [coff, coff+C); ignore / out-of-range labels -> all zero
//   task/sseg/func.py:157-168 (AdvSSL real input), :179-192 (GCT)
__global__ void __launch_bounds__(256)
onehot_nhwc_kernel(const float* __restrict__ labels, float* __restrict__ out, int64_t total, int C, int ldc, int coff) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const float lf = __ldg(labels + i);
        float* o = out + i * ldc + coff;
        for (int c = 0; c < C; ++c) o[c] = (lf == (float)c) ? 1.f : 0.f;
    }
}

extern "C" int pxl_onehot_nhwc(const float* labels, float* out, int64_t pixels, int C, int ldc, int coff, void* stream) {
    if (!labels || !out || pixels <= 0 || C <= 0 || coff < 0 || coff + C > ldc) return PXL_ERR_BAD_ARG;
    int blocks = (int)(pxl_cdiv(pixels, 256) < PXL_NUM_SMS * 8 ? pxl_cdiv(pixels, 256) : PXL_NUM_SMS * 8);
    onehot_nhwc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(labels, out, pixels, C, ldc, coff);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// LeakyReLU (slope 0.2: ssl_adv.py:478, ssl_gct.py:549-563; slope 0 = ReLU) forward / backward
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
leaky_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y, int64_t n4, float slope) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 v = x[i];
        v.x = v.x > 0.f ? v.x : v.x * slope; v.y = v.y > 0.f ? v.y : v.y * slope;
        v.z = v.z > 0.f ? v.z : v.z * slope; v.w = v.w > 0.f ? v.w : v.w * slope;
        y[i] = v;
    }
}
__global__ void __launch_bounds__(256)
leaky_bwd_kernel(const float4* __restrict__ y, const float4* __restrict__ dy, float4* __restrict__ dx, int64_t n4, float slope) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 o = y[i];
        float4 d = dy[i];
        d.x = o.x > 0.f ? d.x : d.x * slope; d.y = o.y > 0.f ? d.y : d.y * slope;
        d.z = o.z > 0.f ? d.z : d.z * slope; d.w = o.w > 0.f ? d.w : d.w * slope;
        dx[i] = d;
    }
}
static int ew_blocks(int64_t n4) { return (int)(pxl_cdiv(n4, 256 * 2) < PXL_NUM_SMS * 8 ? pxl_cdiv(n4, 256 * 2) : PXL_NUM_SMS * 8); }

extern "C" int pxl_leaky_relu_fwd(const float* x, float* y, int64_t n, float slope, void* stream) {
    if (!x || !y || n <= 0 || (n & 3)) return PXL_ERR_BAD_ARG;
    leaky_fwd_kernel<<<ew_blocks(n / 4), 256, 0, (cudaStream_t)stream>>>((const float4*)x, (float4*)y, n / 4, slope);
    PXL_CHECK_LAUNCH();
    return 0;
}
extern "C" int pxl_leaky_relu_bwd(const float* y, const float* dy, float* dx, int64_t n, float slope, void* stream) {
    if (!y || !dy || !dx || n <= 0 || (n & 3)) return PXL_ERR_BAD_ARG;
    leaky_bwd_kernel<<<ew_blocks(n / 4), 256, 0, (cudaStream_t)stream>>>((const float4*)y, (const float4*)dy, (float4*)dx, n / 4, slope);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// masked BCE-with-logits: FCDiscriminatorCriterion (ssl_adv.py:496-503) after
// ssladv_preprocess_fcd_criterion (task/sseg/func.py:137-155): target = `target` everywhere, pixels
// whose task label == ignore_index have BOTH prediction and target multiplied by 0, i.e. they
// contribute bce(0, 0) = ln 2 (not 0) and no gradient.  per_sample[i] = mean over H*W.
// ------------------------------------------------------------------------------------------
template <bool WRITE_GRAD>
__global__ void __launch_bounds__(256)
bce_masked_kernel(const float* __restrict__ pred, const float* __restrict__ labels, float target, int ignore_index,
                  int64_t HW, float* __restrict__ per_sample, float* __restrict__ grad,
                  const float* __restrict__ upstream, float upstream_const) {
    const int b = blockIdx.y;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float loss = 0.f;
    if (p < HW) {
        const int64_t i = (int64_t)b * HW + p;
        bool keep = true;
        if (labels) keep = !(__ldg(labels + i) == (float)ignore_index);
        const float x = keep ? __ldg(pred + i) : 0.f;
        const float z = keep ? target : 0.f;
        loss = fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x)));
        if (WRITE_GRAD) {
            const float g = (upstream ? upstream[b] : upstream_const) / (float)HW;
            const float sig = 1.f / (1.f + expf(-x));
            grad[i] = keep ? g * (sig - z) : 0.f;
        }
    }
    __shared__ float wp[8];
    loss = warp_sum(loss);
    if ((threadIdx.x & 31) == 0) wp[threadIdx.x >> 5] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += wp[i];
        atomicAdd(per_sample + b, s / (float)HW);
    }
}

extern "C" int pxl_bce_logits_masked(const float* pred, const float* labels, float target, int ignore_index, int n,
                                     int64_t HW, float* per_sample, float* grad, const float* upstream,
                                     float upstream_const, void* stream) {
    if (!pred || !per_sample || n <= 0 || HW <= 0 || n > 65535) return PXL_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(per_sample, 0, sizeof(float) * n, st);
    if (e != cudaSuccess) return (int)e;
    dim3 grid((unsigned)pxl_cdiv(HW, 256), (unsigned)n);
    if (grad) bce_masked_kernel<true><<<grid, 256, 0, st>>>(pred, labels, target, ignore_index, HW, per_sample, grad, upstream, upstream_const);
    else bce_masked_kernel<false><<<grid, 256, 0, st>>>(pred, labels, target, ignore_index, HW, per_sample, nullptr, nullptr, 0.f);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam semantics, no amsgrad) over a flat arena: the FC discriminator / flaw
// detector optimiser (ssl_adv.py:101-102, ssl_gct.py:153-154: betas (0.9, 0.99))
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            int64_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float grad = g[i];
        const float pv = p[i];
        if (wd != 0.f) grad = fmaf(wd, pv, grad);
        const float mi = m[i] + (1.f - b1) * (grad - m[i]);          // lerp, like torch
        const float vi = b2 * v[i] + (1.f - b2) * grad * grad;
        m[i] = mi; v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        p[i] = pv - (lr / bc1) * (mi / denom);
    }
}

extern "C" int pxl_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                        float eps, float weight_decay, int step, void* stream) {
    if (!p || !g || !m || !v || n <= 0 || step < 1) return PXL_ERR_BAD_ARG;
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    int blocks = (int)(pxl_cdiv(n, 256 * 4) < PXL_NUM_SMS * 8 ? pxl_cdiv(n, 256 * 4) : PXL_NUM_SMS * 8);
    adam_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, (float)bc1, (float)sqrt(bc2));
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// Gaussian blur of single-channel maps [n, H, W]: ReflectionPad2d(k/2) + k x k depthwise conv
// (nn/module/gaussian_blur.py:30-64).  The reference's k x k kernel is exactly outer(v, v), so the
// blur is run as two 1-D passes (k up to 179 at 713^2: 90x fewer FLOPs than the direct form).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;
}

template <bool VERT>
__global__ void __launch_bounds__(256)
blur1d_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int k, const float* __restrict__ wts,
              float clamp_min) {
    extern __shared__ float sw[];
    for (int i = threadIdx.x; i < k; i += blockDim.x) sw[i] = __ldg(wts + i);
    __syncthreads();
    const int b = blockIdx.z;
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const float* ip = in + (int64_t)b * H * W;
    const int r = k / 2;
    float acc = 0.f;
    if (VERT) {
        for (int t = 0; t < k; ++t) acc = fmaf(sw[t], __ldg(ip + (int64_t)reflect(y + t - r, H) * W + x), acc);
    } else {
        const float* row = ip + (int64_t)y * W;
        for (int t = 0; t < k; ++t) acc = fmaf(sw[t], fmaxf(__ldg(row + reflect(x + t - r, W)), clamp_min), acc);
    }
    out[(int64_t)b * H * W + (int64_t)y * W + x] = acc;
}

// clamp_min: input values below it are raised to it first (FlawmapHandler zeroes negatives before
// blurring, ssl_gct.py:645); pass -INFINITY to disable
extern "C" int pxl_gauss_blur_sep(const float* in, float* tmp, float* out, int n, int H, int W, int k,
                                  const float* weights_1d, float clamp_min, void* stream) {
    if (!in || !tmp || !out || !weights_1d || n <= 0 || H <= 0 || W <= 0 || k <= 0 || !(k & 1)) return PXL_ERR_BAD_ARG;
    if (k / 2 >= H || k / 2 >= W || n > 65535) return PXL_ERR_UNSUPPORTED;      // single reflection only, like ReflectionPad2d
    dim3 grid((unsigned)pxl_cdiv(W, 32), (unsigned)pxl_cdiv(H, 8), (unsigned)n);
    cudaStream_t st = (cudaStream_t)stream;
    blur1d_kernel<false><<<grid, 256, k * sizeof(float), st>>>(in, tmp, H, W, k, weights_1d, clamp_min);
    PXL_CHECK_LAUNCH();
    blur1d_kernel<true><<<grid, 256, k * sizeof(float), st>>>(tmp, out, H, W, k, weights_1d, -3.0e38f);
    PXL_CHECK_LAUNCH();
    return 0;
}

// 3x3 max filter with reflection padding 1 (ssl_gct.py:708-712: ReflectionPad2d(1) + MaxPool2d(3, 1))
__global__ void __launch_bounds__(256)
dilate3x3_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W) {
    const int b = blockIdx.z;
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const float* ip = in + (int64_t)b * H * W;
    float m = -CUDART_INF_F;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx)
            m = fmaxf(m, __ldg(ip + (int64_t)reflect(y + dy, H) * W + reflect(x + dx, W)));
    out[(int64_t)b * H * W + (int64_t)y * W + x] = m;
}

extern "C" int pxl_dilate3x3_reflect(const float* in, float* out, int n, int H, int W, void* stream) {
    if (!in || !out || n <= 0 || H < 2 || W < 2 || n > 65535) return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(W, 32), (unsigned)pxl_cdiv(H, 8), (unsigned)n);
    dilate3x3_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, H, W);
    PXL_CHECK_LAUNCH();
    return 0;
}

// per-sample min-max normalisation (x - min) / (max - min + eps); zero_below: if the sample's max
// is <= zero_below the whole map is zeroed first (FlawmapHandler, ssl_gct.py:641-657; < 0 disables)
// Two launches: (1) per-sample min / max over many CTAs (order-independent, so still deterministic) through ordered-uint
// atomics into a small workspace, (2) the normalisation itself.  A single 512-thread CTA per sample, as in round 1, is
// latency bound on 713x713 maps (0.36 ms per call).
__device__ __forceinline__ unsigned f2ord(float f) { const unsigned u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float ord2f(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

__global__ void minmax_init_kernel(unsigned* ws, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { ws[2 * i] = 0xffffffffu; ws[2 * i + 1] = 0u; }
}

__global__ void __launch_bounds__(256)
minmax_reduce_kernel(const float* __restrict__ in, int64_t HW, float clamp_min, unsigned* __restrict__ ws) {
    const int b = blockIdx.y;
    const float* ip = in + (int64_t)b * HW;
    float mn = CUDART_INF_F, mx = -CUDART_INF_F;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        float v = __ldg(ip + i);
        if (v < clamp_min) v = clamp_min;
        mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
    mn = -warp_max(-mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { atomicMin(ws + 2 * b, f2ord(mn)); atomicMax(ws + 2 * b + 1, f2ord(mx)); }
}

__global__ void __launch_bounds__(256)
minmax_apply_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t HW, float eps, float zero_below,
                    float clamp_min, const unsigned* __restrict__ ws) {
    const int b = blockIdx.y;
    const float mn = ord2f(ws[2 * b]), mx = ord2f(ws[2 * b + 1]);
    // reference quirk kept: min/max are taken BEFORE the map is zeroed (ssl_gct.py:648-654), so a
    // zeroed map becomes the constant -min / (max - min + eps), not 0
    const bool zero = (zero_below >= 0.f) && (mx <= zero_below);
    const float denom = mx - mn + eps;
    const float* ip = in + (int64_t)b * HW;
    float* op = out + (int64_t)b * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        float v = __ldg(ip + i);
        if (v < clamp_min) v = clamp_min;
        if (zero) v = 0.f;
        op[i] = (v - mn) / denom;
    }
}

// clamp_min: values below it are raised to it first (FlawmapHandler clamps negatives to 0; pass
// -inf to disable).  in == out allowed.
extern "C" int pxl_minmax_norm(const float* in, float* out, int n, int64_t HW, float eps, float zero_below,
                               float clamp_min, void* stream) {
    if (!in || !out || n <= 0 || HW <= 0 || n > 65535) return PXL_ERR_BAD_ARG;
    static unsigned* ws = nullptr;
    static int ws_n = 0;
    if (ws_n < n) {
        if (ws) cudaFree(ws);
        if (cudaMalloc(&ws, (size_t)2 * n * sizeof(unsigned)) != cudaSuccess) { ws = nullptr; ws_n = 0; return PXL_ERR_BAD_ARG; }
        ws_n = n;
    }
    cudaStream_t st = (cudaStream_t)stream;
    int bx = (int)pxl_cdiv(HW, 256 * 8);
    if (bx > PXL_NUM_SMS * 2) bx = PXL_NUM_SMS * 2;
    if (bx < 1) bx = 1;
    minmax_init_kernel<<<(n + 127) / 128, 128, 0, st>>>(ws, n);
    minmax_reduce_kernel<<<dim3(bx, n), 256, 0, st>>>(in, HW, clamp_min, ws);
    minmax_apply_kernel<<<dim3(bx, n), 256, 0, st>>>(in, out, HW, eps, zero_below, clamp_min, ws);
    pxl_count_launch_(2);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// GCT generators (ssl_gct.py:660-728)
// ------------------------------------------------------------------------------------------
// DCGTGenerator.forward (ssl_gct.py:668-689): flaw maps above the threshold are raised to 1, the map
// with the smaller (better) flaw value wins the pixel; both_bad marks pixels above the threshold in
// both.  l_fm / r_fm: handled flaw maps [n, HW]; preds / outputs planar [n, C, HW].
__global__ void __launch_bounds__(256)
gct_dcgt_kernel(const float* __restrict__ l_pred, const float* __restrict__ r_pred, const float* __restrict__ l_fm,
                const float* __restrict__ r_fm, float thr, int C, int64_t HW, float* __restrict__ l_dc,
                float* __restrict__ r_dc, float* __restrict__ both_bad) {
    const int b = blockIdx.y;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float lt = __ldg(l_fm + (int64_t)b * HW + p), rt = __ldg(r_fm + (int64_t)b * HW + p);
    const bool lb = lt > thr, rb = rt > thr;
    both_bad[(int64_t)b * HW + p] = (lb && rb) ? 1.f : 0.f;
    // x.mul_(x <= thr).add_(x > thr)
    const float lh = __fadd_rn(__fmul_rn(lt, lb ? 0.f : 1.f), lb ? 1.f : 0.f);
    const float rh = __fadd_rn(__fmul_rn(rt, rb ? 0.f : 1.f), rb ? 1.f : 0.f);
    const float lm = rh >= lh ? 1.f : 0.f, rm = lh >= rh ? 1.f : 0.f;
    const int64_t base = (int64_t)b * C * HW + p;
    for (int c = 0; c < C; ++c) {
        const float lp = __ldg(l_pred + base + (int64_t)c * HW), rp = __ldg(r_pred + base + (int64_t)c * HW);
        l_dc[base + (int64_t)c * HW] = __fadd_rn(__fmul_rn(lm, lp), __fmul_rn(__fsub_rn(1.f, lm), rp));
        r_dc[base + (int64_t)c * HW] = __fadd_rn(__fmul_rn(rm, rp), __fmul_rn(__fsub_rn(1.f, rm), lp));
    }
}

extern "C" int pxl_gct_dcgt(const float* l_pred, const float* r_pred, const float* l_fm, const float* r_fm, float thr,
                            int n, int C, int64_t HW, float* l_dc, float* r_dc, float* both_bad, void* stream) {
    if (!l_pred || !r_pred || !l_fm || !r_fm || !l_dc || !r_dc || !both_bad || n <= 0 || C <= 0 || HW <= 0 || n > 65535)
        return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(HW, 256), (unsigned)n);
    gct_dcgt_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(l_pred, r_pred, l_fm, r_fm, thr, C, HW, l_dc, r_dc, both_bad);
    PXL_CHECK_LAUNCH();
    return 0;
}

// First stage of FDGTGenerator.forward (ssl_gct.py:714-716) fused with sslgct_prepare_task_gt_for_fdgt
// (task/sseg/func.py:179-192): out = mu * sum_c |onehot(label)_c - prob_c|, the one-hot row of an
// ignored / unlabeled pixel being all zero.
__global__ void __launch_bounds__(256)
fdgt_absdiff_kernel(const float* __restrict__ prob, const float* __restrict__ labels, float mu, int C, int64_t HW,
                    float* __restrict__ out) {
    const int b = blockIdx.y;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float lf = __ldg(labels + (int64_t)b * HW + p);
    const int64_t base = (int64_t)b * C * HW + p;
    float s = 0.f;
    for (int c = 0; c < C; ++c) {
        const float oh = (lf == (float)c) ? 1.f : 0.f;
        s += fabsf(oh - __ldg(prob + base + (int64_t)c * HW));
    }
    out[(int64_t)b * HW + p] = s * mu;
}

extern "C" int pxl_fdgt_absdiff(const float* prob, const float* labels, float mu, int n, int C, int64_t HW, float* out,
                                void* stream) {
    if (!prob || !labels || !out || n <= 0 || C <= 0 || HW <= 0 || n > 65535) return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(HW, 256), (unsigned)n);
    fdgt_absdiff_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(prob, labels, mu, C, HW, out);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// CCT auxiliary-decoder pieces (ssl_cct.py:501-745, _pspnet.py:40-54)
// ------------------------------------------------------------------------------------------
// nn.PixelShuffle(2) on NHWC: out[n, 2y+i, 2x+j, c] = in[n, y, x, c*4 + i*2 + j], c < C; output lanes
// [C, ldo) are zero-filled.  dir != 0 runs the inverse (the backward pass).
__global__ void __launch_bounds__(256)
pixel_shuffle2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int h, int w, int C, int ldi, int ldo, int inverse) {
    const int64_t total = (int64_t)N * (2 * h) * (2 * w) * ldo;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int c = (int)(idx % ldo);
        int64_t p = idx / ldo;
        const int X = (int)(p % (2 * w)); p /= (2 * w);
        const int Y = (int)(p % (2 * h));
        const int n = (int)(p / (2 * h));
        const int64_t small = (((int64_t)n * h + (Y >> 1)) * w + (X >> 1)) * ldi + c * 4 + (Y & 1) * 2 + (X & 1);
        if (!inverse) out[idx] = c < C ? __ldg(in + small) : 0.f;
        else if (c < C) out[small] = __ldg(in + idx);       // here `in` is the big tensor, `out` the small one
    }
}

extern "C" int pxl_pixel_shuffle2_nhwc(const float* in, float* out, int N, int h, int w, int C, int ldi, int ldo,
                                       int inverse, void* stream) {
    if (!in || !out || N <= 0 || h <= 0 || w <= 0 || C <= 0 || ldi < 4 * C || ldo < C) return PXL_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (inverse && ldi > 4 * C) {           // padding lanes of the small gradient tensor must be zero
        cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * (size_t)N * h * w * ldi, st);
        if (e != cudaSuccess) return (int)e;
    }
    const int64_t total = (int64_t)N * 4 * h * w * ldo;
    int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 16 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 16);
    pixel_shuffle2_kernel<<<blocks, 256, 0, st>>>(in, out, N, h, w, C, ldi, ldo, inverse);
    PXL_CHECK_LAUNCH();
    return 0;
}

// out = x * pixel_mask[n, hw] * chan_scale[n, c] * (1 + elem_noise[hw, c])   (each factor optional)
//   pixel mask: CutOut / context / object masking / feature drop; channel scale: Dropout2d;
//   element noise: FeatureNoiseDecoder (x.mul(noise) + x, noise shared over the batch)
__global__ void __launch_bounds__(256)
perturb_kernel(const float4* __restrict__ x, const float* __restrict__ pmask, const float* __restrict__ cscale,
               const float4* __restrict__ noise, float4* __restrict__ out, int64_t n4, int c4, int64_t HW) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const int c = (int)(i % c4);
        const int64_t pix = i / c4;          // n * HW + hw
        float4 v = x[i];
        if (pmask) { const float m = __ldg(pmask + pix); v.x *= m; v.y *= m; v.z *= m; v.w *= m; }
        if (cscale) {
            const int64_t n = pix / HW;
            const float4 s = __ldg(reinterpret_cast<const float4*>(cscale) + n * c4 + c);
            v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
        }
        if (noise) {
            const float4 e = __ldg(noise + (pix % HW) * c4 + c);
            v.x = fmaf(v.x, e.x, v.x); v.y = fmaf(v.y, e.y, v.y); v.z = fmaf(v.z, e.z, v.z); v.w = fmaf(v.w, e.w, v.w);
        }
        out[i] = v;
    }
}

extern "C" int pxl_perturb_nhwc(const float* x, const float* pixel_mask, const float* chan_scale, const float* elem_noise,
                                float* out, int N, int64_t HW, int C, void* stream) {
    if (!x || !out || N <= 0 || HW <= 0 || C <= 0 || (C & 3)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = (int64_t)N * HW * (C / 4);
    perturb_kernel<<<ew_blocks(n4), 256, 0, (cudaStream_t)stream>>>((const float4*)x, pixel_mask, chan_scale,
                                                                   (const float4*)elem_noise, (float4*)out, n4, C / 4, HW);
    PXL_CHECK_LAUNCH();
    return 0;
}

// UniMatch feature perturbation: out [2N, HW, C] = [x; x * chan_scale[n, c]] (Dropout2d copies after the clean
// features, one read and two writes); backward dx = g[:N] + g[N:] * chan_scale.  Products and sums are rounded
// separately, as torch's x * s and a + b * s are.
__global__ void __launch_bounds__(256)
fp_dup_kernel(const float4* __restrict__ x, const float* __restrict__ cscale, float4* __restrict__ out, int64_t n4,
              int c4, int64_t HW) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const int c = (int)(i % c4);
        const int64_t n = i / c4 / HW;
        const float4 s = __ldg(reinterpret_cast<const float4*>(cscale) + n * c4 + c);
        const float4 v = x[i];
        out[i] = v;
        out[n4 + i] = make_float4(__fmul_rn(v.x, s.x), __fmul_rn(v.y, s.y), __fmul_rn(v.z, s.z), __fmul_rn(v.w, s.w));
    }
}

__global__ void __launch_bounds__(256)
fp_dup_bwd_kernel(const float4* __restrict__ g, const float* __restrict__ cscale, float4* __restrict__ dx, int64_t n4,
                  int c4, int64_t HW) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const int c = (int)(i % c4);
        const int64_t n = i / c4 / HW;
        const float4 s = __ldg(reinterpret_cast<const float4*>(cscale) + n * c4 + c);
        const float4 a = g[i], b = g[n4 + i];
        dx[i] = make_float4(__fadd_rn(a.x, __fmul_rn(b.x, s.x)), __fadd_rn(a.y, __fmul_rn(b.y, s.y)),
                            __fadd_rn(a.z, __fmul_rn(b.z, s.z)), __fadd_rn(a.w, __fmul_rn(b.w, s.w)));
    }
}

extern "C" int pxl_fp_dup_nhwc(const float* x, const float* chan_scale, float* out, int N, int64_t HW, int C,
                               void* stream) {
    if (!x || !chan_scale || !out || N <= 0 || HW <= 0 || C <= 0 || (C & 3)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = (int64_t)N * HW * (C / 4);
    fp_dup_kernel<<<ew_blocks(n4), 256, 0, (cudaStream_t)stream>>>((const float4*)x, chan_scale, (float4*)out, n4,
                                                                   C / 4, HW);
    PXL_CHECK_LAUNCH();
    return 0;
}

extern "C" int pxl_fp_dup_bwd_nhwc(const float* grad, const float* chan_scale, float* dx, int N, int64_t HW, int C,
                                   void* stream) {
    if (!grad || !chan_scale || !dx || N <= 0 || HW <= 0 || C <= 0 || (C & 3)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = (int64_t)N * HW * (C / 4);
    fp_dup_bwd_kernel<<<ew_blocks(n4), 256, 0, (cudaStream_t)stream>>>((const float4*)grad, chan_scale, (float4*)dx,
                                                                       n4, C / 4, HW);
    PXL_CHECK_LAUNCH();
    return 0;
}

// mean over channels per pixel of an NHWC tensor: FeatureDropDecoder attention (ssl_cct.py:721)
__global__ void __launch_bounds__(256)
channel_mean_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t pixels, int C) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int64_t p = warp; p < pixels; p += nwarps) {
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s += __ldg(x + p * C + c);
        s = warp_sum(s);
        if (lane == 0) out[p] = s / (float)C;
    }
}

extern "C" int pxl_channel_mean_nhwc(const float* x, float* out, int64_t pixels, int C, void* stream) {
    if (!x || !out || pixels <= 0 || C <= 0) return PXL_ERR_BAD_ARG;
    int blocks = (int)(pxl_cdiv(pixels, 8) < PXL_NUM_SMS * 8 ? pxl_cdiv(pixels, 8) : PXL_NUM_SMS * 8);
    channel_mean_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, out, pixels, C);
    PXL_CHECK_LAUNCH();
    return 0;
}

// (argmax_c logits > 0) as a float mask [n, HW]: guided masking / cutout of the CCT decoders
// (ssl_cct.py:609, 666, 693).  argmax returns the FIRST maximum, so class 0 wins ties.
__global__ void __launch_bounds__(256)
argmax_nonzero_kernel(const float* __restrict__ logits, float* __restrict__ mask, int C, int64_t HW) {
    const int b = blockIdx.y;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float* lg = logits + (int64_t)b * C * HW + p;
    const float v0 = __ldg(lg);
    float m = -CUDART_INF_F;
    for (int c = 1; c < C; ++c) m = fmaxf(m, __ldg(lg + (int64_t)c * HW));
    mask[(int64_t)b * HW + p] = m > v0 ? 1.f : 0.f;
}

extern "C" int pxl_argmax_nonzero_mask(const float* logits, float* mask, int n, int C, int64_t HW, void* stream) {
    if (!logits || !mask || n <= 0 || C <= 0 || HW <= 0 || n > 65535) return PXL_ERR_BAD_ARG;
    dim3 grid((unsigned)pxl_cdiv(HW, 256), (unsigned)n);
    argmax_nonzero_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(logits, mask, C, HW);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// PSPNet pyramid pooling pieces on NHWC (task/sseg/module/_pspnet.py:57-102)
// ------------------------------------------------------------------------------------------
// nn.AdaptiveAvgPool2d(bin): window [floor(i*H/bin), ceil((i+1)*H/bin)).  One thread per (bin cell, channel quad,
// window row): it sums its row and adds it into the (zeroed) output - with one thread per cell, as in round 1, the
// 1x1 / 2x2 pyramids summed up to 8100 pixels serially (0.13 ms per call on the 90x90 PSPNet latent).
__global__ void __launch_bounds__(256)
adaptive_pool_fwd_kernel(const float4* __restrict__ x, float* __restrict__ y, int N, int H, int W, int c4, int bin, int maxwin) {
    const int64_t total = (int64_t)N * bin * bin * c4 * maxwin;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = (int)(i % c4);
        int64_t p = i / c4;
        const int r = (int)(p % maxwin); p /= maxwin;
        const int bx = (int)(p % bin); p /= bin;
        const int by = (int)(p % bin);
        const int n = (int)(p / bin);
        const int y0 = (by * H) / bin, y1 = ((by + 1) * H + bin - 1) / bin;
        const int x0 = (bx * W) / bin, x1 = ((bx + 1) * W + bin - 1) / bin;
        const int yy = y0 + r;
        if (yy >= y1) continue;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int xx = x0; xx < x1; ++xx) {
            const float4 v = __ldg(x + ((int64_t)(n * H + yy) * W + xx) * c4 + c);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        const float inv = 1.f / (float)((y1 - y0) * (x1 - x0));
        float* o = y + ((((int64_t)n * bin + by) * bin + bx) * c4 + c) * 4;
        atomicAdd(o, s.x * inv); atomicAdd(o + 1, s.y * inv); atomicAdd(o + 2, s.z * inv); atomicAdd(o + 3, s.w * inv);
    }
}

// backward: each input pixel gathers from the (at most 2 x 2) bins whose window contains it
__global__ void __launch_bounds__(256)
adaptive_pool_bwd_kernel(const float4* __restrict__ dy, float4* __restrict__ dx, int N, int H, int W, int c4, int bin) {
    const int64_t total = (int64_t)N * H * W * c4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = (int)(i % c4);
        int64_t p = i / c4;
        const int xx = (int)(p % W); p /= W;
        const int yy = (int)(p % H);
        const int n = (int)(p / H);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int by = 0; by < bin; ++by) {
            const int y0 = (by * H) / bin, y1 = ((by + 1) * H + bin - 1) / bin;
            if (yy < y0 || yy >= y1) continue;
            for (int bx = 0; bx < bin; ++bx) {
                const int x0 = (bx * W) / bin, x1 = ((bx + 1) * W + bin - 1) / bin;
                if (xx < x0 || xx >= x1) continue;
                const float inv = 1.f / (float)((y1 - y0) * (x1 - x0));
                const float4 g = __ldg(dy + ((int64_t)(n * bin + by) * bin + bx) * c4 + c);
                s.x += g.x * inv; s.y += g.y * inv; s.z += g.z * inv; s.w += g.w * inv;
            }
        }
        dx[i] = s;
    }
}

extern "C" int pxl_adaptive_avgpool_nhwc(const float* x, float* y, int N, int H, int W, int C, int bin, int backward, void* stream) {
    if (!x || !y || N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 3) || bin <= 0) return PXL_ERR_BAD_ARG;
    const int64_t total = backward ? (int64_t)N * H * W * (C / 4) : (int64_t)N * bin * bin * (C / 4);
    int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 8 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 8);
    // backward: x = dy [N,bin,bin,C], y = dx [N,H,W,C]
    if (backward) adaptive_pool_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (float4*)y, N, H, W, C / 4, bin);
    else {
        const int maxwin = (H + bin - 1) / bin + 1;
        const int64_t tot = (int64_t)N * bin * bin * (C / 4) * maxwin;
        int fb = (int)(pxl_cdiv(tot, 256) < PXL_NUM_SMS * 16 ? pxl_cdiv(tot, 256) : PXL_NUM_SMS * 16);
        cudaMemsetAsync(y, 0, (size_t)N * bin * bin * C * sizeof(float), (cudaStream_t)stream);
        adaptive_pool_fwd_kernel<<<fb, 256, 0, (cudaStream_t)stream>>>((const float4*)x, y, N, H, W, C / 4, bin, maxwin);
    }
    PXL_CHECK_LAUNCH();
    return 0;
}

// bilinear resize NHWC -> NHWC lanes [coff, coff+C) of a wider tensor (the pyramid branches are
// written straight into the 4096-lane concat buffer, _pspnet.py:96-101); same index arithmetic as ATen
__device__ __forceinline__ float src_idx(float scale, int dst, bool ac) {
    if (ac) return scale * (float)dst;
    const float s = scale * ((float)dst + 0.5f) - 0.5f;
    return s < 0.f ? 0.f : s;
}

__global__ void __launch_bounds__(256)
bilinear_nhwc_fwd_kernel(const float4* __restrict__ in, float* __restrict__ out, int N, int h, int w, int c4, int H, int W,
                         int ldo, int coff, float sh, float sw, bool ac) {
    const int64_t total = (int64_t)N * H * W * c4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = (int)(i % c4);
        int64_t p = i / c4;
        const int X = (int)(p % W); p /= W;
        const int Y = (int)(p % H);
        const int n = (int)(p / H);
        const float fy = src_idx(sh, Y, ac), fx = src_idx(sw, X, ac);
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
        const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
        const float4 a = __ldg(in + ((int64_t)(n * h + y0) * w + x0) * c4 + c), b = __ldg(in + ((int64_t)(n * h + y0) * w + x1) * c4 + c);
        const float4 d = __ldg(in + ((int64_t)(n * h + y1) * w + x0) * c4 + c), e = __ldg(in + ((int64_t)(n * h + y1) * w + x1) * c4 + c);
        float4 r;
        r.x = ly0 * (lx0 * a.x + lx1 * b.x) + ly1 * (lx0 * d.x + lx1 * e.x);
        r.y = ly0 * (lx0 * a.y + lx1 * b.y) + ly1 * (lx0 * d.y + lx1 * e.y);
        r.z = ly0 * (lx0 * a.z + lx1 * b.z) + ly1 * (lx0 * d.z + lx1 * e.z);
        r.w = ly0 * (lx0 * a.w + lx1 * b.w) + ly1 * (lx0 * d.w + lx1 * e.w);
        *reinterpret_cast<float4*>(out + ((int64_t)(n * H + Y) * W + X) * ldo + coff + 4 * c) = r;
    }
}

// backward: one thread per (input pixel, channel quad, OUTPUT ROW): rows outside the pixel's support exit at once, the
// others walk the output row and add their weighted sum into the (zeroed) input gradient.  Round 1 had one thread per
// input pixel scanning all H*W outputs (0.6 ms per call for the PSPNet pyramid at 90x90).
__global__ void __launch_bounds__(256)
bilinear_nhwc_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gin, int N, int h, int w, int c4, int H, int W,
                         int ldo, int coff, float sh, float sw, bool ac) {
    const int64_t total = (int64_t)N * h * w * c4 * H;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = (int)(i % c4);
        int64_t p = i / c4;
        const int Y = (int)(p % H); p /= H;
        const int xi = (int)(p % w); p /= w;
        const int yi = (int)(p % h);
        const int n = (int)(p / h);
        const float fy = src_idx(sh, Y, ac);
        const int y0 = (int)fy, y1 = y0 + (y0 < h - 1 ? 1 : 0);
        if (y0 != yi && y1 != yi) continue;
        const float ly1 = fy - (float)y0;
        float wy = 0.f;
        if (y0 == yi) wy += 1.f - ly1;
        if (y1 == yi) wy += ly1;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int X = 0; X < W; ++X) {
            const float fx = src_idx(sw, X, ac);
            const int x0 = (int)fx, x1 = x0 + (x0 < w - 1 ? 1 : 0);
            if (x0 != xi && x1 != xi) continue;
            const float lx1 = fx - (float)x0;
            float wx = 0.f;
            if (x0 == xi) wx += 1.f - lx1;
            if (x1 == xi) wx += lx1;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gout + ((int64_t)(n * H + Y) * W + X) * ldo + coff + 4 * c));
            s.x += g.x * wx; s.y += g.y * wx; s.z += g.z * wx; s.w += g.w * wx;
        }
        float* o = gin + ((((int64_t)n * h + yi) * w + xi) * c4 + c) * 4;
        atomicAdd(o, s.x * wy); atomicAdd(o + 1, s.y * wy); atomicAdd(o + 2, s.z * wy); atomicAdd(o + 3, s.w * wy);
    }
}

static inline float rs_scale(int in, int out, int ac) {
    if (ac) return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
    return (float)in / (float)out;
}

extern "C" int pxl_bilinear_nhwc(const float* in, float* out, int N, int h, int w, int C, int H, int W, int ldo, int coff,
                                 int align_corners, int backward, void* stream) {
    if (!in || !out || N <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 3) || (ldo & 3) || (coff & 3) || coff + C > ldo)
        return PXL_ERR_BAD_ARG;
    const float sh = rs_scale(h, H, align_corners), sw = rs_scale(w, W, align_corners);
    cudaStream_t st = (cudaStream_t)stream;
    if (!backward) {
        const int64_t total = (int64_t)N * H * W * (C / 4);
        int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 8 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 8);
        bilinear_nhwc_fwd_kernel<<<blocks, 256, 0, st>>>((const float4*)in, out, N, h, w, C / 4, H, W, ldo, coff, sh, sw, align_corners != 0);
    } else {      // in = grad of the wide output [N,H,W,ldo], out = grad of the small input [N,h,w,C]
        const int64_t total = (int64_t)N * h * w * (C / 4) * H;
        int blocks = (int)(pxl_cdiv(total, 256) < PXL_NUM_SMS * 16 ? pxl_cdiv(total, 256) : PXL_NUM_SMS * 16);
        cudaMemsetAsync(out, 0, (size_t)N * h * w * C * sizeof(float), st);
        bilinear_nhwc_bwd_kernel<<<blocks, 256, 0, st>>>(in, out, N, h, w, C / 4, H, W, ldo, coff, sh, sw, align_corners != 0);
    }
    PXL_CHECK_LAUNCH();
    return 0;
}

// copy a dense NHWC tensor into / out of lanes [coff, coff+C) of a wider one (channel concat)
__global__ void __launch_bounds__(256)
copy_lanes_kernel(const float4* __restrict__ src, float4* __restrict__ dst, int64_t rows, int c4, int ld4, int coff4, int extract) {
    const int64_t total = rows * c4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t r = i / c4;
        const int c = (int)(i % c4);
        if (!extract) dst[r * ld4 + coff4 + c] = src[i];
        else dst[i] = src[r * ld4 + coff4 + c];
    }
}

extern "C" int pxl_copy_lanes_nhwc(const float* src, float* dst, int64_t rows, int C, int ld, int coff, int extract, void* stream) {
    if (!src || !dst || rows <= 0 || C <= 0 || (C & 3) || (ld & 3) || (coff & 3) || coff + C > ld) return PXL_ERR_BAD_ARG;
    const int64_t total = rows * (C / 4);
    copy_lanes_kernel<<<ew_blocks(total), 256, 0, (cudaStream_t)stream>>>((const float4*)src, (float4*)dst, rows, C / 4, ld / 4, coff / 4, extract);
    PXL_CHECK_LAUNCH();
    return 0;
}
