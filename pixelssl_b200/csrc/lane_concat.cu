// DeepLabV3+ head concatenations on NHWC, forward and backward, with no atomics.
//
//   ASPP:     [conv 1x1 | conv 3x3 r1 | r2 | r3 | image pooling (1x1, broadcast)]          -> 1280 lanes
//   decoder:  [bilinear(ASPP out, 1/16 -> 1/4, align_corners=True) | reduced low-level | 0] -> 320 lanes
//
// One forward launch writes every lane of the concatenated tensor.  The backward writes each source's gradient by
// gathering: a same-size source copies its window, a resized source sums, per low-resolution pixel, the bilinear
// contributions of the high-resolution pixels under it (rows, then columns, in ascending order) and a 1x1 source
// sums its whole window (the spatial reduction below).  Every sum is taken in a fixed order, so two runs give
// bit-identical gradients.  Source positions are computed in integer arithmetic, so the interpolation weights are
// the correctly rounded fractions.
#include "common.cuh"

#define LC_MAX_SRC 8

struct LaneSrcs {
    const float* p[LC_MAX_SRC];
    int h[LC_MAX_SRC], w[LC_MAX_SRC], lds[LC_MAX_SRC], c[LC_MAX_SRC], off[LC_MAX_SRC];
    float sh[LC_MAX_SRC], sw[LC_MAX_SRC];
    int n;
};

static inline float ac_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

// source position of output index o for an n -> N resize with align_corners=True, o * (n-1) / (N-1), split into its
// integer part i0 and fraction in exact integer arithmetic (ATen's fp32 scale * o is off by up to ~o ulp of the scale)
__device__ __forceinline__ float ac_src(int o, int n, int N, int& i0) {
    if (N <= 1) { i0 = 0; return 0.f; }
    const unsigned num = (unsigned)o * (unsigned)(n - 1), den = (unsigned)(N - 1);      // sizes <= 65535: no overflow
    const unsigned q = num / den;
    i0 = (int)q;
    return (float)(num - q * den) / (float)den;
}

__global__ void __launch_bounds__(256)
lane_concat_kernel(LaneSrcs s, float* __restrict__ dst, int N, int H, int W, int ld) {
    const int64_t total = (int64_t)N * H * W * ld;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int lane = (int)(i % ld);
        const int64_t pix = i / ld;
        int k = -1;
        for (int j = 0; j < s.n; ++j)
            if (lane >= s.off[j] && lane < s.off[j] + s.c[j]) k = j;
        float v = 0.f;
        if (k >= 0) {
            const int ch = lane - s.off[k];
            const int h = s.h[k], w = s.w[k], lds = s.lds[k];
            const int X = (int)(pix % W), Y = (int)((pix / W) % H), b = (int)(pix / ((int64_t)W * H));
            const float* src = s.p[k];
            if (h == H && w == W) {
                v = __ldg(src + pix * lds + ch);
            } else {
                int y0, x0;
                const float ly1 = ac_src(Y, h, H, y0), lx1 = ac_src(X, w, W, x0);
                const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
                const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
                const float* base = src + (int64_t)b * h * w * lds + ch;
                v = ly0 * (lx0 * __ldg(base + ((int64_t)y0 * w + x0) * lds) + lx1 * __ldg(base + ((int64_t)y0 * w + x1) * lds)) +
                    ly1 * (lx0 * __ldg(base + ((int64_t)y1 * w + x0) * lds) + lx1 * __ldg(base + ((int64_t)y1 * w + x1) * lds));
            }
        }
        dst[i] = v;
    }
}

// window [0, c) of the source's lanes <- window [off, off + c) of the same-size gradient; lanes [c, lds) <- 0
__global__ void __launch_bounds__(256)
lane_copy_bwd_kernel(const float* __restrict__ g, float* __restrict__ dsrc, int64_t pixels, int ld, int lds, int c, int off) {
    const int64_t total = pixels * lds;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i % lds);
        dsrc[i] = ch < c ? __ldg(g + (i / lds) * ld + off + ch) : 0.f;
    }
}

// output rows whose 2-tap support can include low-resolution row i (conservative; the loop tests each row exactly)
__device__ __forceinline__ void ac_support(int i, int H, float s, int& lo, int& hi) {
    if (s <= 0.f) { lo = 0; hi = H - 1; return; }
    lo = (int)floorf(((float)i - 1.f) / s) - 1;
    hi = (int)ceilf(((float)i + 1.f) / s) + 1;
    if (lo < 0) lo = 0;
    if (hi > H - 1) hi = H - 1;
}

// weight of low-resolution index i in the bilinear sample of output index o (align_corners=True)
__device__ __forceinline__ float ac_weight(int o, int i, int n, int N) {
    int a;
    const float l1 = ac_src(o, n, N, a);
    const int b = a + (a < n - 1 ? 1 : 0);
    float wgt = 0.f;
    if (a == i) wgt += 1.f - l1;
    if (b == i) wgt += l1;
    return wgt;
}

__global__ void __launch_bounds__(256)
lane_bilinear_bwd_kernel(const float* __restrict__ g, float* __restrict__ dsrc, int N, int h, int w, int lds, int c,
                         int off, int H, int W, int ld, float sh, float sw) {
    const int64_t total = (int64_t)N * h * w * lds;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i % lds);
        if (ch >= c) { dsrc[i] = 0.f; continue; }
        const int64_t pix = i / lds;
        const int xi = (int)(pix % w), yi = (int)((pix / w) % h), b = (int)(pix / ((int64_t)w * h));
        int ylo, yhi, xlo, xhi;
        ac_support(yi, H, sh, ylo, yhi);
        ac_support(xi, W, sw, xlo, xhi);
        const float* gb = g + (int64_t)b * H * W * ld + off + ch;
        float acc = 0.f;
        for (int Y = ylo; Y <= yhi; ++Y) {
            const float wy = ac_weight(Y, yi, h, H);
            if (wy == 0.f) continue;
            const float* gr = gb + (int64_t)Y * W * ld;
            float row = 0.f;
            for (int X = xlo; X <= xhi; ++X) {
                const float wx = ac_weight(X, xi, w, W);
                if (wx != 0.f) row = fmaf(wx, __ldg(gr + (int64_t)X * ld), row);
            }
            acc = fmaf(wy, row, acc);
        }
        dsrc[i] = acc;
    }
}

// y[b, ch] = scale * sum over the H*W pixels of x[b, :, :, off + ch] for ch < c, 0 for c <= ch < ldy.
// CTA = (32-lane group, sample); warp k sums pixels k, k + 8, ... in fp64, the 8 partials are added in warp order.
__global__ void __launch_bounds__(256)
spatial_sum_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t HW, int ld, int off, int c, int ldy,
                   double scale) {
    __shared__ double part[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ch = blockIdx.x * 32 + lane;
    const int b = blockIdx.y;
    double acc = 0.0;
    if (ch < c) {
        const float* p = x + (int64_t)b * HW * ld + off + ch;
        for (int64_t q = warp; q < HW; q += 8) acc += (double)__ldg(p + q * ld);
    }
    part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && ch < ldy) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += part[k][lane];
        y[(int64_t)b * ldy + ch] = ch < c ? (float)(s * scale) : 0.f;
    }
}

static int spatial_sum(const float* x, float* y, int N, int64_t HW, int ld, int off, int c, int ldy, double scale,
                       cudaStream_t st) {
    if (N > 65535) return PXL_ERR_UNSUPPORTED;
    dim3 grid((unsigned)pxl_cdiv(ldy, 32), (unsigned)N);
    spatial_sum_kernel<<<grid, 256, 0, st>>>(x, y, HW, ld, off, c, ldy, scale);
    PXL_CHECK_LAUNCH();
    return 0;
}

static int grid_for(int64_t total) {
    const int64_t b = pxl_cdiv(total, 256);
    return (int)(b < PXL_NUM_SMS * 16 ? b : PXL_NUM_SMS * 16);
}

static int parse_srcs(const int* geo, int nsrc, int H, int W, int ld, LaneSrcs& s) {
    if (!geo || nsrc <= 0 || nsrc > LC_MAX_SRC) return PXL_ERR_BAD_ARG;
    if (H > 65535 || W > 65535) return PXL_ERR_UNSUPPORTED;
    s.n = nsrc;
    for (int k = 0; k < nsrc; ++k) {
        const int h = geo[5 * k], w = geo[5 * k + 1], lds = geo[5 * k + 2], c = geo[5 * k + 3], off = geo[5 * k + 4];
        if (h <= 0 || w <= 0 || c <= 0 || lds < c || off < 0 || off + c > ld) return PXL_ERR_BAD_ARG;
        if (h > 65535 || w > 65535) return PXL_ERR_UNSUPPORTED;
        for (int j = 0; j < k; ++j)
            if (off < s.off[j] + s.c[j] && s.off[j] < off + c) return PXL_ERR_BAD_ARG;     // windows overlap
        s.h[k] = h; s.w[k] = w; s.lds[k] = lds; s.c[k] = c; s.off[k] = off;
        s.sh[k] = ac_scale(h, H); s.sw[k] = ac_scale(w, W);
        s.p[k] = nullptr;
    }
    return 0;
}

extern "C" int pxl_lane_concat_nhwc(const float* const* srcs_host, const int* geo_host, int nsrc, float* dst, int N, int H,
                                    int W, int ld, void* stream) {
    if (!srcs_host || !dst || N <= 0 || H <= 0 || W <= 0 || ld <= 0) return PXL_ERR_BAD_ARG;
    LaneSrcs s;
    int rc = parse_srcs(geo_host, nsrc, H, W, ld, s);
    if (rc) return rc;
    for (int k = 0; k < nsrc; ++k) {
        if (!srcs_host[k]) return PXL_ERR_BAD_ARG;
        s.p[k] = srcs_host[k];
    }
    const int64_t total = (int64_t)N * H * W * ld;
    lane_concat_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(s, dst, N, H, W, ld);
    PXL_CHECK_LAUNCH();
    return 0;
}

extern "C" int pxl_lane_concat_bwd_nhwc(const float* grad, float* const* src_grads_host, const int* geo_host, int nsrc,
                                        int N, int H, int W, int ld, void* stream) {
    if (!grad || !src_grads_host || N <= 0 || H <= 0 || W <= 0 || ld <= 0) return PXL_ERR_BAD_ARG;
    LaneSrcs s;
    int rc = parse_srcs(geo_host, nsrc, H, W, ld, s);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    for (int k = 0; k < nsrc; ++k) {
        float* d = src_grads_host[k];
        if (!d) continue;                                    // no gradient wanted for this source
        const int h = s.h[k], w = s.w[k];
        if (h == H && w == W) {
            const int64_t pixels = (int64_t)N * H * W;
            lane_copy_bwd_kernel<<<grid_for(pixels * s.lds[k]), 256, 0, st>>>(grad, d, pixels, ld, s.lds[k], s.c[k], s.off[k]);
            PXL_CHECK_LAUNCH();
        } else if (h == 1 && w == 1) {
            rc = spatial_sum(grad, d, N, (int64_t)H * W, ld, s.off[k], s.c[k], s.lds[k], 1.0, st);
            if (rc) return rc;
        } else {
            lane_bilinear_bwd_kernel<<<grid_for((int64_t)N * h * w * s.lds[k]), 256, 0, st>>>(
                grad, d, N, h, w, s.lds[k], s.c[k], s.off[k], H, W, ld, s.sh[k], s.sw[k]);
            PXL_CHECK_LAUNCH();
        }
    }
    return 0;
}

extern "C" int pxl_spatial_mean_nhwc(const float* x, float* y, int N, int H, int W, int C, void* stream) {
    if (!x || !y || N <= 0 || H <= 0 || W <= 0 || C <= 0) return PXL_ERR_BAD_ARG;
    const int64_t HW = (int64_t)H * W;
    return spatial_sum(x, y, N, HW, C, 0, C, C, 1.0 / (double)HW, (cudaStream_t)stream);
}
