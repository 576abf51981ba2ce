// Strong photometric augmentation of UniMatch (Yang et al., CVPR 2023) on a batch of normalised planar images, with
// the semantics of torchvision's float-tensor functional ops (torchvision.transforms.v2.functional):
//   x01 = clamp(x * std + mean, 0, 1)
//   -> [ColorJitter: brightness, contrast, saturation, hue in the view's drawn order]
//   -> [rgb_to_grayscale, 3 channels]
//   -> [gaussian_blur, kernel 2*ks_half+1, reflect padding]
//   -> inside the view's box: the partner image's pixel of the same view
//   -> (x01 - mean) / std
// Views: v = k * ubs + i is view k (0 or 1) of image i; its partner is view k of image (i + ubs/2) mod ubs.  A pasted
// pixel is exactly the value the partner's own view has at that position before its own box is pasted.
// Every parameter comes from the host (ssl_algorithm/ssl_unimatch.py draws them), one row of AUG_COLS floats per view:
//   0 jitter applied, 1 brightness, 2 contrast, 3 saturation, 4 hue, 5..8 op order (0 b, 1 c, 2 s, 3 h),
//   9 grayscale, 10 blur half width (0: no blur), 11 sigma, 12..15 box y0 x0 y1 x1 (empty: y0 == y1),
//   16..16+2*AUG_MAXK normalised 1-D blur weights.
// Launches (all views at once): stats (per-block fp64 partials of the grayscale sum at contrast's position in the
// order) + fixed-order sum, colour, horizontal blur, vertical blur + paste + renormalise.  No atomics: repeated calls
// are bit-identical.
#include "common.cuh"

#define AUG_COLS 32
#define AUG_MAXK 6

struct AugNorm {
    float mean[3], stdv[3];
};

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

__device__ __forceinline__ float aug_gray(float r, float g, float b) {
    // torchvision: r.mul(0.2989).add_(g, alpha=0.587).add_(b, alpha=0.114)
    return __fadd_rn(__fadd_rn(__fmul_rn(r, 0.2989f), __fmul_rn(g, 0.587f)), __fmul_rn(b, 0.114f));
}

// _blend(image1, image2, ratio) = clamp(image1 * ratio + image2 * (1 - ratio), 0, 1)
__device__ __forceinline__ float aug_blend(float a, float b, float f) {
    return clamp01(__fadd_rn(__fmul_rn(a, f), __fmul_rn(b, __fsub_rn(1.f, f))));
}

__device__ __forceinline__ void aug_hue(float& r, float& g, float& b, float hue) {
    // torchvision _rgb_to_hsv / _hsv_to_rgb
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = maxc - minc;
    const float s = cr / (eqc ? 1.f : maxc);
    const float div = eqc ? 1.f : cr;
    const float rc = (maxc - r) / div, gc = (maxc - g) / div, bc = (maxc - b) / div;
    float h;
    if (maxc == r) h = bc - gc;
    else if (maxc == g) h = 2.f + rc - bc;
    else h = 4.f + gc - rc;
    h = fmodf(h * (1.f / 6.f) + 1.f, 1.f);
    h = h + hue;
    h = h - floorf(h);                         // remainder(1.0)
    const float v = maxc;
    const float h6 = h * 6.f;
    const float fi = floorf(h6);
    const float f = h6 - fi;
    int i = ((int)fi) % 6;
    if (i < 0) i += 6;
    const float sxf = s * f;
    const float q = clamp01((1.f - sxf) * v);
    const float t = clamp01((sxf + (1.f - s)) * v);
    const float p = clamp01((1.f - s) * v);
    switch (i) {
        case 0: r = v; g = t; b = p; break;
        case 1: r = q; g = v; b = p; break;
        case 2: r = p; g = v; b = t; break;
        case 3: r = p; g = q; b = v; break;
        case 4: r = t; g = p; b = v; break;
        default: r = v; g = p; b = q; break;
    }
}

__device__ __forceinline__ void aug_op(int op, const float* __restrict__ P, float gray_mean, float& r, float& g,
                                       float& b) {
    if (op == 0) {
        const float f = P[1];
        r = aug_blend(r, 0.f, f); g = aug_blend(g, 0.f, f); b = aug_blend(b, 0.f, f);
    } else if (op == 1) {
        const float f = P[2];
        r = aug_blend(r, gray_mean, f); g = aug_blend(g, gray_mean, f); b = aug_blend(b, gray_mean, f);
    } else if (op == 2) {
        const float f = P[3], gr = aug_gray(r, g, b);
        r = aug_blend(r, gr, f); g = aug_blend(g, gr, f); b = aug_blend(b, gr, f);
    } else {
        aug_hue(r, g, b, P[4]);
    }
}

__device__ __forceinline__ void aug_load(const float* __restrict__ weak, int i, int64_t HW, int64_t p, const AugNorm& nm,
                                         float& r, float& g, float& b) {
    const float* x = weak + (int64_t)i * 3 * HW + p;
    r = clamp01(__fadd_rn(__fmul_rn(x[0], nm.stdv[0]), nm.mean[0]));
    g = clamp01(__fadd_rn(__fmul_rn(x[HW], nm.stdv[1]), nm.mean[1]));
    b = clamp01(__fadd_rn(__fmul_rn(x[2 * HW], nm.stdv[2]), nm.mean[2]));
}

// grayscale sum of each view at contrast's position in its order (zero when the view has no jitter)
__global__ void __launch_bounds__(256)
aug_stats_kernel(const float* __restrict__ weak, const float* __restrict__ table, int ubs, int64_t HW, AugNorm nm,
                 double* __restrict__ part) {
    const int v = blockIdx.y;
    const float* P = table + (int64_t)v * AUG_COLS;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double acc = 0.0;
    if (P[0] != 0.f && p < HW) {
        float r, g, b;
        aug_load(weak, v % ubs, HW, p, nm, r, g, b);
        for (int k = 0; k < 4; ++k) {
            const int op = (int)P[5 + k];
            if (op == 1) break;
            aug_op(op, P, 0.f, r, g, b);
        }
        acc = (double)aug_gray(r, g, b);
    }
    __shared__ double wp[8];
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) wp[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += wp[k];
        part[(int64_t)v * gridDim.x + blockIdx.x] = s;
    }
}

// gray_mean[v] = (sum of view v's partials) / HW: one warp per view, lane-strided then a fixed shuffle tree
__global__ void __launch_bounds__(128)
aug_mean_kernel(const double* __restrict__ part, int nblk, int views, double inv_hw, float* __restrict__ gray_mean) {
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (v >= views) return;                  // warp-uniform
    double s = 0.0;
    for (int k = lane; k < nblk; k += 32) s += __ldg(part + (int64_t)v * nblk + k);
    s = warp_sum_d(s);
    if (lane == 0) gray_mean[v] = (float)(s * inv_hw);
}

__global__ void __launch_bounds__(256)
aug_colour_kernel(const float* __restrict__ weak, const float* __restrict__ table, const float* __restrict__ gray_mean,
                  int ubs, int64_t HW, AugNorm nm, float* __restrict__ out) {
    const int v = blockIdx.y;
    const float* P = table + (int64_t)v * AUG_COLS;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    float r, g, b;
    aug_load(weak, v % ubs, HW, p, nm, r, g, b);
    if (P[0] != 0.f) {
        const float m = gray_mean[v];
        for (int k = 0; k < 4; ++k) aug_op((int)P[5 + k], P, m, r, g, b);
    }
    if (P[9] != 0.f) r = g = b = aug_gray(r, g, b);
    float* o = out + (int64_t)v * 3 * HW + p;
    o[0] = r; o[HW] = g; o[2 * HW] = b;
}

__device__ __forceinline__ int aug_reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

__global__ void __launch_bounds__(256)
aug_hblur_kernel(const float* __restrict__ in, const float* __restrict__ table, int H, int W, float* __restrict__ out) {
    const int v = blockIdx.z, y = blockIdx.y;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const float* P = table + (int64_t)v * AUG_COLS;
    const int k = (int)P[10];
    const int64_t HW = (int64_t)H * W;
    for (int c = 0; c < 3; ++c) {
        const float* row = in + ((int64_t)v * 3 + c) * HW + (int64_t)y * W;
        float s;
        if (k == 0) {
            s = row[x];
        } else {
            s = 0.f;
            for (int j = -k; j <= k; ++j) s += P[16 + j + k] * row[aug_reflect(x + j, W)];
        }
        out[((int64_t)v * 3 + c) * HW + (int64_t)y * W + x] = s;
    }
}

__global__ void __launch_bounds__(256)
aug_vblur_paste_kernel(const float* __restrict__ in, const float* __restrict__ table, int ubs, int H, int W, AugNorm nm,
                       float* __restrict__ out) {
    const int v = blockIdx.z, y = blockIdx.y;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const float* P = table + (int64_t)v * AUG_COLS;
    int u = v;                                   // the view this pixel is taken from
    if (y >= (int)P[12] && y < (int)P[14] && x >= (int)P[13] && x < (int)P[15]) {
        const int k = v / ubs, i = v - k * ubs;
        u = k * ubs + (i + ubs / 2) % ubs;
    }
    const float* Q = table + (int64_t)u * AUG_COLS;
    const int kh = (int)Q[10];
    const int64_t HW = (int64_t)H * W;
    for (int c = 0; c < 3; ++c) {
        const float* plane = in + ((int64_t)u * 3 + c) * HW + x;
        float s;
        if (kh == 0) {
            s = plane[(int64_t)y * W];
        } else {
            s = 0.f;
            for (int j = -kh; j <= kh; ++j) s += Q[16 + j + kh] * plane[(int64_t)aug_reflect(y + j, H) * W];
        }
        out[((int64_t)v * 3 + c) * HW + (int64_t)y * W + x] = __fdiv_rn(__fsub_rn(s, nm.mean[c]), nm.stdv[c]);
    }
}

extern "C" int pxl_strong_aug(const float* weak, const float* table, int ubs, int H, int W, const double* mean3_host,
                              const double* std3_host, float* out, float* tmp_a, float* tmp_b, float* gray_mean,
                              void* stream) {
    if (!weak || !table || !out || !tmp_a || !tmp_b || !gray_mean || !mean3_host || !std3_host) return PXL_ERR_BAD_ARG;
    if (ubs <= 0 || H <= AUG_MAXK || W <= AUG_MAXK) return PXL_ERR_BAD_ARG;
    if (2 * ubs > 65535 || H > 65535) return PXL_ERR_UNSUPPORTED;
    AugNorm nm;
    for (int c = 0; c < 3; ++c) { nm.mean[c] = (float)mean3_host[c]; nm.stdv[c] = (float)std3_host[c]; }
    cudaStream_t st = (cudaStream_t)stream;
    const int views = 2 * ubs;
    const int64_t HW = (int64_t)H * W;
    dim3 grid((unsigned)pxl_cdiv(HW, 256), (unsigned)views);
    int rc = 0;
    double* part = (double*)pxl_workspace_(PXL_WS_STRONG_AUG, stream, (size_t)grid.x * views * sizeof(double), &rc);
    if (rc) return rc;
    aug_stats_kernel<<<grid, 256, 0, st>>>(weak, table, ubs, HW, nm, part);
    PXL_CHECK_LAUNCH();
    aug_mean_kernel<<<(unsigned)pxl_cdiv(views, 4), 128, 0, st>>>(part, (int)grid.x, views, 1.0 / (double)HW, gray_mean);
    PXL_CHECK_LAUNCH();
    aug_colour_kernel<<<grid, 256, 0, st>>>(weak, table, gray_mean, ubs, HW, nm, tmp_a);
    PXL_CHECK_LAUNCH();
    dim3 rows((unsigned)pxl_cdiv(W, 256), (unsigned)H, (unsigned)views);
    aug_hblur_kernel<<<rows, 256, 0, st>>>(tmp_a, table, H, W, tmp_b);
    PXL_CHECK_LAUNCH();
    aug_vblur_paste_kernel<<<rows, 256, 0, st>>>(tmp_b, table, ubs, H, W, nm, out);
    PXL_CHECK_LAUNCH();
    return 0;
}
