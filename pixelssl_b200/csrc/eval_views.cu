// Multi-view evaluation (task/sseg/evaluation.py): view images cut into tiles, the tiles' softmax merged back, the
// views' probabilities resized and summed, the ensemble's mean and clamped log.
//
// A view is (s, f): the batch x [n,3,H,W] resized to hv x wv (bilinear, align_corners=True; a copy when s = 1) and
// flipped along W if f.  Its tiles are UniMatch's sliding window: row origins k*sh for k = 0, 1, ... while k*sh < hv,
// tile height min(gh, hv - k*sh), the same along the columns ('whole' is one tile: gh = sh = hv, gw = sw = wv).
// Rows with k*sh + gh <= hv (a prefix k < nfull_r) have the full height; every later row ("tail") has a height of
// its own.  The row classes are [full rows (if any), tail row nfull_r, tail row nfull_r + 1, ...] (at most three,
// since sh = int(2g/3) leaves room for at most two tails), likewise the column classes; a shape group is a (row
// class, column class) pair, groups numbered row class major.  A group's tiles are the row-major product of its rows
// and columns, stored tile-major: tile t of sample b is row t*n + b of the group's [T*n, ., th, tw] tensor.
//
// All maps are planar fp32, C <= 32 classes.  Every value is written by one thread in a fixed order: no atomics,
// results are bit-identical across runs.
#include <float.h>

#include "resample.cuh"

#define EV_MAXC 32
#define EV_MAXG 9

struct EvAxis {          // one axis of a view's tiling
    int len;             // view length (hv or wv)
    int g;               // tile length
    int stride;
    int n;               // number of origins: ceil(len / stride)
    int nfull;           // origins whose tile has the full length g
};

static inline EvAxis ev_axis(int len, int g, int stride) {
    EvAxis a;
    a.len = len; a.g = g; a.stride = stride;
    a.n = (int)pxl_cdiv(len, stride);
    a.nfull = len >= g ? (len - g) / stride + 1 : 0;
    if (a.nfull > a.n) a.nfull = a.n;
    return a;
}

static inline int ev_classes(const EvAxis& a) { return (a.nfull > 0 ? 1 : 0) + (a.n - a.nfull); }

static inline bool ev_axis_ok(int len, int g, int stride) {
    if (len <= 0 || g <= 0 || stride <= 0 || stride > g) return false;
    const EvAxis a = ev_axis(len, g, stride);
    return ev_classes(a) <= 3;
}

// ---- 1. tiles of one shape group ----------------------------------------------------------------------------------
// out[(t*n + b), ch, ty, tx] = view(b, ch, r + ty, c + tx), (r, c) = (r0 + (t / nc)*sh, c0 + (t % nc)*sw)
__global__ void __launch_bounds__(128)
eval_tiles_kernel(const float* __restrict__ x, float* __restrict__ out, int n, int H, int W, int hv, int wv, bool flip,
                  int r0, int nc, int c0, int sh, int sw, int th, int tw, bool resize, float fy_scale, float fx_scale) {
    const int tx = blockIdx.x * blockDim.x + threadIdx.x;
    if (tx >= tw) return;
    const int ty = blockIdx.y;
    const int tb = blockIdx.z;                  // t*n + b
    const int t = tb / n, b = tb - t * n;
    const int vy = r0 + (t / nc) * sh + ty;
    int vx = c0 + (t % nc) * sw + tx;
    if (flip) vx = wv - 1 - vx;                 // the flipped view's column vx is the resized image's column wv-1-vx
    const int64_t HW = (int64_t)H * W, thw = (int64_t)th * tw;
    const float* xb = x + (int64_t)b * 3 * HW;
    float* ob = out + (int64_t)tb * 3 * thw + (int64_t)ty * tw + tx;
    if (!resize) {
        const float* p = xb + (int64_t)vy * W + vx;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) ob[ch * thw] = __ldg(p + ch * HW);
        return;
    }
    const float fy = src_index(fy_scale, vy, true), fx = src_index(fx_scale, vx, true);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly1 = fy - (float)y0, lx1 = fx - (float)x0;
    const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float* pc = xb + ch * HW;
        ob[ch * thw] = ly0 * (lx0 * __ldg(pc + (int64_t)y0 * W + x0) + lx1 * __ldg(pc + (int64_t)y0 * W + x1)) +
                       ly1 * (lx0 * __ldg(pc + (int64_t)y1 * W + x0) + lx1 * __ldg(pc + (int64_t)y1 * W + x1));
    }
}

extern "C" int pxl_eval_tiles(const float* x, float* out, int n, int H, int W, int hv, int wv, int flip, int r0, int nr,
                              int c0, int nc, int sh, int sw, int th, int tw, void* stream) {
    if (!x || !out || n <= 0 || H <= 0 || W <= 0 || hv <= 0 || wv <= 0 || nr <= 0 || nc <= 0 || sh <= 0 || sw <= 0 ||
        th <= 0 || tw <= 0 || r0 < 0 || c0 < 0)
        return PXL_ERR_BAD_ARG;
    if (r0 + (int64_t)(nr - 1) * sh + th > hv || c0 + (int64_t)(nc - 1) * sw + tw > wv) return PXL_ERR_BAD_ARG;
    if ((int64_t)nr * nc * n > 65535 || th > 65535) return PXL_ERR_UNSUPPORTED;
    const bool resize = hv != H || wv != W;
    dim3 grid((unsigned)pxl_cdiv(tw, 128), (unsigned)th, (unsigned)(nr * nc * n));
    eval_tiles_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x, out, n, H, W, hv, wv, flip != 0, r0, nc, c0, sh, sw, th,
                                                               tw, resize, resize_scale(H, hv, 1), resize_scale(W, wv, 1));
    PXL_CHECK_LAUNCH();
    return 0;
}

// ---- 2. merge of one view's tiles ---------------------------------------------------------------------------------
struct EvGroups {         // __grid_constant__: indexed in parameter space, no local-memory copy
    const float* p[EV_MAXG];
};

// class of origin k on an axis -> (class index, first origin of the class, origins in the class, tile length)
__device__ __forceinline__ void ev_class_of(const EvAxis& a, int k, int& cls, int& first, int& count, int& len) {
    const int r = k * a.stride;
    if (k < a.nfull) { cls = 0; first = 0; count = a.nfull; len = a.g; return; }
    cls = (a.nfull > 0 ? 1 : 0) + (k - a.nfull);
    first = k; count = 1;
    len = a.len - r;
}

// out[b, c, y, xo] (+)= sum over the tiles covering view pixel (y, xv) in row-major tile order of softmax(tile logits),
// xv = flip ? wv-1-xo : xo (the un-flip)
__global__ void __launch_bounds__(128)
eval_merge_kernel(const __grid_constant__ EvGroups groups, int n, int C, EvAxis ay, EvAxis ax, int ncls_x, bool flip,
                  bool accumulate, float* __restrict__ out) {
    const int xo = blockIdx.x * blockDim.x + threadIdx.x;
    if (xo >= ax.len) return;
    const int y = blockIdx.y, b = blockIdx.z;
    const int xv = flip ? ax.len - 1 - xo : xo;
    // rows k with k*stride <= y < k*stride + g (every origin is < len, and y < len)
    const int k_lo = y >= ay.g ? (y - ay.g) / ay.stride + 1 : 0, k_hi = y / ay.stride;
    const int l_lo = xv >= ax.g ? (xv - ax.g) / ax.stride + 1 : 0, l_hi = xv / ax.stride;
    float acc[EV_MAXC];
#pragma unroll
    for (int c = 0; c < EV_MAXC; ++c) acc[c] = 0.f;
    for (int k = k_lo; k <= k_hi; ++k) {
        int rc, rfirst, rcount, th;
        ev_class_of(ay, k, rc, rfirst, rcount, th);
        const int ty = y - k * ay.stride;
        for (int l = l_lo; l <= l_hi; ++l) {
            int cc, cfirst, ccount, tw;
            ev_class_of(ax, l, cc, cfirst, ccount, tw);
            const int tx = xv - l * ax.stride;
            const int t = (k - rfirst) * ccount + (l - cfirst);
            const int64_t thw = (int64_t)th * tw;
            const float* p = groups.p[rc * ncls_x + cc] + ((int64_t)t * n + b) * C * thw + (int64_t)ty * tw + tx;
            float v[EV_MAXC];
            float m = -INFINITY;
#pragma unroll
            for (int c = 0; c < EV_MAXC; ++c) {
                if (c < C) { v[c] = __ldg(p + c * thw); m = fmaxf(m, v[c]); }
            }
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < EV_MAXC; ++c) {
                if (c < C) { v[c] = expf(v[c] - m); s += v[c]; }
            }
#pragma unroll
            for (int c = 0; c < EV_MAXC; ++c) {
                if (c < C) acc[c] += v[c] / s;
            }
        }
    }
    const int64_t HW = (int64_t)ay.len * ax.len;
    float* o = out + (int64_t)b * C * HW + (int64_t)y * ax.len + xo;
#pragma unroll
    for (int c = 0; c < EV_MAXC; ++c) {
        if (c < C) {
            if (accumulate) o[c * HW] += acc[c];
            else o[c * HW] = acc[c];
        }
    }
}

extern "C" int pxl_eval_merge(const float* const* group_logits_host, int ngroups, int n, int C, int hv, int wv, int gh,
                              int gw, int sh, int sw, int flip, int accumulate, float* out, void* stream) {
    if (!group_logits_host || !out || n <= 0 || C <= 0 || hv <= 0 || wv <= 0) return PXL_ERR_BAD_ARG;
    if (C > EV_MAXC) return PXL_ERR_UNSUPPORTED;
    if (!ev_axis_ok(hv, gh, sh) || !ev_axis_ok(wv, gw, sw)) return PXL_ERR_BAD_ARG;
    const EvAxis ay = ev_axis(hv, gh, sh), ax = ev_axis(wv, gw, sw);
    const int ncls_y = ev_classes(ay), ncls_x = ev_classes(ax);
    if (ngroups != ncls_y * ncls_x) return PXL_ERR_BAD_ARG;
    EvGroups groups = {};
    for (int i = 0; i < ngroups; ++i) {
        if (!group_logits_host[i]) return PXL_ERR_BAD_ARG;
        groups.p[i] = group_logits_host[i];
    }
    if (hv > 65535 || n > 65535) return PXL_ERR_UNSUPPORTED;
    dim3 grid((unsigned)pxl_cdiv(wv, 128), (unsigned)hv, (unsigned)n);
    eval_merge_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(groups, n, C, ay, ax, ncls_x, flip != 0, accumulate != 0,
                                                               out);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ---- 3. S (+)= bilinear_ac(P_v) -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
eval_view_add_kernel(const float* __restrict__ P, float* __restrict__ S, int C, int hv, int wv, int H, int W, float sy,
                     float sx, bool accumulate) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const int y = blockIdx.y, b = blockIdx.z;
    const float fy = src_index(sy, y, true), fx = src_index(sx, x, true);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < hv - 1 ? 1 : 0), x1 = x0 + (x0 < wv - 1 ? 1 : 0);
    const float ly1 = fy - (float)y0, lx1 = fx - (float)x0;
    const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const int64_t hw = (int64_t)hv * wv, HW = (int64_t)H * W;
    const float* pb = P + (int64_t)b * C * hw;
    float* s = S + (int64_t)b * C * HW + (int64_t)y * W + x;
    for (int c = 0; c < C; ++c) {
        const float* pc = pb + c * hw;
        const float v = ly0 * (lx0 * __ldg(pc + (int64_t)y0 * wv + x0) + lx1 * __ldg(pc + (int64_t)y0 * wv + x1)) +
                        ly1 * (lx0 * __ldg(pc + (int64_t)y1 * wv + x0) + lx1 * __ldg(pc + (int64_t)y1 * wv + x1));
        if (accumulate) s[c * HW] += v;
        else s[c * HW] = v;
    }
}

extern "C" int pxl_eval_view_add(const float* P, float* S, int n, int C, int hv, int wv, int H, int W, int accumulate,
                                 void* stream) {
    if (!P || !S || n <= 0 || C <= 0 || hv <= 0 || wv <= 0 || H <= 0 || W <= 0) return PXL_ERR_BAD_ARG;
    if (C > EV_MAXC) return PXL_ERR_UNSUPPORTED;
    if (H > 65535 || n > 65535) return PXL_ERR_UNSUPPORTED;
    dim3 grid((unsigned)pxl_cdiv(W, 128), (unsigned)H, (unsigned)n);
    eval_view_add_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(P, S, C, hv, wv, H, W, resize_scale(hv, H, 1),
                                                                  resize_scale(wv, W, 1), accumulate != 0);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ---- 4. mean = S / V, logmean = log(max(mean, FLT_MIN)) --------------------------------------------------------------
__global__ void __launch_bounds__(256)
eval_finish_kernel(const float* __restrict__ S, float* __restrict__ mean, float* __restrict__ logmean, int64_t count,
                   float V) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const float m = __ldg(S + i) / V;
        mean[i] = m;
        logmean[i] = logf(m < FLT_MIN ? FLT_MIN : m);      // NaN stays NaN, as torch.clamp(min=FLT_MIN)
    }
}

extern "C" int pxl_eval_finish(const float* S, float* mean, float* logmean, int64_t count, int V, void* stream) {
    if (!S || !mean || !logmean || count <= 0 || V <= 0) return PXL_ERR_BAD_ARG;
    int64_t blocks = pxl_cdiv(count, 256);
    if (blocks > (int64_t)PXL_NUM_SMS * 16) blocks = (int64_t)PXL_NUM_SMS * 16;
    eval_finish_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(S, mean, logmean, count, (float)V);
    PXL_CHECK_LAUNCH();
    return 0;
}
