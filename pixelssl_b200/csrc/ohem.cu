// Online hard example mining (OHEM) cross-entropy: the "probability OHEM" of ProbOhemCrossEntropy2d, as CPS and
// UniMatch train their supervised term.  Over the whole batch of one call:
//   q      = softmax(logits)[y] on valid pixels (y = trunc(label), y != ignore, 0 <= y < C), 1 on the others
//   V      = number of valid pixels
//   k == 0, k > V or V == 0: every valid pixel is kept (T reported as +inf)
//   else   t_k = k-th smallest q over all n*HW pixels (NaN last, as torch.sort), T = t_k > tau ? t_k : tau,
//          kept = valid && q <= T
//   per_sample[i] = n * sum_{kept in i} (logsumexp - x_y) / K,  grad = g_i * n / K * (softmax - onehot) on kept pixels
// Nothing is read back to the host: V, t_k, T and K are device scalars (stats[4], fp64) the later launches read.
// The only synchronisation is the one every per-block-partials kernel here shares: the scratch buffer
// (pxl_workspace_) grows with cudaFree + cudaMalloc, which synchronise the device, when a call needs more than any
// earlier call on the stream; in steady state (the same shapes every step) no call synchronises.
//
// Launches of one call (stream order):
//   1. memset of the counters and histograms;
//   2. ohem_pixel_kernel: one thread per pixel, writes q, counts V, #(q <= tau) and #(valid, q <= tau), and builds
//      the level-1 radix histogram of the keys (the fp32 bits of q: order-preserving since q >= 0; NaN -> 0x7fffffff)
//      in shared memory, flushed with integer atomics;
//   3. ohem_find_kernel (level 1): resolves the keep-all cases and the exact early exit (#(q <= tau) >= k holds
//      exactly when t_k <= tau, and then T = tau), else picks the bin holding rank k;
//   4-7. ohem_refine_kernel + ohem_find_kernel for levels 2 and 3 over the keys of the selected bin (no-ops after an
//      early exit): the selection is exact, t_k == torch.sort(q)[k-1] bit for bit;
//   8. ohem_loss_kernel: masked CE and its gradient with T and K read from stats; fp64 per-block partials;
//   9. ohem_sum_kernel: per-sample sums in a fixed order.  No floating-point atomics: repeated calls are bit-identical.
// Key bits per level: [30:20] (2048 bins; bit 31 is always 0), [19:8] (4096 bins), [7:0] (256 bins).
//   algorithmic traffic: pass 2 reads 4*C + 4 B/pixel and writes 4; pass 8 reads 4*C + 8 B/pixel and writes 4*C when
//   the gradient is written; each refinement pass that runs reads 4 B/pixel.
#include "common.cuh"
#include <math_constants.h>

#define OHEM_MAXC 32
#define OHEM_THREADS 256
#define OHEM_PIX_PER_THREAD 8
#define OHEM_L1_BINS 2048
#define OHEM_L2_BINS 4096
#define OHEM_L3_BINS 256
#define OHEM_FIND_THREADS 1024

struct OhemState {
    unsigned long long n_valid, n_le_tau, n_valid_le_tau;   // counted by the pixel pass
    unsigned long long below;                               // keys strictly below the selected prefix
    unsigned long long rank;                                // rank of t_k among the keys of the prefix (1-based)
    unsigned int prefix;                                    // key bits selected so far
    int done;                                               // T and K are final (keep-all or early exit)
    unsigned int hist1[OHEM_L1_BINS], hist2[OHEM_L2_BINS], hist3[OHEM_L3_BINS];   // 32-bit: n*HW < 2^32 is checked
};

__device__ __forceinline__ unsigned int ohem_key(float q) { return q != q ? 0x7fffffffu : __float_as_uint(q); }

// warp-aggregated shared-memory histogram increment: lanes holding the same bin add once (ties and the confident
// pixels' q ~ 1 crowd a few bins)
__device__ __forceinline__ void ohem_hist_add(unsigned int* h, unsigned int bin, bool hit) {
    const unsigned int act = __ballot_sync(0xffffffffu, hit);
    if (hit) {
        const unsigned int peers = __match_any_sync(act, bin);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&h[bin], (unsigned int)__popc(peers));
    }
}

__device__ __forceinline__ void ohem_flush(const unsigned int* h, unsigned int* g, int nb) {
    for (int i = threadIdx.x; i < nb; i += blockDim.x)
        if (h[i]) atomicAdd(&g[i], h[i]);
}

__global__ void __launch_bounds__(OHEM_THREADS)
ohem_pixel_kernel(const float* __restrict__ logits, const float* __restrict__ labels, int C, int64_t HW,
                  int ignore_index, float tau, float* __restrict__ q_out, OhemState* __restrict__ st) {
    __shared__ unsigned int h[OHEM_L1_BINS];
    __shared__ unsigned int cnt[3];
    for (int i = threadIdx.x; i < OHEM_L1_BINS; i += OHEM_THREADS) h[i] = 0;
    if (threadIdx.x < 3) cnt[threadIdx.x] = 0;
    __syncthreads();
    const int b = blockIdx.y;
    const float* lg = logits + (int64_t)b * C * HW;
    unsigned int n_valid = 0, n_le = 0, n_valid_le = 0;
    for (int it = 0; it < OHEM_PIX_PER_THREAD; ++it) {
        const int64_t p = ((int64_t)blockIdx.x * OHEM_PIX_PER_THREAD + it) * OHEM_THREADS + threadIdx.x;
        const bool in = p < HW;
        unsigned int key = 0;
        if (in) {
            float v[OHEM_MAXC];
            float m = -CUDART_INF_F;
#pragma unroll
            for (int c = 0; c < OHEM_MAXC; ++c)
                if (c < C) { v[c] = lg[(int64_t)c * HW + p]; m = fmaxf(m, v[c]); }
            const long long lab = (long long)labels[(int64_t)b * HW + p];     // .long(): truncation toward zero
            const bool valid = (lab != (long long)ignore_index) && lab >= 0 && lab < C;
            float se = 0.f, e_y = 0.f;
#pragma unroll
            for (int c = 0; c < OHEM_MAXC; ++c)
                if (c < C) {
                    const float e = expf(v[c] - m);
                    se += e;
                    if (c == (int)lab) e_y = e;      // select in the unrolled loop: no dynamic register indexing
                }
            const float q = valid ? e_y / se : 1.f;
            q_out[(int64_t)b * HW + p] = q;
            key = ohem_key(q);
            n_valid += valid;
            n_le += q <= tau;
            n_valid_le += valid && q <= tau;
        }
        ohem_hist_add(h, key >> 20, in);
    }
    n_valid = __reduce_add_sync(0xffffffffu, n_valid);
    n_le = __reduce_add_sync(0xffffffffu, n_le);
    n_valid_le = __reduce_add_sync(0xffffffffu, n_valid_le);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&cnt[0], n_valid);
        atomicAdd(&cnt[1], n_le);
        atomicAdd(&cnt[2], n_valid_le);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (cnt[0]) atomicAdd(&st->n_valid, (unsigned long long)cnt[0]);
        if (cnt[1]) atomicAdd(&st->n_le_tau, (unsigned long long)cnt[1]);
        if (cnt[2]) atomicAdd(&st->n_valid_le_tau, (unsigned long long)cnt[2]);
    }
    ohem_flush(h, st->hist1, OHEM_L1_BINS);
}

// Histogram of the next level's key bits over the keys whose bits above ``hi_shift`` equal the selected prefix.
template <int NB>
__global__ void __launch_bounds__(OHEM_THREADS)
ohem_refine_kernel(const float* __restrict__ q, int64_t N, OhemState* __restrict__ st, int hi_shift, int shift) {
    if (st->done) return;                     // block-uniform: T and K are already known
    unsigned int* hist = NB == OHEM_L2_BINS ? st->hist2 : st->hist3;
    __shared__ unsigned int h[NB];
    for (int i = threadIdx.x; i < NB; i += OHEM_THREADS) h[i] = 0;
    __syncthreads();
    const unsigned int want = st->prefix >> hi_shift;
    const int64_t stride = (int64_t)gridDim.x * OHEM_THREADS;
    const int64_t iters = (N + stride - 1) / stride;          // the same trip count in every lane (ballots)
    int64_t i = (int64_t)blockIdx.x * OHEM_THREADS + threadIdx.x;
    for (int64_t t = 0; t < iters; ++t, i += stride) {
        unsigned int key = 0;
        bool hit = false;
        if (i < N) {
            key = ohem_key(__ldg(q + i));
            hit = (key >> hi_shift) == want;
        }
        ohem_hist_add(h, (key >> shift) & (NB - 1), hit);
    }
    __syncthreads();
    ohem_flush(h, hist, NB);
}

// One CTA: find the bin of ``hist`` holding rank st->rank, narrow the prefix to it; level 1 first settles the
// keep-all cases and the early exit, the last level settles T and K.  stats = V, K, T, t_k (t_k NaN when the selection
// was not needed).
__global__ void __launch_bounds__(OHEM_FIND_THREADS)
ohem_find_kernel(OhemState* __restrict__ st, int level, int64_t k, int64_t total, float tau,
                 double* __restrict__ stats) {
    __shared__ unsigned long long scan[OHEM_FIND_THREADS / 32];
    const int nb = level == 1 ? OHEM_L1_BINS : level == 2 ? OHEM_L2_BINS : OHEM_L3_BINS;
    const int shift = level == 1 ? 20 : level == 2 ? 8 : 0;
    const unsigned int* hist = level == 1 ? st->hist1 : level == 2 ? st->hist2 : st->hist3;
    const unsigned long long V = st->n_valid;
    if (level == 1) {
        bool fin = true;
        double K = 0.0, T = 0.0;
        if (V == 0 || k == 0 || (unsigned long long)k > V) { K = (double)V; T = CUDART_INF; }
        else if (st->n_le_tau >= (unsigned long long)k) { K = (double)st->n_valid_le_tau; T = (double)tau; }
        else fin = false;
        if (fin) {
            if (threadIdx.x == 0) {
                stats[0] = (double)V; stats[1] = K; stats[2] = T; stats[3] = CUDART_NAN;
                st->done = 1;
            }
            return;
        }
    } else if (st->done) {
        return;
    }
    const unsigned long long r = level == 1 ? (unsigned long long)k : st->rank;
    const unsigned long long below = level == 1 ? 0ull : st->below;
    const unsigned int prefix = level == 1 ? 0u : st->prefix;
    // each thread owns a contiguous run of bins; exclusive scan of the run sums across the block
    const int per = (nb + OHEM_FIND_THREADS - 1) / OHEM_FIND_THREADS;
    const int b0 = threadIdx.x * per;
    unsigned long long own = 0;
    for (int j = 0; j < per; ++j)
        if (b0 + j < nb) own += hist[b0 + j];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) scan[warp] = incl;
    __syncthreads();
    unsigned long long base = 0;
    for (int w = 0; w < warp; ++w) base += scan[w];
    const unsigned long long excl = base + incl - own;
    if (excl < r && r <= excl + own) {            // exactly one thread
        unsigned long long c = excl;
        int bin = b0;
        for (int j = 0; j < per; ++j) {
            const unsigned long long hb = hist[b0 + j];
            if (c + hb >= r) { bin = b0 + j; break; }
            c += hb;
        }
        const unsigned int pre = prefix | ((unsigned int)bin << shift);
        if (level < 3) {
            st->prefix = pre;
            st->below = below + c;
            st->rank = r - c;
            return;
        }
        // the key is complete: hist[bin] keys equal t_k, below + c are smaller
        const float tk = __uint_as_float(pre);
        const unsigned long long le = below + c + hist[bin];
        const bool sel = tk > tau;                // false for a NaN t_k
        // invalid pixels carry q = 1: they are below or at t_k exactly when t_k >= 1
        const unsigned long long invalid_le = (1.f <= tk) ? (unsigned long long)total - V : 0ull;
        stats[0] = (double)V;
        stats[1] = sel ? (double)(le - invalid_le) : (double)st->n_valid_le_tau;
        stats[2] = sel ? (double)tk : (double)tau;
        stats[3] = (double)tk;
        st->done = 1;
    }
}

// masked CE of the kept pixels; gradient g_b * n / K * (softmax - onehot) on kept pixels, 0 elsewhere
template <bool WRITE_GRAD>
__global__ void __launch_bounds__(OHEM_THREADS)
ohem_loss_kernel(const float* __restrict__ logits, const float* __restrict__ labels, const float* __restrict__ q,
                 const double* __restrict__ stats, int n, int C, int64_t HW, int ignore_index,
                 const float* __restrict__ upstream, float upstream_const, double* __restrict__ part,
                 float* __restrict__ grad) {
    const int b = blockIdx.y;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double loss = 0.0;
    if (p < HW) {
        const double T = stats[2];
        const float qp = q[(int64_t)b * HW + p];
        const long long lab = (long long)labels[(int64_t)b * HW + p];
        const int y = (int)lab;
        const bool valid = (lab != (long long)ignore_index) && lab >= 0 && lab < C;
        const bool kept = valid && (isinf(T) || (double)qp <= T);
        const int64_t base = (int64_t)b * C * HW + p;
        if (kept) {
            float v[OHEM_MAXC];
            float m = -CUDART_INF_F;
#pragma unroll
            for (int c = 0; c < OHEM_MAXC; ++c)
                if (c < C) { v[c] = logits[base + (int64_t)c * HW]; m = fmaxf(m, v[c]); }
            float se = 0.f, x_y = 0.f;
#pragma unroll
            for (int c = 0; c < OHEM_MAXC; ++c)
                if (c < C) {
                    if (c == y) x_y = v[c];
                    v[c] = expf(v[c] - m);
                    se += v[c];
                }
            loss = (double)((logf(se) + m) - x_y);
            if (WRITE_GRAD) {
                const float g = (upstream ? upstream[b] : upstream_const) * ((float)n / (float)stats[1]);
                const float inv = g / se;
#pragma unroll
                for (int c = 0; c < OHEM_MAXC; ++c)
                    if (c < C) {
                        float gv = v[c] * inv;
                        if (c == y) gv -= g;
                        grad[base + (int64_t)c * HW] = gv;
                    }
            }
        } else if (WRITE_GRAD) {
            for (int c = 0; c < C; ++c) grad[base + (int64_t)c * HW] = 0.f;
        }
    }
    __shared__ double wp[OHEM_THREADS / 32];
    loss = warp_sum_d(loss);
    if ((threadIdx.x & 31) == 0) wp[threadIdx.x >> 5] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < OHEM_THREADS / 32; ++i) s += wp[i];
        part[(int64_t)b * gridDim.x + blockIdx.x] = s;
    }
}

// per_sample[i] = n * (sum of row i's partials) / K.  One warp per row: lane j adds partials j, j+32, ... in order,
// then a fixed shuffle tree.  K == 0 (no valid pixel) gives 0/0 = NaN, as torch's mean-reduced CE.
#define OHEM_SUM_ROWS 4
__global__ void __launch_bounds__(32 * OHEM_SUM_ROWS)
ohem_sum_kernel(const double* __restrict__ part, int nblk, int n, const double* __restrict__ stats,
                float* __restrict__ per_sample) {
    const int i = blockIdx.x * OHEM_SUM_ROWS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;                        // warp-uniform
    double s = 0.0;
    for (int k = lane; k < nblk; k += 32) s += __ldg(part + (int64_t)i * nblk + k);
    s = warp_sum_d(s);
    if (lane == 0) per_sample[i] = (float)(s * (double)n / stats[1]);
}

static int ohem_loss_launch(const float* logits, const float* labels, const float* q, const double* stats, int n,
                            int C, int64_t HW, int ignore_index, const float* upstream, float upstream_const,
                            float* per_sample, float* grad, cudaStream_t st, double* part) {
    dim3 grid((unsigned)pxl_cdiv(HW, OHEM_THREADS), (unsigned)n);
    if (grad) ohem_loss_kernel<true><<<grid, OHEM_THREADS, 0, st>>>(logits, labels, q, stats, n, C, HW, ignore_index,
                                                                    upstream, upstream_const, part, grad);
    else ohem_loss_kernel<false><<<grid, OHEM_THREADS, 0, st>>>(logits, labels, q, stats, n, C, HW, ignore_index,
                                                                nullptr, 0.f, part, nullptr);
    PXL_CHECK_LAUNCH();
    ohem_sum_kernel<<<(unsigned)pxl_cdiv(n, OHEM_SUM_ROWS), 32 * OHEM_SUM_ROWS, 0, st>>>(part, (int)grid.x, n, stats,
                                                                                         per_sample);
    PXL_CHECK_LAUNCH();
    return 0;
}

static size_t ohem_state_bytes() { return (sizeof(OhemState) + 255) & ~(size_t)255; }

static bool ohem_args_ok(const float* logits, const float* labels, const float* q, const double* stats, int n, int C,
                         int64_t HW) {
    return logits && labels && q && stats && n > 0 && C > 0 && HW > 0;
}

extern "C" int pxl_ohem_ce(const float* logits, const float* labels, int n, int C, int64_t HW, int ignore_index,
                           float thresh, int64_t min_kept, float* per_sample, float* grad_logits,
                           float upstream_const, float* q, double* stats, void* stream) {
    if (!ohem_args_ok(logits, labels, q, stats, n, C, HW) || !per_sample || min_kept < 0 || !isfinite(thresh))
        return PXL_ERR_BAD_ARG;
    // the histogram bins are 32-bit counts: a batch of 2^32 pixels or more could wrap one
    if (C > OHEM_MAXC || n > 65535 || (int64_t)n * HW >= ((int64_t)1 << 32)) return PXL_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t nloss = pxl_cdiv(HW, OHEM_THREADS);
    int rc = 0;
    char* ws = (char*)pxl_workspace_(PXL_WS_OHEM, stream, ohem_state_bytes() + (size_t)nloss * n * sizeof(double), &rc);
    if (rc) return rc;
    OhemState* sta = (OhemState*)ws;
    double* part = (double*)(ws + ohem_state_bytes());
    cudaError_t e = cudaMemsetAsync(sta, 0, sizeof(OhemState), s);
    if (e != cudaSuccess) return (int)e;
    const int64_t N = (int64_t)n * HW;
    dim3 grid((unsigned)pxl_cdiv(HW, (int64_t)OHEM_THREADS * OHEM_PIX_PER_THREAD), (unsigned)n);
    ohem_pixel_kernel<<<grid, OHEM_THREADS, 0, s>>>(logits, labels, C, HW, ignore_index, thresh, q, sta);
    PXL_CHECK_LAUNCH();
    const unsigned rgrid = (unsigned)(pxl_cdiv(N, OHEM_THREADS) < PXL_NUM_SMS * 4 ? pxl_cdiv(N, OHEM_THREADS)
                                                                                    : PXL_NUM_SMS * 4);
    ohem_find_kernel<<<1, OHEM_FIND_THREADS, 0, s>>>(sta, 1, min_kept, N, thresh, stats);
    PXL_CHECK_LAUNCH();
    ohem_refine_kernel<OHEM_L2_BINS><<<rgrid, OHEM_THREADS, 0, s>>>(q, N, sta, 20, 8);
    PXL_CHECK_LAUNCH();
    ohem_find_kernel<<<1, OHEM_FIND_THREADS, 0, s>>>(sta, 2, min_kept, N, thresh, stats);
    PXL_CHECK_LAUNCH();
    ohem_refine_kernel<OHEM_L3_BINS><<<rgrid, OHEM_THREADS, 0, s>>>(q, N, sta, 8, 0);
    PXL_CHECK_LAUNCH();
    ohem_find_kernel<<<1, OHEM_FIND_THREADS, 0, s>>>(sta, 3, min_kept, N, thresh, stats);
    PXL_CHECK_LAUNCH();
    return ohem_loss_launch(logits, labels, q, stats, n, C, HW, ignore_index, nullptr, upstream_const, per_sample,
                            grad_logits, s, part);
}

extern "C" int pxl_ohem_ce_bwd(const float* logits, const float* labels, const float* q, const double* stats, int n,
                               int C, int64_t HW, int ignore_index, const float* upstream, float* per_sample,
                               float* grad_logits, void* stream) {
    if (!ohem_args_ok(logits, labels, q, stats, n, C, HW) || !upstream || !per_sample || !grad_logits)
        return PXL_ERR_BAD_ARG;
    if (C > OHEM_MAXC || n > 65535) return PXL_ERR_UNSUPPORTED;
    const int64_t nloss = pxl_cdiv(HW, OHEM_THREADS);
    int rc = 0;
    char* ws = (char*)pxl_workspace_(PXL_WS_OHEM, stream, ohem_state_bytes() + (size_t)nloss * n * sizeof(double), &rc);
    if (rc) return rc;
    return ohem_loss_launch(logits, labels, q, stats, n, C, HW, ignore_index, upstream, 0.f, per_sample, grad_logits,
                            (cudaStream_t)stream, (double*)(ws + ohem_state_bytes()));
}
