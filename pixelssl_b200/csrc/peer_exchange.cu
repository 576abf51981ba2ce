// Cross-GPU BatchNorm statistics exchange over NVLink peer memory, fused with the BN "finalize".
//
// The reference synchronises BN batch statistics across replicas for every BN layer of every forward and backward
// (sync_batchnorm/batchnorm.py:55-78, comm.py).  With one process per GPU that is ~300 tiny all-reduces per MT step
// (2C fp64 values each); through NCCL each costs a launch + ~15 us of latency on the critical path.  Here every
// rank owns a small mailbox in device memory, mapped into its peers with CUDA IPC.  ONE single-CTA kernel per
// exchange
//   1. stores this rank's partial sums into slot (seq % NSLOT), lane `rank`, of EVERY rank's mailbox (P2P stores
//      over NVLink / NVSwitch) and then publishes flag[rank] = seq with a system-scope release,
//   2. spins until its own mailbox holds flag[q] == seq for every rank q,
//   3. adds the `world` lanes in rank order (so all ranks get bit-identical totals),
//   4. optionally finishes the layer: mean / inv_std / scale / shift and the running statistics
//      (= pxl_bn_finalize, batchnorm.py:113-125), saving a second launch.
// A rank can be at most one exchange ahead of the slowest one (it needs everybody's lane to finish), so two slots
// would do; four are used.  All waits are bounded; on expiry the kernel raises *err and returns.
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"
#include "../../include/pixelssl_b200.h"

#define PX_NSLOT 4
#define PX_MAXW 8
#define PX_MAXN 4096          // 2 * 2048 channels

struct PxSlot {
    double data[PX_MAXW][PX_MAXN];
    unsigned long long flag[PX_MAXW];
    unsigned long long pad[8];
};
struct PxMailbox { PxSlot slot[PX_NSLOT]; };
struct PxPeers { PxMailbox* box[PX_MAXW]; };

extern "C" int pxl_peer_alloc(void** ptr) {
    if (!ptr) return PXL_ERR_BAD_ARG;
    cudaError_t e = cudaMalloc(ptr, sizeof(PxMailbox));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(*ptr, 0, sizeof(PxMailbox));
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

extern "C" int pxl_peer_free(void* ptr) { return ptr ? (int)cudaFree(ptr) : 0; }

extern "C" int pxl_peer_export(void* ptr, unsigned char* handle64) {
    if (!ptr || !handle64) return PXL_ERR_BAD_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
    if (e != cudaSuccess) return (int)e;
    memcpy(handle64, &h, 64);
    return 0;
}

extern "C" int pxl_peer_open(const unsigned char* handle64, void** ptr) {
    if (!handle64 || !ptr) return PXL_ERR_BAD_ARG;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    return (int)cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
}

extern "C" int pxl_peer_close(void* ptr) { return ptr ? (int)cudaIpcCloseMemHandle(ptr) : 0; }

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_volatile_f64(const double* p) {
    double v;
    asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(512)
peer_allreduce_bn_kernel(double* __restrict__ sums, int n, PxPeers peers, int rank, int world, unsigned long long seq,
                         double count, int C, const float* __restrict__ gamma, const float* __restrict__ beta,
                         float* running_mean, float* running_var, float momentum, float eps, int clamp_mode,
                         float* mean, float* invstd, float* scale, float* shift,
                         float* dgamma_acc, float* dbeta_acc, int* err) {
    const int slot = (int)(seq % PX_NSLOT);
    // backward: the parameter gradients come from the LOCAL sums (DDP averages them with the other gradients):
    // dbeta += sum dz, dgamma += sum dz*xhat, straight into the gradient arena, before the lanes are exchanged
    if (dgamma_acc) {
        const int Ch = n >> 1;
        for (int c = threadIdx.x; c < Ch; c += blockDim.x) {
            dbeta_acc[c] += (float)sums[c];
            dgamma_acc[c] += (float)sums[Ch + c];
        }
    }
    __shared__ int failed;
    if (threadIdx.x == 0) failed = 0;
    // 1. push this rank's lane to every mailbox, then publish
    for (int p = 0; p < world; ++p) {
        double* dst = peers.box[p]->slot[slot].data[rank];
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = sums[i];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) st_release_sys(&peers.box[threadIdx.x]->slot[slot].flag[rank], seq);
    // 2. wait for every lane of my own mailbox
    PxSlot* mine = &peers.box[rank]->slot[slot];
    if (threadIdx.x < world) {
        bool ok = false;
        for (unsigned spin = 0; spin < (1u << 27); ++spin) {
            if (ld_acquire_sys(&mine->flag[threadIdx.x]) == seq) { ok = true; break; }
            if ((spin & 0xFFFFu) == 0xFFFFu && *(volatile int*)err != 0) break;
        }
        if (!ok) { atomicCAS(err, 0, 21); failed = 1; }
    }
    __syncthreads();
    if (failed) return;
    // 3. total in rank order (identical on every rank)
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double s = 0.0;
        for (int q = 0; q < world; ++q) s += ld_volatile_f64(&mine->data[q][i]);
        sums[i] = s;
    }
    if (count <= 0.0) return;
    __syncthreads();
    // 4. finalize (same arithmetic as bn_finalize_kernel)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const double m = sums[c] / count;
        double var = sums[C + c] / count - m * m;
        if (var < 0.0) var = 0.0;
        const float mf = (float)m;
        float is;
        if (clamp_mode) is = 1.0f / sqrtf(fmaxf((float)var, eps));
        else is = 1.0f / sqrtf((float)var + eps);
        if (running_mean) {
            const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
            running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mf;
            running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
        }
        mean[c] = mf;
        invstd[c] = is;
        const float sc = gamma[c] * is;
        scale[c] = sc;
        shift[c] = beta[c] - mf * sc;
    }
}

static int* g_peer_err = nullptr;

extern "C" int pxl_peer_allreduce_bn(double* sums, int n, void* const* mailboxes, int rank, int world, int64_t seq,
                                     double count, int C, const float* gamma, const float* beta, float* running_mean,
                                     float* running_var, float momentum, float eps, int clamp_mode, float* mean,
                                     float* invstd, float* scale, float* shift, float* dgamma_acc, float* dbeta_acc,
                                     void* stream) {
    if ((dgamma_acc == nullptr) != (dbeta_acc == nullptr) || (n & 1)) return PXL_ERR_BAD_ARG;
    if (!sums || !mailboxes || n <= 0 || n > PX_MAXN || world < 1 || world > PX_MAXW || rank < 0 || rank >= world || seq <= 0)
        return PXL_ERR_BAD_ARG;
    if (count > 0.0 && (!gamma || !beta || !mean || !invstd || !scale || !shift || C <= 0 || 2 * C != n)) return PXL_ERR_BAD_ARG;
    PxPeers peers;
    for (int p = 0; p < PX_MAXW; ++p) peers.box[p] = p < world ? (PxMailbox*)mailboxes[p] : nullptr;
    for (int p = 0; p < world; ++p) if (!peers.box[p]) return PXL_ERR_BAD_ARG;
    if (!g_peer_err) {
        cudaError_t e = cudaMalloc(&g_peer_err, sizeof(int));
        if (e != cudaSuccess) return (int)e;
        e = cudaMemset(g_peer_err, 0, sizeof(int));
        if (e != cudaSuccess) return (int)e;
    }
    peer_allreduce_bn_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(sums, n, peers, rank, world, (unsigned long long)seq, count, C,
                                                                 gamma, beta, running_mean, running_var, momentum, eps, clamp_mode,
                                                                 mean, invstd, scale, shift, dgamma_acc, dbeta_acc, g_peer_err);
    PXL_CHECK_LAUNCH();
    return 0;
}

// 0 = every exchange so far completed; 21 = a peer never published its lane
extern "C" int pxl_peer_status(void) {
    if (!g_peer_err) return 0;
    int v = 0;
    if (cudaMemcpy(&v, g_peer_err, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return v;
}
