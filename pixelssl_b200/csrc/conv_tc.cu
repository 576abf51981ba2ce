// wgmma (Hopper warpgroup MMA) implicit-GEMM convolution for sm_90a: forward / dgrad (wgrad at the end of the file).
//
//   D[128 output pixels, BN out channels] (fp32, registers) += A[128, K] * B[BN, K]^T  per (tap, 128-byte channel chunk)
//   K per chunk: 64 fp16 values (f16 modes, the benchmarked ones) or 32 tf32 values
//
// * A (activations, NHWC) is staged by TMA as a 4-D box {chunk, BW, BH, 1}: one 128-byte row per
//   output pixel of a BH x BW spatial tile, shifted by the tap offset; out-of-image coordinates
//   are zero-filled by the TMA unit, which IS the convolution's zero padding (im2col-free).
//   1x1 convolutions use the same path with the pixel axis flattened (BW = 128, BH = 1).
// * B (weights [Cout][tap][Cin], K-major) is a 2-D box {chunk, BN}.
// * Both land in shared memory in the canonical K-major SWIZZLE_128B layout and feed wgmma.mma_async directly
//   (four MMAs of 32 bytes of K per operand pair and stage).
// * precision 3 ("f16x3", default of bench.py): both operands arrive as fp16 PAIRS x*s = hi + lo written by the
//   producing kernels (csrc/h16_prep.cu), D += A_hi*B_hi + A_lo*B_hi + A_hi*B_lo recovers fp32-grade products with
//   fp32 accumulation; the epilogue multiplies by the operands' inverse power-of-two scales.  precision 4 ("f16"):
//   hi*hi only.  precision 1 / 2: tf32 single pass / 3xTF32 (raw activations are split hi/lo in shared memory by
//   the consumer warpgroups, "a_inkernel").
// * warp roles: warpgroup 0 = TMA producer (one warp, TMA under elect.sync), warpgroups 1 and 2 = consumers, each
//   owning 64 of the 128 tile rows (wgmma M = 64).  mbarrier full/empty ring.
// * accumulation: the tensor core's own fp32 accumulation truncates (its error grows with the number of MMAs summed
//   into one accumulator), so the MMAs of a stage go into fresh register tiles - the large hi*hi products in two halves
//   of the K slice, the small lo*hi + hi*lo corrections in a tile of their own - which are added to the running sum
//   with IEEE round-to-nearest adds.  The fp16 loops wait for a group only where an add needs it (schedule at the
//   consumer loop): the chains and the adds, and so the results, are bit-identical to waiting for every group.
// * epilogue: registers -> scale / bias -> global (optionally added into the output), and BatchNorm statistics:
//   column sums over each warp's 16 rows by warp shuffles, the eight warps' sums combined in a fixed order, kept per
//   CTA while the CTA stays on one channel block, one fp64 atomic pair per channel and flush.  No fp32 sum depends on
//   the order in which warps or CTAs finish, so a run is reproducible bit for bit.
// * the kernel is persistent (one CTA per SM walks over the tiles) and launched with programmatic stream
//   serialization: everything before PXL_PDL_SYNC() overlaps the previous kernel.
//
// Every mbarrier wait has a watchdog: on expiry the kernel raises a device-side flag and bails
// out, so a protocol bug can never hang the GPU.
#include "common.cuh"
#include <cuda.h>
#include <cstdlib>
#include <type_traits>

// ------------------------------------------------------------------------------------------
// driver entry point for tensor-map encoding (no link-time dependency on libcuda)
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// NHWC tensor viewed as (C, W, H, N), box {one 128-byte row of channels, bw, bh, 1}, 128-byte swizzle, zero OOB fill.
// estride = traversal stride of the W/H dims (2 for stride-2 convolutions: the box spans 2x the pixels
// and the TMA unit picks every 2nd one)
// f16: the tensor holds __half (one half of an fp16 pair, see h16_prep.cu); a 128-byte row is then 64 channels
static int make_act_map(CUtensorMap* m, const void* base, int C, int W, int H, int N, int bw, int bh, int estride = 1, int f16 = 0) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return PXL_ERR_UNSUPPORTED;
    const cuuint64_t eb = f16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * eb, (cuuint64_t)W * C * eb, (cuuint64_t)H * W * C * eb};
    cuuint32_t box[4] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)(bw * estride), (cuuint32_t)(bh * estride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)estride, (cuuint32_t)estride, 1};
    if (box[1] > 256 || box[2] > 256) return PXL_ERR_UNSUPPORTED;
    CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : PXL_ERR_BAD_ARG;
}

// weights [rows][K], box {one 128-byte row of K, bn}
static int make_w_map(CUtensorMap* m, const void* base, int64_t K, int rows, int bn, int f16 = 0) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return PXL_ERR_UNSUPPORTED;
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K * (f16 ? 2 : 4)};
    cuuint32_t box[2] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)bn};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : PXL_ERR_BAD_ARG;
}

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: returns false (and raises *flag) if the barrier never completes
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* flag, int code) {
    for (uint32_t spin = 0; spin < (1u << 22); ++spin) {
        if (mbar_try_wait(bar, parity)) return true;
        if ((spin & 1023u) == 1023u && *(volatile int*)flag != 0) return false;   // another CTA already failed
    }
    atomicCAS(flag, 0, code);
    return false;
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// One lane of a converged warp (deterministic for a given member mask).  The producer warp runs its loop with all
// 32 lanes in uniform control flow and predicates only the TMA instructions with this.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "@px mov.s32 %0, 1;\n\t}"
        : "+r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void named_bar(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma ----
// shared-memory matrix descriptor, SWIZZLE_128B: start address >> 4 | LBO >> 4 << 16 | SBO = 1024 B (8 rows x 128 B)
// >> 4 << 32 | layout SWIZZLE_128B (1) << 62.  K-major operands ignore LBO; MN-major ones (the wgrad kernel) use it
// as the byte distance between 64-element MN slabs.
__device__ __forceinline__ uint64_t sw128_desc(uint32_t smem_addr, uint32_t lbo_bytes = 16) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wg_arrive() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, one MMA: KIND 0 = tf32 (K = 8), 1 = fp16 (K = 16), both K-major;
// 2 = fp16 with both operands MN-major.  scale_d = 0 overwrites D.
template <int N, int KIND>
__device__ __forceinline__ void wgmma_op(float (&d)[N / 2], uint64_t da, uint64_t db, int scale_d);
template <> __device__ __forceinline__ void wgmma_op<32, 0>(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<64, 0>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<128, 0>(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<32, 1>(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<64, 1>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<128, 1>(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<64, 2>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_op<128, 2>(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

// the MMAs of one 128-byte K slice of a stage (4 steps of 32 bytes): hi*hi into `part`, and when the operands are
// split lo*hi + hi*lo into `corr` (both overwritten).  The tensor core truncates while it accumulates; kept apart, the
// small correction terms are not truncated against the large hi*hi sum.
template <int BN, int F16>
__device__ __forceinline__ void mma_slice(float (&part)[BN / 2], float (&corr)[BN / 2], uint64_t da, uint64_t db, uint64_t dal,
                                          uint64_t dbl, bool split3) {
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_op<BN, F16>(part, da + 2 * k, db + 2 * k, k);
    if (split3) {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_op<BN, F16>(corr, dal + 2 * k, db + 2 * k, k);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_op<BN, F16>(corr, da + 2 * k, dbl + 2 * k, 1);
    }
}

__device__ __forceinline__ float4 tf32_split4(float4 v, float4& lo) {
    float4 h;
    const float* vp = &v.x; float* hp = &h.x; float* lp = &lo.x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        uint32_t u;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(vp[e]));
        u &= 0xFFFFE000u;
        hp[e] = __uint_as_float(u);
        lp[e] = vp[e] - hp[e];
    }
    return h;
}

// ------------------------------------------------------------------------------------------
struct TcParams {
    int Cin, Cout, ldo, ntaps, kchunks;
    int N, OH, OW;
    int BW, BH, tilesW, tilesH;
    int stages, nsplit;
    int a_inkernel; // 3xTF32 only: A arrives as raw fp32 and is split hi/lo in shared memory by the consumers
    int in_mul;     // input pixel = output pixel * in_mul + tap (stride-2 forward uses the TMA traversal stride)
    int out_mul, out_offy, out_offx, outH, outW;   // output pixel (oy,ox) is stored at (oy*out_mul+offy, ox*out_mul+offx)
    int ntilesN, pix_tiles, total_tiles;
    int kc;         // K elements per 128-byte operand row: 32 (tf32) or 64 (fp16)
    float out_scale;   // the accumulator is multiplied by this (and by *oscale_ptr) before bias / statistics / store
    int out_acc;       // the epilogue adds into `out` instead of overwriting it
    short dy[PXL_MAX_TAPS], dx[PXL_MAX_TAPS], widx[PXL_MAX_TAPS];
};

#define TC_A_BYTES (128 * 128)          // 128 rows x 128 B
#define TC_MAX_STAGES 8
#define TC_THREADS 384                  // producer warpgroup + two consumer warpgroups

// tile index -> (channel block, pixel tile); channel-block-major so that a persistent CTA mostly stays on one
// channel block (its BatchNorm partial sums then flush rarely)
__device__ __forceinline__ void tc_tile_coords(const TcParams& p, int tile, int bn, int& n0, int& w0, int& h0, int& n) {
    const int nt = tile / p.pix_tiles, pix = tile - nt * p.pix_tiles;
    const int tw = pix % p.tilesW, th = (pix / p.tilesW) % p.tilesH;
    n = pix / (p.tilesW * p.tilesH);
    w0 = tw * p.BW; h0 = th * p.BH; n0 = nt * bn;
}

template <int BN, int F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_wg_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapAlo,
               const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapBlo,
               const TcParams p, const float* __restrict__ bias, float* __restrict__ out,
               double* __restrict__ stats, int* __restrict__ err_flag, const float* __restrict__ oscale_ptr) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ uint64_t full_bar[TC_MAX_STAGES], empty_bar[TC_MAX_STAGES];
    __shared__ float st_warp[2][8][BN];         // per-warp column sums / sums of squares of the current tile

    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    constexpr int B_BYTES = BN * 128;
    constexpr int PER_OP = TC_A_BYTES + B_BYTES;              // A + B of one precision part
    const int stage_bytes = PER_OP * (p.nsplit == 3 ? 2 : 1);
    const int iters = p.ntaps * p.kchunks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    PXL_PDL_SYNC();          // everything above overlapped the previous kernel's tail; global memory from here on

    if (threadIdx.x < 128) {
        // ================= TMA producer (warp 0 converged, TMA under elect.sync) =================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x >= 32) return;
        // bytes the TMA unit will deliver per stage: full boxes, OOB parts are zero-filled but counted
        uint32_t tx = (uint32_t)((p.BW * p.BH * 128 + B_BYTES) * (p.nsplit == 3 ? 2 : 1));
        if (p.a_inkernel) tx -= (uint32_t)(p.BW * p.BH * 128);      // no A_lo box: it is produced in shared memory
        uint32_t s = 0, ph = 0;
        bool ok = true;
        for (int tile = blockIdx.x; tile < p.total_tiles && ok; tile += gridDim.x) {
            int n0, w0, h0, n;
            tc_tile_coords(p, tile, BN, n0, w0, h0, n);
            int tap = 0, c0 = 0;
            for (int it = 0; it < iters; ++it) {
                ok = __all_sync(0xffffffffu, mbar_wait(&empty_bar[s], ph ^ 1u, err_flag, 1));
                if (!ok) break;
                uint8_t* sa = smem + (size_t)s * stage_bytes;
                const int ax = w0 * p.in_mul + p.dx[tap], ay = h0 * p.in_mul + p.dy[tap];
                const int bk = p.widx[tap] * p.Cin + c0;
                if (elect_one()) {
                    mbar_expect_tx(&full_bar[s], tx);
                    tma_load_4d(sa, &mapA, &full_bar[s], c0, ax, ay, n);
                    tma_load_2d(sa + TC_A_BYTES, &mapB, &full_bar[s], bk, n0);
                    if (p.nsplit == 3) {
                        if (!p.a_inkernel) tma_load_4d(sa + PER_OP, &mapAlo, &full_bar[s], c0, ax, ay, n);
                        tma_load_2d(sa + PER_OP + TC_A_BYTES, &mapBlo, &full_bar[s], bk, n0);
                    }
                }
                __syncwarp();
                c0 += p.kc; if (c0 >= p.Cin) { c0 = 0; ++tap; }
                if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ================= consumers: warpgroup cw owns tile rows 64 cw .. 64 cw + 63 =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int ct = threadIdx.x - 128;            // 0..255
    const int cw = ct >> 7, t = ct & 127;
    const int warp = t >> 5, lane = t & 31;
    const float osc = p.out_scale * (oscale_ptr ? __ldg(oscale_ptr) : 1.f);
    const uint32_t smem_base = smem_u32(smem);
    const bool split3 = p.nsplit == 3;
    float acc[BN / 2], part[BN / 2], corr[BN / 2];
    uint32_t s = 0, ph = 0;
    int st_n0 = -1;
    float st_s = 0.f, st_q = 0.f;                // thread ct < BN: column ct of the current channel block
    bool ok = true;
    // BatchNorm partial sums of the current channel block -> one fp64 atomic pair per channel
    auto flush_stats = [&]() {
        if (st_n0 >= 0 && ct < BN && st_n0 + ct < p.Cout && (st_s != 0.f || st_q != 0.f)) {
            atomicAdd(stats + st_n0 + ct, (double)st_s);
            atomicAdd(stats + p.Cout + st_n0 + ct, (double)st_q);
        }
        st_s = 0.f; st_q = 0.f;
    };
    // fp16 operands: the K loop of one tile.  It makes the adds of a loop that waits for every MMA group before it
    // adds, on the same MMA chains and in the same order, so its results are bit-identical to that loop's; only the
    // waits that order nothing are gone:
    //   f16x3:  P1 part = hi*hi (k0,k1) | acc += corr (the previous stage's part + corr)
    //           C corr = lo*hi + hi*lo (k0..k3) | wait 1, acc += part                            (C still runs)
    //           P2 part = hi*hi (k2,k3)         | wait 0, corr = part + corr
    //   f16:    P1 part = hi*hi (k0,k1) | wait 1, acc += corr (P2 of the previous stage)
    //           P2 corr = hi*hi (k2,k3) | wait 1, acc += part
    // The last add of an f16x3 stage, acc += (part + corr), needs its second hi*hi half and its corrections in
    // registers at once, and at BN = 128 there is no room for a fourth register tile (acc, part, corr take 192 of the
    // 232 registers), so its wait empties this warpgroup's queue.  Only the inner sum is taken there; it frees `part`,
    // and the outer add follows once the next stage's P1 is issued (or at the end of the tile), so the tensor pipe
    // runs P1 during it.  The values and the order of the adds into acc are those of the one-line add.  The loop is
    // not limited by operand delivery: loading no B_lo plane, a quarter of a stage's bytes, shortens it by under 1 %
    // (DESIGN.md section 7).  In f16 a stage is read until its last group completes, which the first wait of the next
    // stage (or the tile's final wait) proves: its `empty` arrive comes then.  The ring stays as it was: at BN = 128
    // three 64 KB stages fill the shared memory.
    auto f16_tile = [&](auto split3_c) -> bool {
        constexpr bool S3 = decltype(split3_c)::value;
        uint32_t prev = 0;
        for (int it = 0; it < iters; ++it) {
            if (!__all_sync(0xffffffffu, mbar_wait(&full_bar[s], ph, err_flag, 2))) { wg_wait0(); return false; }
            const uint32_t sa32 = smem_base + s * (uint32_t)stage_bytes;
            const uint32_t arow = (uint32_t)cw * (TC_A_BYTES / 2);
            const uint64_t da = sw128_desc(sa32 + arow), db = sw128_desc(sa32 + TC_A_BYTES);
            const uint64_t dal = sw128_desc(sa32 + PER_OP + arow), dbl = sw128_desc(sa32 + PER_OP + TC_A_BYTES);
            wg_arrive();
            fence_regs(part);
            if (S3) fence_regs(corr);
#pragma unroll
            for (int k = 0; k < 2; ++k) wgmma_op<BN, 1>(part, da + 2 * k, db + 2 * k, k);
            wg_commit();
            if (S3) {
                if (it > 0) {
                    fence_regs(corr);
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] += corr[i];     // the previous stage's last add
                    wg_arrive();
                    fence_regs(corr);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_op<BN, 1>(corr, dal + 2 * k, db + 2 * k, k);
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_op<BN, 1>(corr, da + 2 * k, dbl + 2 * k, 1);
                wg_commit();
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
                fence_regs(part);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
                wg_arrive();
                fence_regs(part);
#pragma unroll
                for (int k = 2; k < 4; ++k) wgmma_op<BN, 1>(part, da + 2 * k, db + 2 * k, k - 2);
                wg_commit();
                wg_wait0();
                fence_regs(part);
                fence_regs(corr);
                mbar_arrive(&empty_bar[s]);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) corr[i] = part[i] + corr[i];   // added into acc after the next P1
            } else {
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
                fence_regs(corr);
                if (it > 0) {
                    mbar_arrive(&empty_bar[prev]);
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] += corr[i];
                }
                wg_arrive();
                fence_regs(corr);
#pragma unroll
                for (int k = 2; k < 4; ++k) wgmma_op<BN, 1>(corr, da + 2 * k, db + 2 * k, k - 2);
                wg_commit();
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
                fence_regs(part);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
            }
            prev = s;
            if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
        }
        if (!S3) {
            wg_wait0();
            fence_regs(corr);
            mbar_arrive(&empty_bar[prev]);
        }
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += corr[i];
        return true;
    };
    for (int tile = blockIdx.x; tile < p.total_tiles && ok; tile += gridDim.x) {
        int n0, w0, h0, n;
        tc_tile_coords(p, tile, BN, n0, w0, h0, n);
        if (stats && n0 != st_n0) { flush_stats(); st_n0 = n0; }
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        if constexpr (F16 != 0) ok = split3 ? f16_tile(std::true_type{}) : f16_tile(std::false_type{});
        else for (int it = 0; it < iters; ++it) {
            ok = __all_sync(0xffffffffu, mbar_wait(&full_bar[s], ph, err_flag, 2));
            if (!ok) break;
            uint8_t* sa = smem + (size_t)s * stage_bytes;
            if (p.a_inkernel) {
                // raw fp32 A rows of this warpgroup -> hi (in place) / lo; elementwise, so the TMA swizzle is preserved
                float4* a_hi = reinterpret_cast<float4*>(sa + cw * (TC_A_BYTES / 2));
                float4* a_lo = reinterpret_cast<float4*>(sa + PER_OP + cw * (TC_A_BYTES / 2));
#pragma unroll
                for (int c = 0; c < TC_A_BYTES / 2 / 16 / 128; ++c) {
                    float4 lo;
                    const float4 hi = tf32_split4(a_hi[t + c * 128], lo);
                    a_hi[t + c * 128] = hi;
                    a_lo[t + c * 128] = lo;
                }
                fence_async_smem();                   // generic-proxy writes -> visible to the tensor core
                named_bar(2 + cw, 128);
            }
            const uint32_t sa32 = smem_base + s * (uint32_t)stage_bytes;
            const uint32_t arow = (uint32_t)cw * (TC_A_BYTES / 2);
            const uint64_t da = sw128_desc(sa32 + arow), db = sw128_desc(sa32 + TC_A_BYTES);
            const uint64_t dal = sw128_desc(sa32 + PER_OP + arow), dbl = sw128_desc(sa32 + PER_OP + TC_A_BYTES);
            // hi*hi in two halves of the K slice, each added to the running sum as soon as it is complete: the
            // tensor core truncates while it accumulates, so it never sums more than two MMAs of the large terms
            wg_arrive();
            fence_regs(part);
            fence_regs(corr);
#pragma unroll
            for (int k = 0; k < 2; ++k) wgmma_op<BN, F16>(part, da + 2 * k, db + 2 * k, k);
            if (split3) {
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_op<BN, F16>(corr, dal + 2 * k, db + 2 * k, k);
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_op<BN, F16>(corr, da + 2 * k, dbl + 2 * k, 1);
            }
            wg_commit();
            wg_wait0();
            fence_regs(part);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
            wg_arrive();
            fence_regs(part);
#pragma unroll
            for (int k = 2; k < 4; ++k) wgmma_op<BN, F16>(part, da + 2 * k, db + 2 * k, k - 2);
            wg_commit();
            wg_wait0();
            fence_regs(part);
            fence_regs(corr);
            mbar_arrive(&empty_bar[s]);              // this thread's share of the stage has been consumed
            if (split3) {
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] += part[i] + corr[i];
            } else {
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
            }
            if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
        }
        if (!ok) break;
        // ---- epilogue.  Fragment of m64nN: rows warp*16 + lane/4 (+8), columns 8j + 2(lane%4) (+1) ----
        int64_t obase[2];
        bool valid[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = cw * 64 + warp * 16 + (lane >> 2) + 8 * h;
            const int hy = r / p.BW, wx = r - hy * p.BW;
            const int oy = h0 + hy, ox = w0 + wx;
            valid[h] = hy < p.BH && oy < p.OH && ox < p.OW;
            obase[h] = ((int64_t)(n * p.outH + oy * p.out_mul + p.out_offy) * p.outW + ox * p.out_mul + p.out_offx) * p.ldo;
        }
        const bool vec2 = (p.ldo & 1) == 0 && ((uintptr_t)out & 7) == 0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int cl = j * 8 + 2 * (lane & 3);
            const int col = n0 + cl;
            const bool c0ok = col < p.Cout, c1ok = col + 1 < p.Cout;
            const float b0 = (bias && c0ok) ? __ldg(bias + col) : 0.f, b1 = (bias && c1ok) ? __ldg(bias + col + 1) : 0.f;
            float v[2][2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                v[h][0] = acc[j * 4 + 2 * h] * osc + b0;
                v[h][1] = acc[j * 4 + 2 * h + 1] * osc + b1;
                if (!valid[h]) continue;
                float* o = out + obase[h] + col;
                if (p.out_acc) {
                    if (c0ok) o[0] += v[h][0];
                    if (c1ok) o[1] += v[h][1];
                } else if (c1ok && vec2) {
                    *reinterpret_cast<float2*>(o) = make_float2(v[h][0], v[h][1]);
                } else {
                    if (c0ok) o[0] = v[h][0];
                    if (c1ok) o[1] = v[h][1];
                }
            }
            if (stats) {
                float s0 = (valid[0] ? v[0][0] : 0.f) + (valid[1] ? v[1][0] : 0.f);
                float s1 = (valid[0] ? v[0][1] : 0.f) + (valid[1] ? v[1][1] : 0.f);
                float q0 = (valid[0] ? v[0][0] * v[0][0] : 0.f) + (valid[1] ? v[1][0] * v[1][0] : 0.f);
                float q1 = (valid[0] ? v[0][1] * v[0][1] : 0.f) + (valid[1] ? v[1][1] * v[1][1] : 0.f);
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                    q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
                }
                if (lane < 4) {
                    const int slot = cw * 4 + warp;
                    st_warp[0][slot][cl] = s0; st_warp[0][slot][cl + 1] = s1;
                    st_warp[1][slot][cl] = q0; st_warp[1][slot][cl + 1] = q1;
                }
            }
        }
        if (stats) {
            named_bar(1, 256);
            if (ct < BN) {
#pragma unroll
                for (int w8 = 0; w8 < 8; ++w8) { st_s += st_warp[0][w8][ct]; st_q += st_warp[1][w8][ct]; }
            }
            named_bar(1, 256);                   // the slots may be rewritten by the next tile
        }
    }
    if (stats && ok) flush_stats();
}

// ------------------------------------------------------------------------------------------
// tf32 split: hi = x with the low 13 mantissa bits cleared after round-to-nearest, lo = x - hi
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo, int64_t n4) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 l;
        hi[i] = tf32_split4(__ldcs(x + i), l);
        lo[i] = l;
    }
}

extern "C" int pxl_split_tf32(const float* x, float* hi, float* lo, int64_t n, void* stream) {
    if (!x || !hi || !lo || n <= 0 || (n & 3)) return PXL_ERR_BAD_ARG;
    const int64_t n4 = n / 4;
    int blocks = (int)(pxl_cdiv(n4, 256 * 2) < PXL_NUM_SMS * 8 ? pxl_cdiv(n4, 256 * 2) : PXL_NUM_SMS * 8);
    split_tf32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (float4*)hi, (float4*)lo, n4);
    PXL_CHECK_LAUNCH();
    return 0;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static int* g_err_flag = nullptr;

static int ensure_err_flag() {
    if (g_err_flag) return 0;
    cudaError_t e = cudaMalloc(&g_err_flag, sizeof(int));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(g_err_flag, 0, sizeof(int));
    return e == cudaSuccess ? 0 : (int)e;
}

// Largest dynamic shared memory a CTA of `kernel` may request: the device's opt-in limit minus the kernel's own static
// shared memory, both queried, so the budget follows the kernel when its __shared__ variables change.  <= 0: unknown.
template <typename K>
static int query_dyn_smem_limit(K kernel) {
    int dev = 0, optin = 0;
    cudaFuncAttributes a;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&a, kernel) != cudaSuccess)
        return 0;
    return optin - (int)a.sharedSizeBytes;
}

static void pick_tile(int OH, int OW, bool flat, int& BW, int& BH) {
    if (flat) { BW = 128; BH = 1; return; }
    // choose BW x BH <= 128 maximising useful pixels per 128-row MMA tile
    double best = -1.0;
    BW = 16; BH = 8;
    for (int bw = 4; bw <= 128 && bw <= 256; ++bw) {
        int bh = 128 / bw;
        if (bh < 1) break;
        if (bh > 256) bh = 256;
        const int64_t tiles = (int64_t)((OW + bw - 1) / bw) * ((OH + bh - 1) / bh);
        const double eff = (double)OH * OW / ((double)tiles * 128.0);
        if (eff > best + 1e-9) { best = eff; BW = bw; BH = bh; }
    }
}

template <int BN, int F16>
static int fwd_smem_limit() {
    static const int v = query_dyn_smem_limit(conv_wg_kernel<BN, F16>);
    return v;
}

template <int BN, int F16>
static int launch_fwd(const CUtensorMap& mA, const CUtensorMap& mAlo, const CUtensorMap& mB, const CUtensorMap& mBlo,
                      const TcParams& p, size_t smem, cudaStream_t st, const float* bias, float* out, double* stats,
                      const float* oscale_ptr) {
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(conv_wg_kernel<BN, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, fwd_smem_limit<BN, F16>());
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    const unsigned nblk = (unsigned)(p.total_tiles < PXL_NUM_SMS ? p.total_tiles : PXL_NUM_SMS);
    cudaError_t le = pxl_launch_pdl(conv_wg_kernel<BN, F16>, dim3(nblk), dim3(TC_THREADS), smem, st, mA, mAlo, mB, mBlo, p,
                                    bias, out, stats, g_err_flag, oscale_ptr);
    if (le != cudaSuccess) return (int)le;
    PXL_CHECK_LAUNCH();
    return 0;
}

static int conv_tc_launch_core(const pxl_conv_geom* g, const int* taps, const pxl_conv_tc_ext* ext,
                               const void* in_hi, const void* in_lo, const void* w_hi, const void* w_lo,
                               const float* bias, float* out, void* stream);

// lo parts: for precision 2 the caller passes hi/lo through `in`/`w` (hi) and the extra pointers
extern "C" int pxl_conv_tc_launch_ex(const pxl_conv_geom* g, const int* taps, const pxl_conv_tc_ext* ext,
                                     const float* in_hi, const float* in_lo, const float* w_hi, const float* w_lo,
                                     const float* bias, float* out, void* stream) {
    if (g && g->precision > 2) return PXL_ERR_BAD_ARG;      // fp16 operands go through pxl_conv_h16_launch
    return conv_tc_launch_core(g, taps, ext, in_hi, in_lo, w_hi, w_lo, bias, out, stream);
}

// fp16-pair operands (h16_prep.cu): precision 3 = hi*hi + lo*hi + hi*lo (fp32-grade), 4 = hi*hi only (11-bit
// significands = TF32-grade)
extern "C" int pxl_conv_h16_launch(const pxl_conv_geom* g, const int* taps, const pxl_conv_tc_ext* ext,
                                   const void* in_hi, const void* in_lo, const void* w_hi, const void* w_lo,
                                   const float* bias, float* out, void* stream) {
    if (!g || (g->precision != 3 && g->precision != 4)) return PXL_ERR_BAD_ARG;
    return conv_tc_launch_core(g, taps, ext, in_hi, in_lo, w_hi, w_lo, bias, out, stream);
}

static int conv_tc_launch_core(const pxl_conv_geom* g, const int* taps, const pxl_conv_tc_ext* ext,
                               const void* in_hi, const void* in_lo, const void* w_hi, const void* w_lo,
                               const float* bias, float* out, void* stream) {
    if (!g || !taps || !in_hi || !w_hi || !out) return PXL_ERR_BAD_ARG;
    if ((g->mul != 1 && g->mul != 2) || g->div != 1) return PXL_ERR_UNSUPPORTED;
    const int f16 = g->precision >= 3 ? 1 : 0;
    const int kc = f16 ? 64 : 32;
    if (g->Cin % kc != 0 || g->ntaps > PXL_MAX_TAPS) return PXL_ERR_UNSUPPORTED;
    const int wtaps = ext && ext->w_ntaps > 0 ? ext->w_ntaps : g->ntaps;    // taps in the weight tensor
    const int nsplit = (g->precision == 2 || g->precision == 3) ? 3 : 1;
    if (nsplit == 3 && !w_lo) return PXL_ERR_BAD_ARG;
    if (f16 && nsplit == 3 && !in_lo) return PXL_ERR_BAD_ARG;    // fp16 pairs are always split by their producer
    const int a_inkernel = (!f16 && nsplit == 3 && !in_lo) ? 1 : 0;       // in_hi then holds the raw fp32 activations
    const int omul = (ext && ext->out_mul > 0) ? ext->out_mul : 1;
    const bool has_out_xform = ext && (omul != 1 || ext->out_offy != 0 || ext->out_offx != 0);
    bool flat = (g->ntaps == 1 && taps[0] == 0 && taps[1] == 0 && g->OH == g->H && g->OW == g->W && g->mul == 1 &&
                 !has_out_xform);
    TcParams p;
    p.Cin = g->Cin; p.Cout = g->Cout; p.ldo = g->ldo; p.ntaps = g->ntaps; p.kchunks = g->Cin / kc;
    p.nsplit = nsplit; p.a_inkernel = a_inkernel; p.kc = kc;
    p.out_scale = (ext && ext->out_scale != 0.f) ? ext->out_scale : 1.f;
    const float* oscale_ptr = ext ? ext->out_scale_dev : nullptr;
    for (int t = 0; t < g->ntaps; ++t) {
        p.dy[t] = (short)taps[2 * t]; p.dx[t] = (short)taps[2 * t + 1];
        p.widx[t] = (short)((ext && ext->widx_host) ? ext->widx_host[t] : t);
        if (p.widx[t] < 0 || p.widx[t] >= wtaps) return PXL_ERR_BAD_ARG;
    }
    p.in_mul = g->mul;
    p.out_mul = omul; p.out_offy = has_out_xform ? ext->out_offy : 0; p.out_offx = has_out_xform ? ext->out_offx : 0;
    int mapW, mapH, mapN;
    if (flat) {
        const int64_t M = (int64_t)g->N * g->H * g->W;
        if (M >= (1ll << 31)) return PXL_ERR_UNSUPPORTED;
        p.N = 1; p.OH = 1; p.OW = (int)M;
        mapW = (int)M; mapH = 1; mapN = 1;
        p.outH = 1; p.outW = (int)M;
    } else {
        p.N = g->N; p.OH = g->OH; p.OW = g->OW;
        mapW = g->W; mapH = g->H; mapN = g->N;
        p.outH = has_out_xform ? ext->out_H : g->OH; p.outW = has_out_xform ? ext->out_W : g->OW;
    }
    pick_tile(p.OH, p.OW, flat, p.BW, p.BH);
    if (g->mul == 2 && (p.BW > 128 || p.BH > 128)) return PXL_ERR_UNSUPPORTED;
    // N tile: the accumulator and the per-stage partial of a consumer thread take BN / 2 registers each
    const int BN = g->Cout > 64 ? 128 : (g->Cout > 32 ? 64 : 32);
    const int stage_bytes = (TC_A_BYTES + BN * 128) * (nsplit == 3 ? 2 : 1);
    p.tilesW = (p.OW + p.BW - 1) / p.BW; p.tilesH = (p.OH + p.BH - 1) / p.BH;
    p.pix_tiles = p.N * p.tilesH * p.tilesW;
    p.ntilesN = (g->Cout + BN - 1) / BN;
    const int64_t n_tiles = (int64_t)p.pix_tiles * p.ntilesN;
    if (n_tiles >= (1ll << 31)) return PXL_ERR_UNSUPPORTED;
    p.total_tiles = (int)n_tiles;
    const int smem_limit = f16 ? (BN == 128 ? fwd_smem_limit<128, 1>() : BN == 64 ? fwd_smem_limit<64, 1>() : fwd_smem_limit<32, 1>())
                               : (BN == 128 ? fwd_smem_limit<128, 0>() : BN == 64 ? fwd_smem_limit<64, 0>() : fwd_smem_limit<32, 0>());
    if (smem_limit <= 0) return PXL_ERR_UNSUPPORTED;
    p.stages = (smem_limit - 1024) / stage_bytes;
    if (p.stages > TC_MAX_STAGES) p.stages = TC_MAX_STAGES;
    if (p.stages < 2) return PXL_ERR_UNSUPPORTED;
    const size_t smem = (size_t)p.stages * stage_bytes + 1024;     // + alignment slack

    CUtensorMap mA, mAlo, mB, mBlo;
    int rc = make_act_map(&mA, in_hi, g->Cin, mapW, mapH, mapN, p.BW, p.BH, g->mul, f16);
    if (rc) return rc;
    rc = make_w_map(&mB, w_hi, (int64_t)wtaps * g->Cin, g->Cout, BN, f16);
    if (rc) return rc;
    if (nsplit == 3) {
        if (a_inkernel) mAlo = mA;
        else {
            rc = make_act_map(&mAlo, in_lo, g->Cin, mapW, mapH, mapN, p.BW, p.BH, g->mul, f16);
            if (rc) return rc;
        }
        rc = make_w_map(&mBlo, w_lo, (int64_t)wtaps * g->Cin, g->Cout, BN, f16);
        if (rc) return rc;
    } else {
        mAlo = mA; mBlo = mB;
    }
    p.out_acc = (ext && ext->out_accumulate) ? 1 : 0;
    if ((rc = ensure_err_flag())) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    double* st_ptr = ext ? (double*)ext->bn_stats : nullptr;
    if (f16) {
        if (BN == 128) return launch_fwd<128, 1>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
        if (BN == 64) return launch_fwd<64, 1>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
        return launch_fwd<32, 1>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
    }
    if (BN == 128) return launch_fwd<128, 0>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
    if (BN == 64) return launch_fwd<64, 0>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
    return launch_fwd<32, 0>(mA, mAlo, mB, mBlo, p, smem, st, bias, out, st_ptr, oscale_ptr);
}

// watchdog status: 0 = fine, otherwise the role (1 producer, 2 consumer; 11/12 the same in wgrad) that timed out
extern "C" int pxl_conv_tc_status(void) {
    if (!g_err_flag) return 0;
    int v = 0;
    if (cudaMemcpy(&v, g_err_flag, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return v;
}

// ==========================================================================================
// wgrad on wgmma:  dW[co][tap][ci] += sum_pixels dY[pix][co] * X[pix + tap][ci]
//
//   D[128 co, BN ci] (registers of the two consumer warpgroups, 64 co each) += A^T[K = pixels, co] * B[K = pixels, ci]
//
// A TMA box {one 128-byte row of channels, BW, BH, 1} of an NHWC tensor is (BW*BH pixel rows) x 128 B: both
// operands arrive "MN-major" (the reduction index = pixel row is the slow one) in the SWIZZLE_128B layout.
// * fp16 operands: wgmma reads MN-major fp16 directly (transpose bits set): 64-channel slabs, 16 pixel rows per MMA.
//   The MMAs per stage (rows_alloc / 16: 1-4 in f16x3, 1-8 in f16) are a template constant of fully unrolled loop
//   variants (a runtime trip count makes ptxas serialise the MMAs with extra warpgroup.arrive instructions).
// * tf32 operands: wgmma takes tf32 K-major only, so the consumers transpose each stage (32 pixel rows) into a
//   K-major tile in shared memory - splitting raw fp32 hi/lo for 3xTF32 in the same pass - and the MMAs read that.
// Rows between BW*BH and the allocated rows are zeroed once and never written.  The pixel range is split over
// gridDim.z CTAs: with one split the epilogue adds its tile into dW, otherwise each split stores its tile in a
// workspace and wgrad_reduce_kernel adds the splits into dW in split order (reproducible, unlike atomics).
// ==========================================================================================
struct WgParams {
    int Cin, Cout, ldo, ntaps;
    int N, OH, OW, mul;
    int BW, BH, tilesW, tilesH, rows, rows_alloc;
    int stages, nsplit;
    int inkernel;      // 3xTF32: dY / X arrive raw and are split hi/lo by the transposing consumers
    int slab_ch;       // channels per 128-byte slab row: 32 (tf32) or 64 (fp16)
    float out_scale;   // the tile is multiplied by this (and by *oscale_ptr) before it is added into dW
    int tiles_ci, ktiles_per_cta, ktiles_total;
    short dy[PXL_MAX_TAPS], dx[PXL_MAX_TAPS];
};

template <int BN, int F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_wgrad_wg_kernel(const __grid_constant__ CUtensorMap mapDy, const __grid_constant__ CUtensorMap mapDyLo,
                     const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapXLo,
                     const WgParams p, float* __restrict__ dw, float* __restrict__ ws, int* __restrict__ err_flag,
                     const float* __restrict__ oscale_ptr) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ uint64_t full_bar[TC_MAX_STAGES], empty_bar[TC_MAX_STAGES];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);

    const int slab_bytes = p.rows_alloc * 128;
    const int slabsA = 128 / p.slab_ch;                  // dY slabs (128 output channels)
    const int slabsB = BN / p.slab_ch;
    const int per_op = (slabsA + slabsB) * slab_bytes;
    const int stage_bytes = per_op * (p.nsplit == 3 ? 2 : 1);
    // tf32: K-major copy of one stage (A^T rows 0..127, B^T rows 128..128+BN-1; lo part after it)
    constexpr int KT_BYTES = (128 + BN) * 128;
    uint8_t* kt = smem + (size_t)p.stages * stage_bytes;
    const int tile_co = blockIdx.x / p.tiles_ci, tile_ci = blockIdx.x % p.tiles_ci;
    const int co0 = tile_co * 128, ci0 = tile_ci * BN;
    const int tap = blockIdx.y;
    const int kt0 = blockIdx.z * p.ktiles_per_cta;
    int kt1 = kt0 + p.ktiles_per_cta;
    if (kt1 > p.ktiles_total) kt1 = p.ktiles_total;
    const int iters = kt1 - kt0;
    // slabs that actually exist (the others stay zero)
    int nsA = (p.ldo - co0 + p.slab_ch - 1) / p.slab_ch; if (nsA > slabsA) nsA = slabsA;
    int nsB = (p.Cin - ci0 + p.slab_ch - 1) / p.slab_ch; if (nsB > slabsB) nsB = slabsB;

    // zero the operand ring once: rows the TMA never writes must contribute nothing
    {
        uint4 z = make_uint4(0, 0, 0, 0);
        const int total16 = p.stages * stage_bytes / 16;
        for (int i = threadIdx.x; i < total16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = z;
        fence_async_smem();
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    PXL_PDL_SYNC();          // everything above overlapped the previous kernel's tail; global memory from here on
    if (iters <= 0) return;

    if (threadIdx.x < 128) {
        // TMA producer: warp 0 converged, TMA under elect.sync
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x >= 32) return;
        const uint32_t box_bytes = (uint32_t)(p.rows * 128);
        const int nparts = (p.nsplit == 3 && !p.inkernel) ? 2 : 1;
        const uint32_t tx = box_bytes * (uint32_t)(nsA + nsB) * (uint32_t)nparts;
        const int tdy = p.dy[tap], tdx = p.dx[tap];
        int tw = kt0 % p.tilesW, th = (kt0 / p.tilesW) % p.tilesH, n = kt0 / (p.tilesW * p.tilesH);
        uint32_t s = 0, ph = 0;
        for (int it = 0; it < iters; ++it) {
            if (!__all_sync(0xffffffffu, mbar_wait(&empty_bar[s], ph ^ 1u, err_flag, 11))) break;
            const int w0 = tw * p.BW, h0 = th * p.BH;
            uint8_t* sa = smem + (size_t)s * stage_bytes;
            if (elect_one()) {
                mbar_expect_tx(&full_bar[s], tx);
                for (int part = 0; part < nparts; ++part) {
                    uint8_t* base = sa + (size_t)part * per_op;
                    const CUtensorMap* mdy = part ? &mapDyLo : &mapDy;
                    const CUtensorMap* mx = part ? &mapXLo : &mapX;
                    for (int j = 0; j < nsA; ++j)
                        tma_load_4d(base + (size_t)j * slab_bytes, mdy, &full_bar[s], co0 + p.slab_ch * j, w0, h0, n);
                    for (int j = 0; j < nsB; ++j)
                        tma_load_4d(base + (size_t)(slabsA + j) * slab_bytes, mx, &full_bar[s], ci0 + p.slab_ch * j,
                                    w0 * p.mul + tdx, h0 * p.mul + tdy, n);
                }
            }
            __syncwarp();
            if (++tw == p.tilesW) { tw = 0; if (++th == p.tilesH) { th = 0; ++n; } }
            if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int ct = threadIdx.x - 128;
    const int cw = ct >> 7, t = ct & 127;
    const int warp = t >> 5, lane = t & 31;
    const bool split3 = p.nsplit == 3;
    const uint32_t smem_base = smem_u32(smem);
    float acc[BN / 2], part[BN / 2], corr[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    uint32_t s = 0, ph = 0;
    bool ok = true;
    if constexpr (F16 != 0) {
        // fp16 operands: the K loop with KM = rows_alloc / 16 MMAs per operand pair and stage, fully unrolled.  A
        // stage's hi*hi MMAs go into `part`, its f16x3 corrections into `corr`, and both are added once they are done.
        auto f16_loop = [&](auto km_c, auto split3_c) -> bool {
            constexpr int KM = decltype(km_c)::value;
            constexpr bool S3 = decltype(split3_c)::value;
            constexpr uint64_t kstep = (16 * 128) >> 4;            // 16 pixel rows per MMA
            constexpr uint32_t SLAB = KM * 16 * 128;                // slab_bytes: rows_alloc = 16 KM
            constexpr uint32_t PER_OP = (128 + BN) / 64 * SLAB;     // per_op: 64-channel slabs of dY and X
            for (int it = 0; it < iters; ++it) {
                if (!__all_sync(0xffffffffu, mbar_wait(&full_bar[s], ph, err_flag, 12))) return false;
                const uint32_t sa32 = smem_base + s * (uint32_t)stage_bytes;
                const uint32_t sb32 = sa32 + 2 * SLAB;
                const uint64_t da = sw128_desc(sa32 + cw * SLAB, SLAB);
                const uint64_t db = sw128_desc(sb32, SLAB);
                wg_arrive();
                fence_regs(part);
                fence_regs(corr);
#pragma unroll
                for (int k = 0; k < KM; ++k) wgmma_op<BN, 2>(part, da + kstep * k, db + kstep * k, k);
                if (S3) {
                    const uint64_t dal = sw128_desc(sa32 + PER_OP + cw * SLAB, SLAB);
                    const uint64_t dbl = sw128_desc(sb32 + PER_OP, SLAB);
#pragma unroll
                    for (int k = 0; k < KM; ++k) wgmma_op<BN, 2>(corr, dal + kstep * k, db + kstep * k, k);
#pragma unroll
                    for (int k = 0; k < KM; ++k) wgmma_op<BN, 2>(corr, da + kstep * k, dbl + kstep * k, 1);
                }
                wg_commit();
                wg_wait0();
                fence_regs(part);
                fence_regs(corr);
                mbar_arrive(&empty_bar[s]);
                if (S3) {
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] += part[i] + corr[i];
                } else {
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
                }
                if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
            }
            return true;
        };
        // rows_alloc <= 64 for f16x3 and <= 128 for f16 (conv_wgrad_tc_core's maxrows)
        using std::integral_constant;
        using T = std::true_type;
        using F = std::false_type;
        if (split3) {
            switch (p.rows_alloc / 16) {
                case 1: ok = f16_loop(integral_constant<int, 1>{}, T{}); break;
                case 2: ok = f16_loop(integral_constant<int, 2>{}, T{}); break;
                case 3: ok = f16_loop(integral_constant<int, 3>{}, T{}); break;
                default: ok = f16_loop(integral_constant<int, 4>{}, T{}); break;
            }
        } else {
            switch (p.rows_alloc / 16) {
                case 1: ok = f16_loop(integral_constant<int, 1>{}, F{}); break;
                case 2: ok = f16_loop(integral_constant<int, 2>{}, F{}); break;
                case 3: ok = f16_loop(integral_constant<int, 3>{}, F{}); break;
                case 4: ok = f16_loop(integral_constant<int, 4>{}, F{}); break;
                case 5: ok = f16_loop(integral_constant<int, 5>{}, F{}); break;
                case 6: ok = f16_loop(integral_constant<int, 6>{}, F{}); break;
                case 7: ok = f16_loop(integral_constant<int, 7>{}, F{}); break;
                default: ok = f16_loop(integral_constant<int, 8>{}, F{}); break;
            }
        }
    } else for (int it = 0; it < iters; ++it) {
        ok = __all_sync(0xffffffffu, mbar_wait(&full_bar[s], ph, err_flag, 12));
        if (!ok) break;
        uint8_t* sa = smem + (size_t)s * stage_bytes;
        // transpose the stage (32 pixel rows) into K-major tiles: unit u = (channel row R, pixels 4g .. 4g+3)
        named_bar(1, 256);                                // both warpgroups are done reading the previous tiles
        const int units = (128 + BN) * 8;
        for (int u = ct; u < units; u += 256) {
            const int R = u >> 3, g = u & 7;
            const int slab = R < 128 ? (R >> 5) : slabsA + ((R - 128) >> 5);
            const int c = R & 31;
            const uint8_t* src = sa + (size_t)slab * slab_bytes + (c & 3) * 4;
            float4 v, vl = make_float4(0.f, 0.f, 0.f, 0.f);
            float* vp = &v.x; float* lp = &vl.x;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int px = 4 * g + e;
                const int off = px * 128 + ((((c >> 2) ^ (px & 7))) << 4);
                vp[e] = *reinterpret_cast<const float*>(src + off);
                if (split3 && !p.inkernel) lp[e] = *reinterpret_cast<const float*>(src + per_op + off);
            }
            if (p.inkernel) v = tf32_split4(v, vl);
            const int doff = R * 128 + ((g ^ (R & 7)) << 4);
            *reinterpret_cast<float4*>(kt + doff) = v;
            if (split3) *reinterpret_cast<float4*>(kt + KT_BYTES + doff) = vl;
        }
        fence_async_smem();
        named_bar(1, 256);
        mbar_arrive(&empty_bar[s]);                      // the ring slot has been copied out
        const uint32_t k32 = smem_u32(kt);
        const uint32_t arow = (uint32_t)cw * 64 * 128;
        const uint64_t da = sw128_desc(k32 + arow), db = sw128_desc(k32 + 128 * 128);
        const uint64_t dal = sw128_desc(k32 + KT_BYTES + arow), dbl = sw128_desc(k32 + KT_BYTES + 128 * 128);
        wg_arrive();
        fence_regs(part);
        fence_regs(corr);
        mma_slice<BN, 0>(part, corr, da, db, dal, dbl, split3);
        wg_commit();
        wg_wait0();
        fence_regs(part);
        fence_regs(corr);
        if (split3) {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] += part[i] + corr[i];
        } else {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        }
        if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
    }
    if (!ok) return;
    const float osc = p.out_scale * (oscale_ptr ? __ldg(oscale_ptr) : 1.f);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int co = co0 + cw * 64 + warp * 16 + (lane >> 2) + 8 * h;
        if (co >= p.Cout) continue;
        const int64_t row = ((int64_t)co * p.ntaps + tap) * p.Cin;
        float* drow = gridDim.z == 1 ? dw + row : ws + (int64_t)blockIdx.z * p.Cout * p.ntaps * p.Cin + row;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int ci = ci0 + j * 8 + 2 * (lane & 3);
            const float v0 = acc[j * 4 + 2 * h] * osc, v1 = acc[j * 4 + 2 * h + 1] * osc;
            if (gridDim.z == 1) {                 // this CTA alone owns these dW entries
                if (ci < p.Cin) drow[ci] += v0;
                if (ci + 1 < p.Cin) drow[ci + 1] += v1;
            } else {
                if (ci < p.Cin) drow[ci] = v0;
                if (ci + 1 < p.Cin) drow[ci + 1] = v1;
            }
        }
    }
}

// dW[i] += sum over the splits s = 0, 1, ... of ws[s][i]
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, int64_t n, int splits) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float s = __ldg(ws + i);
        for (int z = 1; z < splits; ++z) s += __ldg(ws + (int64_t)z * n + i);
        dw[i] += s;
    }
}

// activation map for wgrad: optional traversal stride (stride-2 convolutions read every 2nd pixel)
static int make_act_map_strided(CUtensorMap* m, const void* base, int C, int W, int H, int N, int bw, int bh, int estride, int f16 = 0) {
    return make_act_map(m, base, C, W, H, N, bw, bh, estride, f16);
}

static void pick_ktile(int OH, int OW, bool flat, int maxrows, int& BW, int& BH, int unit = 8) {
    if (flat) { BW = maxrows; BH = 1; return; }
    double best = -1.0;
    BW = 8; BH = maxrows / 8;
    for (int bw = 1; bw <= maxrows && bw <= 256; ++bw) {
        int bh = maxrows / bw;
        if (bh < 1) break;
        if (bh > 256) bh = 256;
        const int alloc = (bw * bh + unit - 1) / unit * unit;
        const int64_t tiles = (int64_t)((OW + bw - 1) / bw) * ((OH + bh - 1) / bh);
        const double eff = (double)OH * OW / ((double)tiles * alloc);
        if (eff > best + 1e-9) { best = eff; BW = bw; BH = bh; }
    }
}

static int conv_wgrad_tc_core(const pxl_conv_geom* g, const int* taps, const void* in_hi, const void* in_lo,
                              const void* dy_hi, const void* dy_lo, float* dw, float out_scale, const float* oscale_ptr,
                              void* stream);

extern "C" int pxl_conv_wgrad_tc_launch(const pxl_conv_geom* g, const int* taps, const float* in_hi, const float* in_lo,
                                        const float* dy_hi, const float* dy_lo, float* dw, void* stream) {
    if (g && g->precision > 2) return PXL_ERR_BAD_ARG;      // fp16 operands go through pxl_conv_wgrad_h16_launch
    return conv_wgrad_tc_core(g, taps, in_hi, in_lo, dy_hi, dy_lo, dw, 1.f, nullptr, stream);
}

// fp16-pair operands; dw += out_scale * (*out_scale_dev) * sum(dy * x)
extern "C" int pxl_conv_wgrad_h16_launch(const pxl_conv_geom* g, const int* taps, const void* in_hi, const void* in_lo,
                                         const void* dy_hi, const void* dy_lo, float* dw, float out_scale,
                                         const float* out_scale_dev, void* stream) {
    if (!g || (g->precision != 3 && g->precision != 4)) return PXL_ERR_BAD_ARG;
    return conv_wgrad_tc_core(g, taps, in_hi, in_lo, dy_hi, dy_lo, dw, out_scale != 0.f ? out_scale : 1.f, out_scale_dev, stream);
}

template <int BN, int F16>
static int wgrad_smem_limit() {
    static const int v = query_dyn_smem_limit(conv_wgrad_wg_kernel<BN, F16>);
    return v;
}

template <int BN, int F16>
static int launch_wgrad(const CUtensorMap& mDy, const CUtensorMap& mDyLo, const CUtensorMap& mX, const CUtensorMap& mXLo,
                        const WgParams& p, dim3 grid, size_t smem, cudaStream_t st, float* dw, const float* oscale_ptr) {
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(conv_wgrad_wg_kernel<BN, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, wgrad_smem_limit<BN, F16>());
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    const int64_t n = (int64_t)p.Cout * p.ntaps * p.Cin;
    float* ws = nullptr;
    if (grid.z > 1) {
        int rc = 0;
        ws = (float*)pxl_workspace_(PXL_WS_WGRAD, st, (size_t)n * grid.z * sizeof(float), &rc);
        if (rc) return rc;
    }
    cudaError_t le = pxl_launch_pdl(conv_wgrad_wg_kernel<BN, F16>, grid, dim3(TC_THREADS), smem, st, mDy, mDyLo, mX, mXLo, p, dw,
                                    ws, g_err_flag, oscale_ptr);
    if (le != cudaSuccess) return (int)le;
    PXL_CHECK_LAUNCH();
    if (grid.z > 1) {
        const int blocks = (int)(pxl_cdiv(n, 256) < PXL_NUM_SMS * 8 ? pxl_cdiv(n, 256) : PXL_NUM_SMS * 8);
        wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(ws, dw, n, (int)grid.z);
        PXL_CHECK_LAUNCH();
    }
    return 0;
}

static int conv_wgrad_tc_core(const pxl_conv_geom* g, const int* taps, const void* in_hi, const void* in_lo,
                              const void* dy_hi, const void* dy_lo, float* dw, float out_scale, const float* oscale_ptr,
                              void* stream) {
    if (!g || !taps || !in_hi || !dy_hi || !dw) return PXL_ERR_BAD_ARG;
    if (g->div != 1 || (g->mul != 1 && g->mul != 2)) return PXL_ERR_UNSUPPORTED;   // stride 2 via TMA traversal stride
    const int f16 = g->precision >= 3 ? 1 : 0;
    const int slab_ch = f16 ? 64 : 32;
    if (g->Cin % slab_ch != 0 || g->ldo % slab_ch != 0 || g->ntaps > PXL_MAX_TAPS) return PXL_ERR_UNSUPPORTED;
    const int nsplit = (g->precision == 2 || g->precision == 3) ? 3 : 1;
    if (nsplit == 3 && ((in_lo == nullptr) != (dy_lo == nullptr))) return PXL_ERR_BAD_ARG;
    if (f16 && nsplit == 3 && !in_lo) return PXL_ERR_BAD_ARG;
    const int inkernel = (!f16 && nsplit == 3 && !in_lo) ? 1 : 0;         // in_hi / dy_hi then hold the raw fp32 tensors
    const bool flat = (g->ntaps == 1 && taps[0] == 0 && taps[1] == 0 && g->OH == g->H && g->OW == g->W && g->mul == 1);
    WgParams p;
    p.Cin = g->Cin; p.Cout = g->Cout; p.ldo = g->ldo; p.ntaps = g->ntaps; p.mul = g->mul; p.nsplit = nsplit; p.inkernel = inkernel;
    p.slab_ch = slab_ch; p.out_scale = out_scale;
    for (int t = 0; t < g->ntaps; ++t) { p.dy[t] = (short)taps[2 * t]; p.dx[t] = (short)taps[2 * t + 1]; }
    int mapW, mapH, mapN, inW, inH;
    if (flat) {
        const int64_t M = (int64_t)g->N * g->H * g->W;
        if (M >= (1ll << 31)) return PXL_ERR_UNSUPPORTED;
        p.N = 1; p.OH = 1; p.OW = (int)M; mapW = (int)M; mapH = 1; mapN = 1; inW = (int)M; inH = 1;
    } else {
        p.N = g->N; p.OH = g->OH; p.OW = g->OW; mapW = g->OW; mapH = g->OH; mapN = g->N; inW = g->W; inH = g->H;
    }
    // pixel rows per stage: tf32 stages are transposed into one 128-byte K row (32 pixels); fp16 stages feed the MMAs
    // directly in steps of 16 rows
    const int maxrows = f16 ? (nsplit == 3 ? 64 : 128) : 32;
    const int kunit = f16 ? 16 : 8;
    pick_ktile(p.OH, p.OW, flat, maxrows, p.BW, p.BH, kunit);
    p.rows = p.BW * p.BH;
    p.rows_alloc = f16 ? (p.rows + kunit - 1) / kunit * kunit : 32;
    p.tilesW = (p.OW + p.BW - 1) / p.BW; p.tilesH = (p.OH + p.BH - 1) / p.BH;
    const int BN = f16 ? (g->Cin > 64 ? 128 : 64) : (g->Cin > 64 ? 128 : (g->Cin > 32 ? 64 : 32));
    p.tiles_ci = (g->Cin + BN - 1) / BN;
    const int tiles_co = (g->Cout + 127) / 128;
    const int stage_bytes = (128 / slab_ch + BN / slab_ch) * p.rows_alloc * 128 * (nsplit == 3 ? 2 : 1);
    const int kt_bytes = f16 ? 0 : (128 + BN) * 128 * (nsplit == 3 ? 2 : 1);
    const int smem_limit = f16 ? (BN == 128 ? wgrad_smem_limit<128, 1>() : wgrad_smem_limit<64, 1>())
                               : (BN == 128 ? wgrad_smem_limit<128, 0>() : BN == 64 ? wgrad_smem_limit<64, 0>() : wgrad_smem_limit<32, 0>());
    if (smem_limit <= 0) return PXL_ERR_UNSUPPORTED;
    p.stages = (smem_limit - 1024 - kt_bytes) / stage_bytes;
    if (p.stages > 4) p.stages = 4;
    if (p.stages < 2) return PXL_ERR_UNSUPPORTED;
    p.ktiles_total = p.N * p.tilesH * p.tilesW;
    // split the pixel range: enough CTAs to fill the GPU; pick the split that minimises
    //   rounds x (main-loop iterations per CTA + a fixed prologue/epilogue cost)
    // so that the grid fills whole waves instead of leaving a mostly idle last one
    const int64_t base_ctas = (int64_t)tiles_co * p.tiles_ci * g->ntaps;
    int64_t split = 1, best_cost = -1;
    int64_t hi = pxl_cdiv((int64_t)PXL_NUM_SMS * 4, base_ctas) + 1;
    if (hi > p.ktiles_total) hi = p.ktiles_total;
    for (int64_t sp = 1; sp <= hi; ++sp) {
        const int64_t per = pxl_cdiv(p.ktiles_total, sp);
        const int64_t ctas = base_ctas * pxl_cdiv(p.ktiles_total, per);
        const int64_t cost = pxl_cdiv(ctas, PXL_NUM_SMS) * (per + 6);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; split = sp; }
    }
    if (split > p.ktiles_total) split = p.ktiles_total;
    if (split < 1) split = 1;
    if (split > 65535) split = 65535;
    p.ktiles_per_cta = (int)pxl_cdiv(p.ktiles_total, split);
    split = pxl_cdiv(p.ktiles_total, p.ktiles_per_cta);

    CUtensorMap mDy, mDyLo, mX, mXLo;
    int rc = make_act_map_strided(&mDy, dy_hi, g->ldo, mapW, mapH, mapN, p.BW, p.BH, 1, f16);
    if (rc) return rc;
    rc = make_act_map_strided(&mX, in_hi, g->Cin, inW, inH, mapN, p.BW, p.BH, g->mul, f16);
    if (rc) return rc;
    if (nsplit == 3 && !inkernel) {
        rc = make_act_map_strided(&mDyLo, dy_lo, g->ldo, mapW, mapH, mapN, p.BW, p.BH, 1, f16);
        if (rc) return rc;
        rc = make_act_map_strided(&mXLo, in_lo, g->Cin, inW, inH, mapN, p.BW, p.BH, g->mul, f16);
        if (rc) return rc;
    } else { mDyLo = mDy; mXLo = mX; }
    if ((rc = ensure_err_flag())) return rc;
    const size_t smem = (size_t)p.stages * stage_bytes + kt_bytes + 1024;
    dim3 grid((unsigned)(tiles_co * p.tiles_ci), (unsigned)g->ntaps, (unsigned)split);
    cudaStream_t st = (cudaStream_t)stream;
    if (f16) {
        if (BN == 128) return launch_wgrad<128, 1>(mDy, mDyLo, mX, mXLo, p, grid, smem, st, dw, oscale_ptr);
        return launch_wgrad<64, 1>(mDy, mDyLo, mX, mXLo, p, grid, smem, st, dw, oscale_ptr);
    }
    if (BN == 128) return launch_wgrad<128, 0>(mDy, mDyLo, mX, mXLo, p, grid, smem, st, dw, oscale_ptr);
    if (BN == 64) return launch_wgrad<64, 0>(mDy, mDyLo, mX, mXLo, p, grid, smem, st, dw, oscale_ptr);
    return launch_wgrad<32, 0>(mDy, mDyLo, mX, mXLo, p, grid, smem, st, dw, oscale_ptr);
}
