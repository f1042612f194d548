// linear_wgmma.cu -- out[M,128] = act(x[M,128] @ W[128,128] + bias) on the Hopper tensor cores (wgmma.mma_async
// m64n128k8 .tf32, operands in shared memory, x tiles staged by TMA), with 3xTF32 error compensation
// (x_lo*w_hi + x_hi*w_lo + x_hi*w_hi accumulated in one fp32 accumulator: fp32-level accuracy).
// The K = N = 128 fast path of pglb_linear_tf32x3_f32 (the dense transform of the conv layers, reference
// pgl/nn/conv.py:238-251); other shapes stay on the mma.sync kernel in linear_tc.cu.
//
//   * x tiles arrive by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B): one thread keeps STAGES x 16 KB in flight, and
//     the bytes land in the canonical K-major layout wgmma reads.  The raw fp32 tile IS the "hi" operand (.tf32 ignores
//     the low 13 mantissa bits); each consumer warpgroup derives lo = x - trunc_tf32(x) for its own 64 rows.
//   * W^T hi / lo are built once per CTA in the same swizzled K-major layout (B operand: rows = output columns).
//   * bias + ReLU are applied to the accumulator registers on the way out.
// One persistent CTA per SM, 3 warpgroups: 0 = TMA producer (one thread), 1 and 2 = consumers, each owning 64 rows of
// every 128-row tile.  Shared memory: W^T hi / lo (128 KB), STAGES x (raw + lo) K blocks of the x tile (32 KB each).
#include <cuda.h>

#include "common.cuh"

namespace pglb {
namespace wg {

constexpr int BM = 128, BN = 128, BK = 32, KTOT = 128, KBLOCKS = KTOT / BK;
constexpr int STAGES = 3;
constexpr int KB_BYTES = BM * BK * 4;                  // 16 KB: one [128][32] fp32 block
constexpr int HALF_BYTES = KB_BYTES / 2;               // one consumer's 64 rows of it
constexpr int W_BYTES = 2 * KBLOCKS * KB_BYTES;        // W^T hi + lo
constexpr int A_STAGE_BYTES = 2 * KB_BYTES;            // raw (= hi) + lo
constexpr int SMEM_BYTES = 1024 + W_BYTES + STAGES * A_STAGE_BYTES + 256;
constexpr int CONSUMERS = 2;
constexpr int THREADS = (1 + CONSUMERS) * 128;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// a barrier that never completes (a protocol bug, a tensor map that does not describe the buffer) must surface as a
// launch failure on the host, not as a hung device
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try(bar, parity))
        if (++spins > (1u << 24)) __trap();
}

// K-major SWIZZLE_128B operand block [rows][32 fp32]: row r at r * 128 B, its 16-byte chunk c at (c ^ (r & 7)).
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// wgmma shared-memory matrix descriptor: start >> 4 [0,14) | LBO >> 4 [16,30) (unused by K-major swizzled operands) |
// SBO >> 4 [32,46) = 1024 B between 8-row core-matrix groups | layout SWIZZLE_128B = 1 [62,64).  Blocks are 1024-byte
// aligned, so stepping K inside the 128-byte swizzle atom is a plain add to the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// d[64 rows of this warpgroup][128 columns] (+)= A[64][8] B[128][8]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// the previous commit group is complete (the one just committed may still run)
__device__ __forceinline__ void wgmma_wait_prev() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
template <typename T>
__device__ __forceinline__ void wgmma_wait_all(T &d) {
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");   // the accumulator is final only now
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
        "l"(tm), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}

__global__ void __launch_bounds__(THREADS, 1)
linear_wgmma_kernel(const __grid_constant__ CUtensorMap tmx, const float *__restrict__ w,
                    const float *__restrict__ bias, float *__restrict__ out, int64_t ldo, int64_t M, int act) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char *w_hi = smem;                            // [KBLOCKS][128 n][32 k]
    unsigned char *w_lo = smem + KBLOCKS * KB_BYTES;
    unsigned char *a_st = smem + W_BYTES;                  // [STAGES][raw, lo][128 m][32 k]
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + W_BYTES + STAGES * A_STAGE_BYTES);
    // barriers: full[S] (TMA bytes landed), empty[S] (both consumers' MMAs are done with the stage)
    const uint32_t bar0 = smem_u32(bars);
    auto full = [&](int s) { return bar0 + 8 * s; };
    auto empty = [&](int s) { return bar0 + 8 * (STAGES + s); };

    const int tid = threadIdx.x, wgi = tid >> 7;

    // ---- one-time setup: barriers, W^T split into hi / lo in the swizzled K-major layout ----
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full(s), 1);
            mbar_init(empty(s), CONSUMERS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < KTOT * BN; i += THREADS) {
        const int k = i / BN, n = i - k * BN;              // coalesced read of W[k][n]
        const float f = w[i];
        const uint32_t hi = to_tf32(f);
        const uint32_t lo = to_tf32(f - __uint_as_float(hi));
        const int kb = k / BK, kk = k - kb * BK;
        const uint32_t off = kb * KB_BYTES + sw128_offset(n, kk >> 2) + (kk & 3) * 4;
        *reinterpret_cast<uint32_t *>(w_hi + off) = hi;
        *reinterpret_cast<uint32_t *>(w_lo + off) = lo;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const int64_t tiles = (M + BM - 1) / BM;

    if (wgi == 0) {
        // ================= TMA producer (one thread) =================
        if (tid == 0) {
            uint32_t it = 0;
            for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                for (int kb = 0; kb < KBLOCKS; ++kb, ++it) {
                    const int s = it % STAGES;
                    const uint32_t ph = (it / STAGES) & 1;
                    mbar_wait(empty(s), ph ^ 1);           // both consumers have drained this stage (passes on the first lap)
                    mbar_expect_tx(full(s), KB_BYTES);
                    // rows past M are zero-filled by the TMA unit
                    tma_load_2d(smem_u32(a_st + s * A_STAGE_BYTES), &tmx, kb * BK, (int)(tile * BM), full(s));
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup c owns rows [64 c, 64 c + 64) of every tile =================
    const int c = wgi - 1;
    const int t = tid & 127, warp = t >> 5, lane = t & 31;
    const int g = lane >> 2, q = lane & 3;
    float acc[64];
    uint32_t it = 0;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int prev = 0;
        for (int kb = 0; kb < KBLOCKS; ++kb, ++it) {
            const int s = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            mbar_wait(full(s), ph);
            unsigned char *raw = a_st + s * A_STAGE_BYTES + c * HALF_BYTES;
            unsigned char *lo_b = raw + KB_BYTES;
            // lo = x - trunc_tf32(x), at the same swizzled position (any 16-byte piece: lo sits where hi sits)
#pragma unroll
            for (int i = 0; i < HALF_BYTES / 16 / 128; ++i) {
                const int off = (t + i * 128) * 16;
                const float4 v = *reinterpret_cast<const float4 *>(raw + off);
                float4 l;
                l.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
                l.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
                l.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
                l.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
                *reinterpret_cast<float4 *>(lo_b + off) = l;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("bar.sync %0, 128;" ::"r"(1 + c) : "memory");   // this warpgroup's lo half is complete
            wgmma_fence();
            const uint32_t x_hi = smem_u32(raw), x_lo = smem_u32(lo_b);
            const uint32_t wt_hi = smem_u32(w_hi + kb * KB_BYTES), wt_lo = smem_u32(w_lo + kb * KB_BYTES);
#pragma unroll
            for (int k = 0; k < BK / 8; ++k) {             // 32 bytes of K per instruction inside the 128-B atom
                const uint32_t ko = k * 32;
                wgmma_tf32(acc, make_desc(x_lo + ko), make_desc(wt_hi + ko), (kb | k) ? 1u : 0u);
                wgmma_tf32(acc, make_desc(x_hi + ko), make_desc(wt_lo + ko), 1u);
                wgmma_tf32(acc, make_desc(x_hi + ko), make_desc(wt_hi + ko), 1u);
            }
            wgmma_commit();
            // the MMAs of this K block run while the next block is split; the previous block's stage is free
            if (kb > 0) {
                wgmma_wait_prev();
                if (t == 0) mbar_arrive(empty(prev));
            }
            prev = s;
        }
        wgmma_wait_all(acc);
        if (t == 0) mbar_arrive(empty(prev));
        // epilogue: accumulator j of n8 block i holds (row g (+8 for j & 2), column 8 i + 2 q + (j & 1))
        const int64_t r0 = tile * BM + c * 64 + warp * 16 + g;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            const int col = i * 8 + 2 * q;
            float bx = 0.f, by = 0.f;
            if (bias) {
                bx = __ldg(bias + col);
                by = __ldg(bias + col + 1);
            }
            float2 v0 = make_float2(acc[4 * i] + bx, acc[4 * i + 1] + by);
            float2 v1 = make_float2(acc[4 * i + 2] + bx, acc[4 * i + 3] + by);
            if (act == 1) {
                v0.x = fmaxf(v0.x, 0.f); v0.y = fmaxf(v0.y, 0.f);
                v1.x = fmaxf(v1.x, 0.f); v1.y = fmaxf(v1.y, 0.f);
            }
            if (r0 < M) __stcs(reinterpret_cast<float2 *>(out + r0 * ldo + col), v0);
            if (r0 + 8 < M) __stcs(reinterpret_cast<float2 *>(out + (r0 + 8) * ldo + col), v1);
        }
    }
}

typedef CUresult (*TmapEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                 const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace wg

// K = N = 128, x rows 16-byte aligned (ldx % 4 == 0), out 8-byte aligned with even ldo: checked by the caller
int linear_wgmma_run(const float *x, int64_t ldx, const float *w, const float *bias, float *out, int64_t ldo,
                     int64_t M, int act, cudaStream_t stream) {
    using namespace wg;
    static std::atomic<void *> enc_fn{nullptr};
    void *f = enc_fn.load(std::memory_order_acquire);
    if (!f) {
        cudaDriverEntryPointQueryResult q;
        void *g = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &g, cudaEnableDefault, &q) == cudaSuccess && g) {
            enc_fn.store(g, std::memory_order_release);
            f = g;
        }
    }
    PGLB_CHECK_ARG(f != nullptr, PGLB_EINVAL, "cuTensorMapEncodeTiled not available from the driver");
    CUtensorMap tm;
    cuuint64_t dims[2] = {(cuuint64_t)KTOT, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)ldx * 4};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    cuuint32_t es[2] = {1, 1};
    const CUresult r = reinterpret_cast<TmapEncodeFn>(f)(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(x), dims,
                                                         strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PGLB_CHECK_ARG(r == CUDA_SUCCESS, PGLB_EINVAL, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(linear_wgmma_kernel, SMEM_BYTES, attr_done));
    const int64_t tiles = (M + BM - 1) / BM;
    const unsigned grid = (unsigned)(tiles < sm_count() ? tiles : sm_count());
    linear_wgmma_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(tm, w, bias, out, ldo, M, act);
    PGLB_LAUNCH_CHECK("linear_wgmma_kernel");
    return PGLB_OK;
}

}  // namespace pglb
