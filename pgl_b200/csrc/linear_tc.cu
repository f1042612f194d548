// linear_tc.cu -- out = act(x @ W + bias) for the conv layers' dense transform (reference
// pgl/nn/conv.py:238-251 `self.linear(...)`, `+ self.bias`, activation) on the tensor cores with
// fp32-level accuracy: 3xTF32 error-compensated products
//     x*w ~= x_hi*w_hi + x_lo*w_hi + x_hi*w_lo,   x_hi = tf32(x), x_lo = tf32(x - x_hi)
// accumulated in fp32 (`mma.sync.m16n8k8.tf32`), with bias + ReLU fused into the epilogue so the
// [M, N] result is written exactly once.  M is the node count (10^7 at cfg5), K, N <= 128: the GEMM is
// "tall and skinny", W (64 KB) is split once into interleaved {hi, lo} pairs and stays resident in
// shared memory, a persistent CTA per SM streams 64-row tiles of x through a cp.async double buffer.
// HBM traffic = one read of x + one write of out (10.24 GB at cfg5; the fp32 cuBLAS addmm + separate
// ReLU it replaces moved 20.5 GB and ran on the CUDA cores).
//
// K = N = 128 goes to the wgmma kernel of linear_wgmma.cu; this kernel takes every other shape.
#include <algorithm>

#include "common.cuh"

namespace pglb {

constexpr int LT_ROWS = 64;        // rows of x per tile: 4 row blocks of 16
constexpr int LT_WARPS = 8;  // 4 row blocks x 2 column groups
constexpr int LT_KMAX = 128;
constexpr int LT_XS = LT_KMAX + 4;  // x tile row stride (floats): 132 = 4 mod 32 -> conflict-free A loads

__device__ __forceinline__ void cp_async16_zfill(void *smem, const void *gmem, int src_bytes) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes)
                 : "memory");
}

// N = output width (64 or 128).  Dynamic shared memory:
//   W2 [LT_KMAX][N + 4] of {hi, lo} tf32 pairs (rows >= K are zero)
//   X  [2][LT_ROWS][LT_XS] fp32 (columns >= K stay zero)
template <int N>
__global__ void __launch_bounds__(LT_WARPS * 32, 1)
linear_tf32x3_kernel(const float *__restrict__ x, int64_t ldx, const float *__restrict__ w,
                     const float *__restrict__ bias, float *__restrict__ out, int64_t ldo, int64_t M,
                     int K, int act) {
    constexpr int WS = N + 4;    // W2 row stride in pairs: (N+4) = 4 mod 16 -> conflict-free LDS.64
    constexpr int LT_THREADS = LT_WARPS * 32;
    constexpr int CG = LT_WARPS / 4;    // column groups
    constexpr int WCOLS = N / CG;    // columns owned by one warp
    constexpr int NT = WCOLS / 8;    // 8-wide column tiles per warp
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint2 *W2 = reinterpret_cast<uint2 *>(smem_raw);
    float *X = reinterpret_cast<float *>(smem_raw + sizeof(uint2) * LT_KMAX * WS);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int K8 = (K + 7) & ~7;

    // W -> {hi, lo}; zero rows beyond K; zero both x buffers (their pad columns are never written)
    for (int i = tid; i < LT_KMAX * WS; i += LT_THREADS) {
        const int k = i / WS, n = i - k * WS;
        uint2 v = make_uint2(0u, 0u);
        if (k < K && n < N) {
            const float f = w[(int64_t)k * N + n];
            const uint32_t hi = to_tf32(f);
            v = make_uint2(hi, to_tf32(f - __uint_as_float(hi)));
        }
        W2[i] = v;
    }
    for (int i = tid; i < 2 * LT_ROWS * LT_XS; i += LT_THREADS) X[i] = 0.f;
    __syncthreads();

    const int64_t tiles = (M + LT_ROWS - 1) / LT_ROWS;
    const int kchunks = K >> 2;  // 16-byte chunks per row (K % 4 == 0)
    auto prefetch = [&](int64_t tile, int buf) {
        float *dst = X + buf * (LT_ROWS * LT_XS);
        const int64_t r0 = tile * LT_ROWS;
        for (int i = tid; i < LT_ROWS * kchunks; i += LT_THREADS) {
            const int r = i / kchunks, c = i - r * kchunks;
            const int64_t row = r0 + r;
            const bool ok = row < M;
            const float *src = x + (ok ? row : 0) * ldx + c * 4;
            cp_async16_zfill(dst + r * LT_XS + c * 4, src, ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    int64_t tile = blockIdx.x;
    if (tile < tiles) prefetch(tile, 0);
    int buf = 0;
    for (; tile < tiles; tile += gridDim.x, buf ^= 1) {
        const int64_t next = tile + gridDim.x;
        if (next < tiles) {
            prefetch(next, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();

        const float *xt = X + buf * (LT_ROWS * LT_XS) + (wm * 16) * LT_XS;
        float acc[NT][4];
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;

        for (int k0 = 0; k0 < K8; k0 += 8) {
            float af[4];
            af[0] = xt[g * LT_XS + k0 + t];
            af[1] = xt[(g + 8) * LT_XS + k0 + t];
            af[2] = xt[g * LT_XS + k0 + t + 4];
            af[3] = xt[(g + 8) * LT_XS + k0 + t + 4];
            uint32_t ahi[4], alo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                ahi[i] = to_tf32(af[i]);
                alo[i] = to_tf32(af[i] - __uint_as_float(ahi[i]));
            }
            uint2 b0[NT], b1[NT];
            const uint2 *wr0 = W2 + (k0 + t) * WS + wn * WCOLS + g;
            const uint2 *wr1 = wr0 + 4 * WS;
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                b0[j] = wr0[j * 8];
                b1[j] = wr1[j * 8];
            }
            // small terms first; the three passes keep NT independent accumulators in flight
#pragma unroll
            for (int j = 0; j < NT; ++j) mma_tf32(acc[j], alo, b0[j].x, b1[j].x);
#pragma unroll
            for (int j = 0; j < NT; ++j) mma_tf32(acc[j], ahi, b0[j].y, b1[j].y);
#pragma unroll
            for (int j = 0; j < NT; ++j) mma_tf32(acc[j], ahi, b0[j].x, b1[j].x);
        }

        // epilogue: + bias, activation, one write.  c0,c1 -> (row g, cols 2t, 2t+1); c2,c3 -> row g+8
        const int64_t row0 = tile * LT_ROWS + wm * 16 + g;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int col = wn * WCOLS + j * 8 + 2 * t;
            float bx = 0.f, by = 0.f;
            if (bias) {
                bx = __ldg(bias + col);
                by = __ldg(bias + col + 1);
            }
            float2 v0 = make_float2(acc[j][0] + bx, acc[j][1] + by);
            float2 v1 = make_float2(acc[j][2] + bx, acc[j][3] + by);
            if (act == 1) {
                v0.x = fmaxf(v0.x, 0.f);
                v0.y = fmaxf(v0.y, 0.f);
                v1.x = fmaxf(v1.x, 0.f);
                v1.y = fmaxf(v1.y, 0.f);
            }
            if (row0 < M) *reinterpret_cast<float2 *>(out + row0 * ldo + col) = v0;
            if (row0 + 8 < M) *reinterpret_cast<float2 *>(out + (row0 + 8) * ldo + col) = v1;
        }
        __syncthreads();  // everyone is done with X[buf] before the next prefetch overwrites it
    }
}

template <int N>
static int launch(const float *x, int64_t ldx, const float *w, const float *bias, float *out,
                  int64_t ldo, int64_t M, int K, int act, cudaStream_t stream) {
    const size_t smem = sizeof(uint2) * LT_KMAX * (N + 4) + sizeof(float) * 2 * LT_ROWS * LT_XS;
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(linear_tf32x3_kernel<N>, (int)smem, attr_done));
    const int64_t tiles = (M + LT_ROWS - 1) / LT_ROWS;
    const unsigned grid = (unsigned)std::min<int64_t>(tiles, sm_count());
    linear_tf32x3_kernel<N><<<grid, LT_WARPS * 32, smem, stream>>>(x, ldx, w, bias, out, ldo, M, K, act);
    PGLB_LAUNCH_CHECK("linear_tf32x3_kernel");
    return PGLB_OK;
}

}  // namespace pglb

namespace pglb {
int linear_wgmma_run(const float *x, int64_t ldx, const float *w, const float *bias, float *out, int64_t ldo,
                     int64_t M, int act, cudaStream_t stream);
}  // namespace pglb

extern "C" int pglb_linear_tf32x3_f32(const float *x, int64_t ldx, const float *w, const float *bias,
                                      float *out, int64_t ldo, int64_t M, int64_t K, int64_t N,
                                      int act, void *stream) {
    using namespace pglb;
    PGLB_CHECK_ARG(M >= 0, PGLB_EINVAL, "pglb_linear_tf32x3_f32: negative row count");
    PGLB_CHECK_ARG(K >= 4 && K <= LT_KMAX && K % 4 == 0, PGLB_ESHAPE,
                   "pglb_linear_tf32x3_f32: K must be a multiple of 4 in [4, 128] (got %lld)", (long long)K);
    PGLB_CHECK_ARG(N == 64 || N == 128, PGLB_ESHAPE,
                   "pglb_linear_tf32x3_f32: N must be 64 or 128 (got %lld)", (long long)N);
    PGLB_CHECK_ARG(act == 0 || act == 1, PGLB_EINVAL, "pglb_linear_tf32x3_f32: act must be 0 (none) or 1 (relu)");
    if (M == 0) return PGLB_OK;
    PGLB_CHECK_ARG(x && w && out, PGLB_EINVAL, "pglb_linear_tf32x3_f32: NULL pointer");
    PGLB_CHECK_ARG(ldx >= K && ldx % 4 == 0 && ldo >= N && ldo % 2 == 0, PGLB_ESHAPE,
                   "pglb_linear_tf32x3_f32: ldx must be >= K and a multiple of 4, ldo >= N and even");
    PGLB_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 8) == 0, PGLB_EINVAL,
                   "pglb_linear_tf32x3_f32: x must be 16-byte and out 8-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    // K = N = 128 (the conv layers' hidden size): wgmma / TMA kernel (csrc/linear_wgmma.cu)
    if (K == 128 && N == 128) return linear_wgmma_run(x, ldx, w, bias, out, ldo, M, act, s);
    if (N == 128) return launch<128>(x, ldx, w, bias, out, ldo, M, (int)K, act, s);
    return launch<64>(x, ldx, w, bias, out, ldo, M, (int)K, act, s);
}
