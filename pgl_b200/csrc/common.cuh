// common.cuh -- shared helpers for libpglb (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "pglb.h"

namespace pglb {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;

int fail(int code, const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define PGLB_CHECK_ARG(cond, code, ...)                  \
    do {                                                 \
        if (!(cond)) return ::pglb::fail(code, __VA_ARGS__); \
    } while (0)

#define PGLB_CUDA(call)                                             \
    do {                                                            \
        cudaError_t _e = (call);                                    \
        if (_e != cudaSuccess) return ::pglb::cuda_fail(_e, #call); \
    } while (0)

#define PGLB_LAUNCH_CHECK(name)                                     \
    do {                                                            \
        ::pglb::count_launch();                                     \
        cudaError_t _e = cudaGetLastError();                        \
        if (_e != cudaSuccess) return ::pglb::cuda_fail(_e, name);  \
    } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}

// SM count of the CURRENT device (cached per device: a process may drive several GPUs).
inline int sm_count() {
    static std::atomic<int> cache[64];
    const int dev = current_device();
    int n = cache[dev & 63].load(std::memory_order_relaxed);
    if (n == 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        cache[dev & 63].store(n, std::memory_order_relaxed);
    }
    return n;
}

// Opt a kernel into more than 48 KB of dynamic shared memory.  The attribute is per device, so the
// "already done" flag is a bit per device (one mask per kernel instantiation, owned by the caller).
template <typename K>
inline cudaError_t ensure_dyn_smem(K kernel, int bytes, std::atomic<unsigned long long> &done) {
    const unsigned long long bit = 1ull << (current_device() & 63);
    if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
    return e;
}

// multi-block int64 prefix sum (csr_build.cu): in and out may alias, tmp holds scan_i64_ws_bytes(n) bytes
size_t scan_i64_ws_bytes(int64_t n);
int scan_i64(const int64_t *in, int64_t *out, int64_t n, int inclusive, void *tmp, cudaStream_t stream);

// the stable LSD radix sort of pglb_csr_build (csr_build.cu) over (uint64 key, uint64 value) pairs, key bits [0, bits):
// equal keys keep their input order.  keys_alt / vals_alt are n-element scratch; *result_in_alt says which pair of
// buffers holds the sorted result.  tmp: radix_sort_u64_ws_bytes(n) bytes, 256-byte aligned.
size_t radix_sort_u64_ws_bytes(int64_t n);
int radix_sort_u64(uint64_t *keys, uint64_t *vals, uint64_t *keys_alt, uint64_t *vals_alt, int64_t n, int bits,
                   void *tmp, cudaStream_t stream, int *result_in_alt);

// ---- device helpers -------------------------------------------------------------------

// streaming (evict-first) loads for index data that is read exactly once
__device__ __forceinline__ int64_t ld_stream(const int64_t *p) { return __ldcs((const long long *)p); }
__device__ __forceinline__ int64_t ld_ro(const int64_t *p) { return __ldg((const long long *)p); }

// Row epilogue of pglb_propagate_f32 / pglb_propagate_narrow_f32 (include/pglb.h), read only by the kernel
// instantiations with PROP = true.  With t the row the plain aggregation would write:
//   y = a t (+ b h),  out = y,  acc_out = acc_in + c y  (c = *c_dev when c_dev is set)
// Every product and sum is rounded on its own (no FMA contraction), the order torch's op-by-op hop rounds in.
struct PropEpi {
    const float *h;       // nullable [n, ldh]
    int64_t ldh;
    const float *acc_in;  // nullable [n, ld_acc_in]; may be acc_out itself (in place)
    int64_t ld_acc_in;
    float *acc_out;       // nullable [n, ld_acc_out]
    int64_t ld_acc_out;
    float a, b, c;
    const float *c_dev;   // nullable: device copy of c
};
__device__ __forceinline__ float prop_c(const PropEpi &e) { return e.c_dev ? __ldg(e.c_dev) : e.c; }
// y for one element; hv is read only when e.h is set
__device__ __forceinline__ float prop_y(const PropEpi &e, float t, float hv) {
    return e.h ? __fadd_rn(__fmul_rn(e.a, t), __fmul_rn(e.b, hv)) : __fmul_rn(e.a, t);
}
__device__ __forceinline__ float4 prop_y4(const PropEpi &e, float4 t, float4 hv) {
    return make_float4(prop_y(e, t.x, hv.x), prop_y(e, t.y, hv.y), prop_y(e, t.z, hv.z), prop_y(e, t.w, hv.w));
}
__device__ __forceinline__ float4 prop_acc4(float4 ai, float c, float4 y) {
    return make_float4(__fadd_rn(ai.x, __fmul_rn(c, y.x)), __fadd_rn(ai.y, __fmul_rn(c, y.y)),
                       __fadd_rn(ai.z, __fmul_rn(c, y.z)), __fadd_rn(ai.w, __fmul_rn(c, y.w)));
}
// h and acc_in of row r at column c0, loaded when the row opens (row < n_rows, active lanes)
__device__ __forceinline__ void prop_open4(const PropEpi &e, int64_t r, int64_t n_rows, bool act, int c0, float4 &hv,
                                           float4 &ai) {
    if (!act || r >= n_rows) return;
    if (e.h) hv = __ldg(reinterpret_cast<const float4 *>(e.h + r * e.ldh + c0));
    if (e.acc_out) ai = *reinterpret_cast<const float4 *>(e.acc_in + r * e.ld_acc_in + c0);
}
// the epilogue of a 4-column piece of row r at column c0 (16-byte aligned rows): writes out and acc_out.  acc_in is
// read with a plain load: in place it is the row acc_out is about to receive.
__device__ __forceinline__ void prop_store4(const PropEpi &e, float c, float *out, int64_t ldo, int64_t r, int c0,
                                            float4 t) {
    const float4 hv = e.h ? __ldg(reinterpret_cast<const float4 *>(e.h + r * e.ldh + c0)) : t;
    const float4 y = prop_y4(e, t, hv);
    *reinterpret_cast<float4 *>(out + r * ldo + c0) = y;
    if (e.acc_out) {
        const float4 ai = *reinterpret_cast<const float4 *>(e.acc_in + r * e.ld_acc_in + c0);
        *reinterpret_cast<float4 *>(e.acc_out + r * e.ld_acc_out + c0) = prop_acc4(ai, c, y);
    }
}

// 3xTF32 products (linear_tc.cu, rgcn.cu): x*w ~= x_lo*w_hi + x_hi*w_lo + x_hi*w_hi with x_hi = tf32(x),
// x_lo = tf32(x - x_hi), each term one mma.sync.m16n8k8 accumulating in fp32
__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 16-bit feature elements of pglb_spmm_csr_x16, handled as raw bits: widen() is exact, round() is the one
// round-to-nearest-even of a value computed in fp32.  lo / hi = the element in the low / high half of a 32-bit word.
template <typename T>
struct X16;
template <>
struct X16<__nv_bfloat16> {
    static __device__ __forceinline__ float widen(unsigned short b) { return __uint_as_float((unsigned)b << 16); }
    static __device__ __forceinline__ float lo(unsigned w) { return __uint_as_float(w << 16); }
    static __device__ __forceinline__ float hi(unsigned w) { return __uint_as_float(w & 0xffff0000u); }
    static __device__ __forceinline__ unsigned short round(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }
};
template <>
struct X16<__half> {
    static __device__ __forceinline__ float widen(unsigned short b) { return __half2float(__ushort_as_half(b)); }
    static __device__ __forceinline__ float lo(unsigned w) { return widen((unsigned short)(w & 0xffffu)); }
    static __device__ __forceinline__ float hi(unsigned w) { return widen((unsigned short)(w >> 16)); }
    static __device__ __forceinline__ unsigned short round(float f) { return __half_as_ushort(__float2half_rn(f)); }
};
// four consecutive 16-bit elements (8 bytes) <-> float4
template <typename T>
__device__ __forceinline__ float4 widen4(uint2 v) {
    return make_float4(X16<T>::lo(v.x), X16<T>::hi(v.x), X16<T>::lo(v.y), X16<T>::hi(v.y));
}
template <typename T>
__device__ __forceinline__ uint2 round4(float4 v) {
    return make_uint2((unsigned)X16<T>::round(v.x) | ((unsigned)X16<T>::round(v.y) << 16),
                      (unsigned)X16<T>::round(v.z) | ((unsigned)X16<T>::round(v.w) << 16));
}
// four consecutive elements of a row in global memory (read-only path) as fp32: 16 bytes of float32, or 8 bytes of a
// 16-bit type widened exactly
template <typename T>
__device__ __forceinline__ float4 ldg_row4(const T *p) {
    if constexpr (sizeof(T) == 4) return __ldg(reinterpret_cast<const float4 *>(p));
    else return widen4<T>(__ldg(reinterpret_cast<const uint2 *>(p)));
}

// The score of the dot-product attention kernels (spmm_gat5_kernel<DOT>, dot_attn_bwd_edge_kernel): a lane's 4-term
// partial dot, then the sum over the lph lanes of its head (lph a power of two, warp-uniform, every lane of the warp
// calling).  The forward and the edge backward both call these two, so they form the same score bit for bit, and
// every lane of a head holds the same bits.
__device__ __forceinline__ float dot4_lane(const float4 &a, const float4 &b) {
    return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}
// the edge-feature operand of the dot-product attention (spmm_gat5_kernel<kScoreDotE>, dot_attn_bwd_edge_kernel<EF>):
// k + e and v + e, formed the same way in the forward and the backward
__device__ __forceinline__ float4 add4(const float4 &a, const float4 &b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float head_sum_lanes(float v, int lph) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1)
        if (o < lph) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The GATv2 score (spmm_gat5_kernel<kScoreV2>, gatv2_bwd_edge_kernel, gatv2_score_grad_kernel): a lane's 4-term
// partial sum_c a_c lrelu(fs_c + fd_c), then head_sum_lanes over its head.  lrelu(x) = max(x, slope x) for
// 0 <= slope <= 1.  The forward and the edge backward call the same function, so they form the same score bit for bit.
__device__ __forceinline__ float lrelu_of(float x, float slope) { return fmaxf(x, x * slope); }
__device__ __forceinline__ float gatv2_lane(const float4 &a, const float4 &fs, const float4 &fd, float slope) {
    return fmaf(a.w, lrelu_of(fs.w + fd.w, slope),
                fmaf(a.z, lrelu_of(fs.z + fd.z, slope),
                     fmaf(a.y, lrelu_of(fs.y + fd.y, slope), a.x * lrelu_of(fs.x + fd.x, slope))));
}

// The FAConv edge weight (spmm_gat5_kernel<kScoreFA>, fa_bwd_edge_kernel): t = tanh(gs + gd) in full precision
// (tanhf, not tanh.approx), w = (t * nu) * nd -- the reference's h * src_norm * dst_norm -- and, with dropout (DROP),
// w = keep ? s * w : 0.  The forward and the edge backward call this one function, so the backward's beta is the forward's weight
// bit for bit; *t receives t for the backward's (1 - t^2).
template <bool DROP>
__host__ __device__ __forceinline__ float fa_weight(float gs, float gd, float nu, float nd, bool keep, float s,
                                                    float *t) {
    *t = tanhf(gs + gd);
    const float w = (*t * nu) * nd;
    if constexpr (DROP) return keep ? s * w : 0.0f;
    else return w;
}

// ---- attention dropout of the fused GAT training path (the *_drop_* entries) ----------------------------------------
// The keep decision of dst-CSR slot j (absolute slot index) and head h, for drop probability p:
//   draw = Philox4x32-10(counter = (j lo32, j hi32, h / 4, offset / 4), key = (seed lo32, seed hi32)) word h % 4
//   kept iff draw >= thresh,  thresh = min(floor(p * 2^32), 2^32 - 1);  a kept weight is scaled by s = 1 / (1 - p)
// (Philox: Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011).  attn_keep_word is the
// only statement of this rule: the forward kernel, the backward edge kernel and pglb_attn_dropout_keep_host call it,
// so the forward and the backward recompute the same mask in registers and no [E, H] mask exists.
struct AttnDrop {
    uint64_t seed;
    uint32_t ctr3;     // offset / 4: counter word 3
    uint32_t thresh;   // kept iff draw >= thresh
    float scale;       // s = (float)(1 / (1 - p))
};

// the argument checks every attention-dropout entry makes before anything else: 0 < p < 1 (NaN fails), offset % 4 == 0
inline int attn_drop_check(const char *name, float p, uint64_t offset) {
    PGLB_CHECK_ARG(p > 0.0f && p < 1.0f, PGLB_EINVAL, "%s: attn_drop must lie in (0, 1)", name);
    PGLB_CHECK_ARG(offset % 4 == 0, PGLB_EINVAL, "%s: offset must be a multiple of 4", name);
    return PGLB_OK;
}

// thresh and s derived in double from the float p an entry receives (after attn_drop_check)
inline AttnDrop attn_drop_of(float p, uint64_t seed, uint64_t offset) {
    AttnDrop d;
    const double t = floor((double)p * 4294967296.0);
    d.seed = seed;
    d.ctr3 = (uint32_t)(offset / 4);
    d.thresh = t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
    d.scale = (float)(1.0 / (1.0 - (double)p));
    return d;
}

__host__ __device__ __forceinline__ uint32_t mulhilo32(uint32_t a, uint32_t b, uint32_t *hi) {
#ifdef __CUDA_ARCH__
    *hi = __umulhi(a, b);
    return a * b;
#else
    const uint64_t m = (uint64_t)a * b;
    *hi = (uint32_t)(m >> 32);
    return (uint32_t)m;
#endif
}

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        uint32_t hi0, hi1;
        const uint32_t lo0 = mulhilo32(0xD2511F53u, c.x, &hi0);
        const uint32_t lo1 = mulhilo32(0xCD9E8D57u, c.z, &hi1);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// keep word of slot j: bit h = head h kept (H % 4 == 0, H <= 32: one Philox call per four heads)
__host__ __device__ __forceinline__ uint32_t attn_keep_word(const AttnDrop &d, uint64_t j, int H) {
    uint32_t w = 0;
    for (int q = 0; q < H / 4; ++q) {
        const uint4 r = philox4x32_10(make_uint4((uint32_t)j, (uint32_t)(j >> 32), (uint32_t)q, d.ctr3),
                                      (uint32_t)d.seed, (uint32_t)(d.seed >> 32));
        const uint32_t b = (uint32_t)(r.x >= d.thresh) | ((uint32_t)(r.y >= d.thresh) << 1) |
                           ((uint32_t)(r.z >= d.thresh) << 2) | ((uint32_t)(r.w >= d.thresh) << 3);
        w |= b << (4 * q);
    }
    return w;
}

}  // namespace pglb
