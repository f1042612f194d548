// common.cuh -- shared helpers for libpglb (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
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

// ---- device helpers -------------------------------------------------------------------

// streaming (evict-first) loads for index data that is read exactly once
__device__ __forceinline__ int64_t ld_stream(const int64_t *p) { return __ldcs((const long long *)p); }
__device__ __forceinline__ int64_t ld_ro(const int64_t *p) { return __ldg((const long long *)p); }

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

}  // namespace pglb
