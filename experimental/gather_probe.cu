// gather_probe.cu -- what is the ceiling of a random 512-byte row gather on one GPU, by mechanism?
//
// Standalone (nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o gather_probe gather_probe.cu).
// Not part of libpglb.so.  This probe strips everything but the gather + an in-order sum so the
// mechanisms the aggregation kernels can use are compared on equal terms:
//   mode 0  LDG.128 per lane per row, 8 rows in flight per lane (registers)
//   mode 1  cp.async.bulk (UBLKCP) 512 B per row from an elected lane, mbarrier per group of GR rows
//   mode 2  cp.async.bulk 512 B per row from the lane that holds the row id (spmm_v5's mechanism)
//   mode 3  LDGSTS per lane per row (cp.async.cg 16 B), commit groups of 4
//   mode 4  hybrid: a row whose id has bit 31 set is fetched by all 32 lanes (cp.async.cg 16 B, L2 evict_last) into
//           its ring slot, every other row by mode 2's bulk copy (evict_first); the mbarrier expects only the bulk bytes
// Every warp reduces chunks of T indices; the sum is written once per chunk (keeps the loads live).
// dist 2 draws ids as cfg5 draws sources: w_i = (i+1)^-0.8, scattered by a fixed permutation, and marks the hot_k
// heaviest rows with bit 31 (the packed ids of the aggregation); every mode gathers id & 0x7fffffff.  With a small N
// (say 40000 rows = 20 MB) every row stays in L2 and each mechanism shows its rate with no DRAM behind it.
// usage: gather_probe N E dist(0 uniform | 1 skewed | 2 cfg5 power law) [T] [hot_k (dist 2), default 65536 = 32 MB]
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <vector>

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e_ = (x);                                                          \
        if (e_ != cudaSuccess) {                                                       \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            exit(2);                                                                   \
        }                                                                              \
    } while (0)

__device__ __forceinline__ float4 ldg128(const float *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ float4 lds128(unsigned a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned cnt) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(cnt));
}
__device__ __forceinline__ void mbar_expect(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    // bounded: a wrong tensor-map box (fewer bytes than expected) must trap, not hang the box
    for (unsigned spin = 0; spin < (1u << 22); ++spin) {
        unsigned ok;
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok)
                     : "r"(bar), "r"(parity)
                     : "memory");
        if (ok) return;
    }
    __trap();
}
__device__ __forceinline__ void bulk_row(unsigned dst, const void *src, unsigned bytes, unsigned bar) {
    asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_row_hint(unsigned dst, const void *src, unsigned bytes, unsigned bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
        "l"(src), "r"(bytes), "r"(bar), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void cp_async16_hint(unsigned dst, const void *src, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ uint64_t policy(bool keep) {
    uint64_t p;
    if (keep) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    else asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
#define ID_MASK 0x7fffffffu

// ---- mode 0 ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ldg(const float *__restrict__ x, const unsigned *__restrict__ idx, float *out,
                                             long long E, int T) {
    const int lane = threadIdx.x & 31;
    const long long chunk = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long a = chunk * T;
    if (a >= E) return;
    const int cnt = (int)((E - a) < T ? (E - a) : T);
    float4 acc = make_float4(0, 0, 0, 0);
    for (int b = 0; b < cnt; b += 32) {
        const unsigned c = (b + lane < cnt) ? __ldcs(idx + a + b + lane) : 0u;
        const int nb = (cnt - b) < 32 ? (cnt - b) : 32;
        for (int k = 0; k < nb; k += 8) {
            float4 v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const unsigned cj = __shfl_sync(~0u, c, k + j);
                v[j] = (k + j < nb) ? ldg128(x + (size_t)(cj & ID_MASK) * 128 + lane * 4) : make_float4(0, 0, 0, 0);
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                acc.x += v[j].x; acc.y += v[j].y; acc.z += v[j].z; acc.w += v[j].w;
            }
        }
    }
    *reinterpret_cast<float4 *>(out + chunk * 128 + lane * 4) = acc;
}

// ---- modes 1, 2, 4 --------------------------------------------------------------------------------
// per warp: NG group slots of GR rows (GR*512 B each), one mbarrier per slot; LAG = NG - 1 groups in flight.
// HINT (mode 2): bit-31 rows evict_last, the rest evict_first, as spmm_v5 with L2 hints
template <int MODE, int NG, int GR, int W, bool HINT = false>
__global__ void __launch_bounds__(W * 32) k_tma(const float *__restrict__ x, const unsigned *__restrict__ idx, float *out, long long E, int T) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long bars[W * NG];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long chunk = (long long)blockIdx.x * W + wib;
    const long long a = chunk * T;
    const unsigned ring = (unsigned)__cvta_generic_to_shared(smem) + wib * (NG * GR * 512);
    const unsigned bar0 = (unsigned)__cvta_generic_to_shared(&bars[wib * NG]);
    if (lane == 0)
        for (int s = 0; s < NG; ++s) mbar_init(bar0 + s * 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    if (a >= E) return;
    const int cnt = (int)((E - a) < T ? (E - a) : T);  // multiple of 32 in this probe
    const int ngroups = cnt / GR;
    constexpr int LAG = NG - 1;
    constexpr int GPB = 32 / GR;
    float4 acc = make_float4(0, 0, 0, 0);
    const uint64_t pol_keep = (MODE == 4 || HINT) ? policy(true) : 0;
    const uint64_t pol_cold = (MODE == 4 || HINT) ? policy(false) : 0;
    const char *xl = reinterpret_cast<const char *>(x) + lane * 16;
    unsigned lane_slots = 0;  // mode 4: bit s = slot s was last written by per-lane cp.async (generic proxy)
    unsigned c = __ldcs(idx + a + lane);
#pragma unroll 1
    for (int g = 0; g < ngroups + LAG; ++g) {
        if (g < ngroups) {
            const int sub = g % GPB;
            if (sub == 0 && g > 0) c = __ldcs(idx + a + g * GR + lane);
            const int s = g % NG;
            const int k = lane - sub * GR;
            const bool holder = k >= 0 && k < GR;
            const char *src = reinterpret_cast<const char *>(x) + (size_t)(c & ID_MASK) * 512;
            if (MODE == 4 && ((lane_slots >> s) & 1u))
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes, then bulk ones
            __syncwarp();  // every lane is done reading slot s (consumed LAG+1 groups ago)
            if (MODE == 1) {
                if (lane == 0) mbar_expect(bar0 + s * 8, GR * 512);
#pragma unroll
                for (int kk = 0; kk < GR; ++kk) {
                    const unsigned ck = __shfl_sync(~0u, c, sub * GR + kk);
                    if (lane == 0) bulk_row(ring + (s * GR + kk) * 512, x + (size_t)(ck & ID_MASK) * 128, 512, bar0 + s * 8);
                }
            } else if (MODE == 2) {
                if (lane == 0) mbar_expect(bar0 + s * 8, GR * 512);
                __syncwarp();
                if (holder) {
                    if (HINT) bulk_row_hint(ring + (s * GR + k) * 512, src, 512, bar0 + s * 8, (c >> 31) ? pol_keep : pol_cold);
                    else bulk_row(ring + (s * GR + k) * 512, src, 512, bar0 + s * 8);
                }
            } else {
                const unsigned hot = (__ballot_sync(~0u, (c >> 31) != 0) >> (sub * GR)) & ((1u << GR) - 1u);
#pragma unroll
                for (int kk = 0; kk < GR; ++kk) {
                    if ((hot >> kk) & 1u) {
                        const unsigned ck = __shfl_sync(~0u, c, sub * GR + kk);
                        cp_async16_hint(ring + (s * GR + kk) * 512 + lane * 16, xl + (size_t)(ck & ID_MASK) * 512, pol_keep);
                    }
                }
                lane_slots = (lane_slots & ~(1u << s)) | (hot ? 1u << s : 0u);
                if (lane == 0) mbar_expect(bar0 + s * 8, (GR - __popc(hot)) * 512);
                __syncwarp();
                if (holder && !(c >> 31)) bulk_row_hint(ring + (s * GR + k) * 512, src, 512, bar0 + s * 8, pol_cold);
            }
        }
        if (MODE == 4) asm volatile("cp.async.commit_group;" ::: "memory");
        if (g >= LAG) {
            const int gc = g - LAG;
            const int s = gc % NG;
            if (MODE == 4) asm volatile("cp.async.wait_group %0;" ::"n"(LAG) : "memory");
            mbar_wait(bar0 + s * 8, (gc / NG) & 1);
            const unsigned base = ring + s * GR * 512 + lane * 16;
#pragma unroll
            for (int k = 0; k < GR; ++k) {
                const float4 v = lds128(base + k * 512);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
        }
    }
    *reinterpret_cast<float4 *>(out + chunk * 128 + lane * 4) = acc;
}

// ---- mode 3 --------------------------------------------------------------------------------------
template <int RING, int GRP, int W>
__global__ void __launch_bounds__(W * 32) k_ldgsts(const float *__restrict__ x, const unsigned *__restrict__ idx,
                                                   float *out, long long E, int T) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long chunk = (long long)blockIdx.x * W + wib;
    const long long a = chunk * T;
    if (a >= E) return;
    const unsigned ring = (unsigned)__cvta_generic_to_shared(smem) + wib * (RING * 512) + lane * 16;
    const int cnt = (int)((E - a) < T ? (E - a) : T);
    const int ngroups = cnt / GRP;
    constexpr int LAG = RING / GRP - 1, GPB = 32 / GRP, RG = RING / GRP;
    const char *xl = reinterpret_cast<const char *>(x) + lane * 16;
    float4 acc = make_float4(0, 0, 0, 0);
    unsigned c = __ldcs(idx + a + lane);
#pragma unroll 1
    for (int g = 0; g < ngroups + LAG; ++g) {
        if (g < ngroups) {
            const int sub = g % GPB;
            if (sub == 0 && g > 0) c = __ldcs(idx + a + g * GRP + lane);
            const unsigned ga = ring + (g % RG) * (GRP * 512);
#pragma unroll
            for (int k = 0; k < GRP; ++k) {
                const unsigned ck = __shfl_sync(~0u, c, sub * GRP + k);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ga + k * 512), "l"(xl + (size_t)(ck & ID_MASK) * 512)
                             : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (g >= LAG) {
            asm volatile("cp.async.wait_group %0;" ::"n"(LAG) : "memory");
            const unsigned ga = ring + ((g - LAG) % RG) * (GRP * 512);
#pragma unroll
            for (int k = 0; k < GRP; ++k) {
                const float4 v = lds128(ga + k * 512);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
        }
    }
    *reinterpret_cast<float4 *>(out + chunk * 128 + lane * 4) = acc;
}

__global__ void fill_x(float *x, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i >> 7;
        x[i] = (float)((row * 7 + (i & 127)) % 1021) * 0.001f;
    }
}
__device__ __host__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z ^= z >> 31; z *= 0xBF58476D1CE4E5B9ull; z ^= z >> 29; z *= 0x94D049BB133111EBull; z ^= z >> 32;
    return z;
}
// dist 2: rank r ~ Cat(w) by the inverse of the normalised cumulative weights, id = perm[r], bit 31 for r < hot_k
__global__ void fill_idx_pow(unsigned *idx, long long E, unsigned N, const double *cdf, const unsigned *perm,
                             unsigned hot_k) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
        const double u = (double)(mix64((unsigned long long)i * 0x9E3779B97F4A7C15ull + 0x1234567ull) >> 11) *
                         (1.0 / 9007199254740992.0);
        unsigned lo = 0, hi = N - 1;  // first r with cdf[r] > u
        while (lo < hi) {
            const unsigned mid = (lo + hi) >> 1;
            if (cdf[mid] > u) hi = mid;
            else lo = mid + 1;
        }
        idx[i] = perm[lo] | (lo < hot_k ? 0x80000000u : 0u);
    }
}
__global__ void fill_idx(unsigned *idx, long long E, unsigned N, int dist) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long z = mix64((unsigned long long)i * 0x9E3779B97F4A7C15ull + 0x1234567ull);
        double u = (double)(z >> 11) * (1.0 / 9007199254740992.0);
        if (dist == 1) u = u * u * u * u;  // skewed: a quarter of the draws hit the first 0.4 % of the rows
        unsigned r = (unsigned)(u * N);
        if (r >= N) r = N - 1;
        if (dist == 1) r = (unsigned)(((unsigned long long)r * 2654435761ull) % N);  // scatter the hot rows
        idx[i] = r;
    }
}

template <typename F>
static float time_ms(F launch, int reps) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    launch();
    launch();
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    for (int i = 0; i < reps; ++i) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms / reps;
}

static double checksum(const float *d_out, long long n) {
    std::vector<float> h(n);
    CK(cudaMemcpy(h.data(), d_out, n * 4, cudaMemcpyDeviceToHost));
    double s = 0;
    for (long long i = 0; i < n; ++i) s += h[i];
    return s;
}

int main(int argc, char **argv) {
    const long long N = argc > 1 ? atoll(argv[1]) : 10000000;
    long long E = argc > 2 ? atoll(argv[2]) : 100000000;
    const int dist = argc > 3 ? atoi(argv[3]) : 0;
    const int T = argc > 4 ? atoi(argv[4]) : 2048;
    const long long hot_k = argc > 5 ? atoll(argv[5]) : 65536;
    if (N < 1 || N > 0x7fffffffLL || T < 32 || T % 32 != 0 || E < T || dist < 0 || dist > 2 || hot_k < 0) {
        printf("usage: gather_probe N E dist(0|1|2) [T (multiple of 32)] [hot_k]\n");
        return 1;
    }
    E = E / T * T;
    float *x, *out;
    unsigned *idx;
    CK(cudaMalloc(&x, N * 512));
    CK(cudaMalloc(&idx, E * 4));
    const long long chunks = E / T;
    CK(cudaMalloc(&out, chunks * 512));
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    fill_x<<<sms * 8, 256>>>(x, N * 128);
    double hot_share = 0;
    if (dist == 2) {
        std::vector<double> cdf(N);
        double s = 0;
        for (long long i = 0; i < N; ++i) cdf[i] = (s += pow((double)(i + 1), -0.8));
        const long long k = hot_k < N ? hot_k : N;
        hot_share = k > 0 ? cdf[k - 1] / s : 0.0;
        for (long long i = 0; i < N; ++i) cdf[i] /= s;
        std::vector<unsigned> perm(N);
        for (long long i = 0; i < N; ++i) perm[i] = (unsigned)i;
        for (long long i = N - 1; i > 0; --i) std::swap(perm[i], perm[mix64(0xC0FFEEull + i) % (i + 1)]);
        double *d_cdf;
        unsigned *d_perm;
        CK(cudaMalloc(&d_cdf, N * 8));
        CK(cudaMalloc(&d_perm, N * 4));
        CK(cudaMemcpy(d_cdf, cdf.data(), N * 8, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_perm, perm.data(), N * 4, cudaMemcpyHostToDevice));
        fill_idx_pow<<<sms * 8, 256>>>(idx, E, (unsigned)N, d_cdf, d_perm, (unsigned)(hot_k < N ? hot_k : N));
        CK(cudaDeviceSynchronize());
        CK(cudaFree(d_cdf));
        CK(cudaFree(d_perm));
    } else {
        fill_idx<<<sms * 8, 256>>>(idx, E, (unsigned)N, dist);
    }
    CK(cudaDeviceSynchronize());
    const double gb = (double)E * 512 / 1e9;
    printf("N=%lld E=%lld dist=%d T=%d hot_k=%lld (expected share of gathers %.3f) gather bytes %.2f GB; "
           "rate in G rows/s = E / time\n", N, E, dist, T, dist == 2 ? hot_k : 0LL, hot_share, gb);

    double ref = 0;
    auto report = [&](const char *label, float ms, double cs) {
        printf("%s : %8.3f ms  %7.1f GB/s  %6.2f G rows/s  checksum %.6e %s\n", label, ms, gb / ms * 1e3,
               (double)E / ms * 1e-6, cs, fabs(cs - ref) <= 1e-6 * fabs(ref) ? "OK" : "MISMATCH");
    };
    // mode 0
    {
        const int wpb = 8;
        const unsigned grid = (unsigned)((chunks + wpb - 1) / wpb);
        float ms = time_ms([&] { k_ldg<<<grid, wpb * 32>>>(x, idx, out, E, T); }, 5);
        CK(cudaGetLastError());
        ref = checksum(out, chunks * 128);
        report("mode0 LDG.128 x8        ", ms, ref);
    }
    // mode 3: product geometry (16-slot ring, groups of 4, 14 warps x 2 CTAs) and a deeper one
    {
        constexpr int W = 14;
        CK(cudaFuncSetAttribute(k_ldgsts<16, 4, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, W * 16 * 512));
        const unsigned grid = (unsigned)((chunks + W - 1) / W);
        float ms = time_ms([&] { k_ldgsts<16, 4, W><<<grid, W * 32, W * 16 * 512>>>(x, idx, out, E, T); }, 5);
        CK(cudaGetLastError());
        report("mode3 LDGSTS r16 g4 w14 ", ms, checksum(out, chunks * 128));
    }
    {
        constexpr int W = 7;
        CK(cudaFuncSetAttribute(k_ldgsts<32, 8, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, W * 32 * 512));
        const unsigned grid = (unsigned)((chunks + W - 1) / W);
        float ms = time_ms([&] { k_ldgsts<32, 8, W><<<grid, W * 32, W * 32 * 512>>>(x, idx, out, E, T); }, 5);
        CK(cudaGetLastError());
        report("mode3 LDGSTS r32 g8 w7  ", ms, checksum(out, chunks * 128));
    }
#define RUN_TMA(MODE, NG, GR, W, LABEL, ...)                                                                    \
    {                                                                                                               \
        auto kern = k_tma<MODE, NG, GR, W, ##__VA_ARGS__>;                                                          \
        const int smem = W * NG * GR * 512;                                                                         \
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));                          \
        const unsigned grid = (unsigned)((chunks + W - 1) / W);                                                     \
        CK(cudaMemset(out, 0, chunks * 512));                                                                       \
        float ms = time_ms([&] { kern<<<grid, W * 32, smem>>>(x, idx, out, E, T); }, 5);                        \
        cudaError_t e = cudaDeviceSynchronize();                                                                    \
        if (e != cudaSuccess) {                                                                                     \
            printf("%s : FAILED %s\n", LABEL, cudaGetErrorString(e));                                               \
            return 3;                                                                                               \
        }                                                                                                           \
        report(LABEL, ms, checksum(out, chunks * 128));                                                             \
    }
    // bulk copy per row: smem per warp = NG*GR*512
    RUN_TMA(1, 4, 8, 7, "mode1 bulk  ng4 gr8 w7  ");    // 16 KB/warp, 112 KB/CTA x2
    RUN_TMA(1, 4, 4, 14, "mode1 bulk  ng4 gr4 w14 ");   // 8 KB/warp
    RUN_TMA(1, 8, 4, 7, "mode1 bulk  ng8 gr4 w7  ");
    RUN_TMA(1, 4, 8, 4, "mode1 bulk  ng4 gr8 w4  ");    // 64 KB/CTA x3
    RUN_TMA(2, 4, 8, 7, "mode2 lane  ng4 gr8 w7  ");
    RUN_TMA(2, 4, 4, 14, "mode2 lane  ng4 gr4 w14 ");
    RUN_TMA(2, 3, 8, 9, "mode2 lane  ng3 gr8 w9  ");    // spmm_v5 geometry 2
    // L2 hints and the hybrid issue: bit-31 rows (dist 2 only) evict_last, the rest evict_first
    RUN_TMA(2, 4, 4, 14, "mode2 hint  ng4 gr4 w14 ", true);
    RUN_TMA(2, 3, 8, 9, "mode2 hint  ng3 gr8 w9  ", true);
    RUN_TMA(4, 4, 4, 14, "mode4 hyb   ng4 gr4 w14 ");
    RUN_TMA(4, 3, 8, 9, "mode4 hyb   ng3 gr8 w9  ");
    return 0;
}
