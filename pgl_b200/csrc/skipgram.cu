// skipgram.cu -- skip-gram training pairs from a batch of padded walks, and alias-table sampling (the reference's
// graph_kernel.pyx:343-365 skip_gram_gen_pair and examples/metapath2vec/datasets/sampling.py:133-146 alias_sample).
//
// The rules (include/pglb.h).
//   - Walk b is row b of walks [B, L]; its length n_b is the index of the first entry < 0, or L.
//   - Centre i < n_b draws its window w = 1 + mulhi32(word0, win_size) from Philox4x32-10(counter = (b lo32, b hi32,
//     i, PGLB_SKIPGRAM_TAG), key = (seed lo32, seed hi32)), and emits (walk[i], walk[j]) for every j in
//     [max(0, i - w), min(n_b - 1, i + w)] ascending with walk[j] != walk[i].  Output order: walk, centre, j.
//   - Alias draw k: Philox4x32-10((k lo32, k hi32, 0, PGLB_ALIAS_TAG), seed); slot = mulhi64(word1:word0, n);
//     u = (word2:word3 >> 11) 2^-53; the draw is slot if u < alias[slot], else events[slot].
// skipgram_window / skipgram_emits / alias_draw are the only statements of these rules: the kernels and the host twins
// (pglb_skipgram_host, pglb_alias_sample_host) all call them.
//
// Pairs: count -> scan -> fill.  A warp owns a walk in both kernels and enumerates its (centre, j) candidates in the
// same order, so the fill writes exactly the slots the count reserved.  With span = 2 win_size + 1 <= 32, one pass of
// the warp covers floor(32 / span) whole centres (lane = centre-in-pass * span + offset); wider windows take one centre
// at a time in 32-position chunks.  Every pass is one ballot: a kept lane's slot is the walk's cursor plus the kept
// lanes below it, so a pass stores one contiguous run of pairs.  The walk row is read through L1.
#include "common.cuh"

namespace pglb {

constexpr int SG_THREADS = 256;
constexpr int SG_WARPS = SG_THREADS / 32;

__host__ __device__ __forceinline__ int64_t sg_ld(const int64_t *p) {
#ifdef __CUDA_ARCH__
    return __ldg(reinterpret_cast<const long long *>(p));
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ double sg_ldf(const double *p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ uint64_t sg_mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// the window of centre i of walk b: 1 + mulhi32(word0, win_size), in [1, win_size]
__host__ __device__ __forceinline__ int64_t skipgram_window(uint64_t seed, uint64_t b, int64_t i, int64_t win_size) {
    const uint4 d = philox4x32_10(make_uint4((uint32_t)b, (uint32_t)(b >> 32), (uint32_t)i, PGLB_SKIPGRAM_TAG),
                                  (uint32_t)seed, (uint32_t)(seed >> 32));
    return 1 + (int64_t)(((uint64_t)d.x * (uint64_t)win_size) >> 32);
}

// does centre i (window w) of a walk of n nodes pair with position j?
__host__ __device__ __forceinline__ bool skipgram_emits(const int64_t *row, int64_t n, int64_t i, int64_t w,
                                                        int64_t j) {
    return j >= 0 && j < n && j >= i - w && j <= i + w && sg_ld(row + j) != sg_ld(row + i);
}

// alias draw k of the table (alias, events) of n entries
__host__ __device__ __forceinline__ int64_t alias_draw(const double *alias, const int64_t *events, uint64_t n,
                                                       uint64_t seed, uint64_t k) {
    const uint4 d = philox4x32_10(make_uint4((uint32_t)k, (uint32_t)(k >> 32), 0u, PGLB_ALIAS_TAG), (uint32_t)seed,
                                  (uint32_t)(seed >> 32));
    const uint64_t slot = sg_mulhi64(((uint64_t)d.y << 32) | d.x, n);
    const double u = (double)((((uint64_t)d.z << 32) | d.w) >> 11) * 0x1p-53;
    return u < sg_ldf(alias + slot) ? (int64_t)slot : sg_ld(events + slot);
}

// The pairs of one walk by one warp: returns their count; WRITE stores them from src[base], pos[base] on.
template <bool WRITE>
__device__ __forceinline__ int64_t skipgram_warp(const int64_t *row, int64_t L, int64_t win_size, uint64_t seed,
                                                 uint64_t b, int64_t base, int64_t *src, int64_t *pos) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    int64_t n = L;
    for (int64_t c = 0; c < L; c += 32) {
        const unsigned neg = __ballot_sync(full, c + lane < L && sg_ld(row + c + lane) < 0);
        if (neg) {
            n = c + __ffs(neg) - 1;
            break;
        }
    }
    int64_t cur = base;
    if (2 * win_size + 1 <= 32) {
        const int span = 2 * (int)win_size + 1;
        const int per = 32 / span;  // whole centres per pass
        const int c = lane / span, off = lane % span;
        for (int64_t i0 = 0; i0 < n; i0 += per) {
            // lane q < per draws the window of centre i0 + q; lane (c, off) reads it from lane c
            const int64_t wq = lane < per && i0 + lane < n ? skipgram_window(seed, b, i0 + lane, win_size) : 0;
            const int64_t w = __shfl_sync(full, wq, c);
            const int64_t i = i0 + c;
            const int64_t j = i - win_size + off;
            const bool keep = c < per && i < n && skipgram_emits(row, n, i, w, j);
            const unsigned m = __ballot_sync(full, keep);
            if (WRITE && keep) {
                const int64_t o = cur + __popc(m & below);
                src[o] = sg_ld(row + i);
                pos[o] = sg_ld(row + j);
            }
            cur += __popc(m);
        }
    } else {
        for (int64_t i = 0; i < n; ++i) {
            const int64_t w = skipgram_window(seed, b, i, win_size);
            const int64_t lo = i - w > 0 ? i - w : 0, hi = i + w < n - 1 ? i + w : n - 1;
            const int64_t ci = sg_ld(row + i);
            for (int64_t j0 = lo; j0 <= hi; j0 += 32) {
                const int64_t j = j0 + lane;
                const bool keep = j <= hi && skipgram_emits(row, n, i, w, j);
                const unsigned m = __ballot_sync(full, keep);
                if (WRITE && keep) {
                    const int64_t o = cur + __popc(m & below);
                    src[o] = ci;
                    pos[o] = sg_ld(row + j);
                }
                cur += __popc(m);
            }
        }
    }
    return cur - base;
}

// offsets[b + 1] = pair count of walk b; offsets[0] = 0
__global__ void __launch_bounds__(SG_THREADS) skipgram_count_kernel(const int64_t *__restrict__ walks, int64_t B,
                                                                    int64_t L, int64_t win_size, uint64_t seed,
                                                                    int64_t *__restrict__ offsets) {
    if (blockIdx.x == 0 && threadIdx.x == 0) offsets[0] = 0;
    const int64_t b = (int64_t)blockIdx.x * SG_WARPS + (threadIdx.x >> 5);
    if (b >= B) return;  // warp-uniform
    const int64_t c = skipgram_warp<false>(walks + b * L, L, win_size, seed, (uint64_t)b, 0, nullptr, nullptr);
    if ((threadIdx.x & 31) == 0) offsets[b + 1] = c;
}

__global__ void __launch_bounds__(SG_THREADS) skipgram_fill_kernel(const int64_t *__restrict__ walks, int64_t B,
                                                                   int64_t L, int64_t win_size, uint64_t seed,
                                                                   const int64_t *__restrict__ offsets,
                                                                   int64_t *__restrict__ src,
                                                                   int64_t *__restrict__ pos) {
    const int64_t b = (int64_t)blockIdx.x * SG_WARPS + (threadIdx.x >> 5);
    if (b >= B) return;
    skipgram_warp<true>(walks + b * L, L, win_size, seed, (uint64_t)b, sg_ld(offsets + b), src, pos);
}

__global__ void __launch_bounds__(256) alias_sample_kernel(const double *__restrict__ alias,
                                                           const int64_t *__restrict__ events, uint64_t n,
                                                           int64_t count, uint64_t seed, int64_t *__restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride)
        out[k] = alias_draw(alias, events, n, seed, (uint64_t)k);
}

// the checks of every skip-gram entry, before anything else
inline int skipgram_check(const char *name, const int64_t *walks, int64_t B, int64_t L, int64_t win_size,
                          const int64_t *offsets) {
    PGLB_CHECK_ARG(B >= 0, PGLB_EINVAL, "%s: negative B", name);
    PGLB_CHECK_ARG(L >= 0 && L < INT32_MAX, PGLB_EINVAL, "%s: L must lie in [0, 2^31 - 1), got %lld", name,
                   (long long)L);
    PGLB_CHECK_ARG(win_size >= 1 && win_size < INT32_MAX + 1LL, PGLB_EINVAL,
                   "%s: win_size must lie in [1, 2^31), got %lld", name, (long long)win_size);
    PGLB_CHECK_ARG(B == 0 || (offsets && (walks || L == 0)), PGLB_EINVAL, "%s: NULL pointer", name);
    return PGLB_OK;
}

inline int alias_check(const char *name, const double *alias, const int64_t *events, int64_t n, int64_t count,
                       const int64_t *out) {
    PGLB_CHECK_ARG(n >= 1 && n < (1LL << 32), PGLB_EINVAL, "%s: n must lie in [1, 2^32), got %lld", name,
                   (long long)n);
    PGLB_CHECK_ARG(count >= 0, PGLB_EINVAL, "%s: negative count", name);
    PGLB_CHECK_ARG(count == 0 || (alias && events && out), PGLB_EINVAL, "%s: NULL pointer", name);
    return PGLB_OK;
}

inline unsigned sg_grid(int64_t B) { return (unsigned)((B + SG_WARPS - 1) / SG_WARPS); }

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_skipgram_count_ws(int64_t B, size_t *ws_bytes) {
    PGLB_CHECK_ARG(B >= 0 && ws_bytes, PGLB_EINVAL, "pglb_skipgram_count_ws: bad args");
    *ws_bytes = scan_i64_ws_bytes(B);
    return PGLB_OK;
}

extern "C" int pglb_skipgram_count(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed,
                                   int64_t *offsets, void *ws, size_t ws_bytes, void *stream) {
    const char *name = "pglb_skipgram_count";
    if (const int rc = skipgram_check(name, walks, B, L, win_size, offsets)) return rc;
    if (B == 0) return PGLB_OK;
    PGLB_CHECK_ARG(ws && ws_bytes >= scan_i64_ws_bytes(B), PGLB_EWORKSPACE, "%s: workspace too small", name);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    skipgram_count_kernel<<<sg_grid(B), SG_THREADS, 0, s>>>(walks, B, L, win_size, seed, offsets);
    PGLB_LAUNCH_CHECK("skipgram_count_kernel");
    return scan_i64(offsets + 1, offsets + 1, B, /*inclusive=*/1, ws, s);
}

extern "C" int pglb_skipgram_fill(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed,
                                  const int64_t *offsets, int64_t *src, int64_t *pos, void *stream) {
    const char *name = "pglb_skipgram_fill";
    if (const int rc = skipgram_check(name, walks, B, L, win_size, offsets)) return rc;
    if (B == 0 || L == 0) return PGLB_OK;
    PGLB_CHECK_ARG(src && pos, PGLB_EINVAL, "%s: NULL output", name);
    skipgram_fill_kernel<<<sg_grid(B), SG_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        walks, B, L, win_size, seed, offsets, src, pos);
    PGLB_LAUNCH_CHECK("skipgram_fill_kernel");
    return PGLB_OK;
}

// The same pairs on the host, walk after walk, through the kernels' skipgram_window / skipgram_emits.
extern "C" int pglb_skipgram_host(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed,
                                  int64_t *offsets, int64_t *src, int64_t *pos) {
    const char *name = "pglb_skipgram_host";
    if (const int rc = skipgram_check(name, walks, B, L, win_size, offsets)) return rc;
    if (B == 0) return PGLB_OK;
    offsets[0] = 0;
    int64_t o = 0;
    for (int64_t b = 0; b < B; ++b) {
        const int64_t *row = walks + b * L;
        int64_t n = 0;
        while (n < L && row[n] >= 0) ++n;
        for (int64_t i = 0; i < n; ++i) {
            const int64_t w = skipgram_window(seed, (uint64_t)b, i, win_size);
            const int64_t lo = i - w > 0 ? i - w : 0, hi = i + w < n - 1 ? i + w : n - 1;
            for (int64_t j = lo; j <= hi; ++j) {
                if (!skipgram_emits(row, n, i, w, j)) continue;
                if (src) {
                    src[o] = row[i];
                    pos[o] = row[j];
                }
                ++o;
            }
        }
        offsets[b + 1] = o;
    }
    return PGLB_OK;
}

extern "C" int pglb_alias_sample(const double *alias, const int64_t *events, int64_t n, int64_t count, uint64_t seed,
                                 int64_t *out, void *stream) {
    const char *name = "pglb_alias_sample";
    if (const int rc = alias_check(name, alias, events, n, count, out)) return rc;
    if (count == 0) return PGLB_OK;
    const int64_t want = (count + 255) / 256, cap = (int64_t)sm_count() * 64;
    const unsigned grid = (unsigned)(want < cap ? want : cap);
    alias_sample_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(alias, events, (uint64_t)n, count,
                                                                                   seed, out);
    PGLB_LAUNCH_CHECK("alias_sample_kernel");
    return PGLB_OK;
}

// The same draws on the host through the kernel's alias_draw.
extern "C" int pglb_alias_sample_host(const double *alias, const int64_t *events, int64_t n, int64_t count,
                                      uint64_t seed, int64_t *out) {
    if (const int rc = alias_check("pglb_alias_sample_host", alias, events, n, count, out)) return rc;
    for (int64_t k = 0; k < count; ++k) out[k] = alias_draw(alias, events, (uint64_t)n, seed, (uint64_t)k);
    return PGLB_OK;
}
