// walk.cu -- random walks on the src-keyed CSR: random_walk, node2vec_walk and node2vec_walk_plus
// (reference pgl/sampling/walk.py:23-183, graph_kernel.pyx:142-224).  One walker per thread; every walker runs its whole
// walk in one launch.
//
// The rule (include/pglb.h).  Walker i starts at nodes[i]; a step from cur picks one of cur's successor slots
// (adj_src_index: cols[indptr[cur] .. indptr[cur + 1])); a walk ends early exactly when cur has no successors.
//   - Every draw is Philox4x32-10(counter = (i lo32, i hi32, step, trial), key = (seed lo32, seed hi32)), so a walk is a
//     pure function of (graph, start, seed, walker index), whatever the launch geometry.
//   - A uniform slot is mulhi64(r64, deg), r64 = (word1 << 32) | word0.
//   - node2vec (KnightKing, SOSP'19: rejection sampling): the candidate of trial k is the uniform slot of trial k; it is
//     accepted iff word2 < thr[class], thr = floor(w / w_max * 2^32) computed once on the host from the weights
//     w = 1/p (return: candidate == prev), 1 (near: candidate is a successor of prev; node2vec_plus: of any earlier node
//     of the walk), 1/q (far).  After cap = max(WALK_TRIALS, deg) rejected trials the step is drawn exactly: an inverse
//     CDF over the row in slot order, in float64, with the uniform of trial cap.  No float arithmetic decides a trial, and
//     the fallback's sums run in a fixed order, so pglb_walk_host replays the device bit for bit.
//   - The first step of a node2vec walk has no prev: every weight is 1/q, so it is the uniform slot of trial 0, the
//     same draw as a random_walk step.
// walk_step is the only statement of one step; the kernels and pglb_walk_host all call walk_one, which calls it.
//
// Metapath walks (pglb_metapath_walk; the reference's examples/metapath2vec metapath_randomwalk): step t follows
// relation metapath[t % m], each relation its own src-keyed CSR, and is walk_uniform's step on that relation's row
// with the draw of (walker, t, trial 0).  With m = 1 a metapath walk is therefore a random_walk bit for bit.
//
// Membership ("near") is a binary search in the row-sorted copy of the successor columns (`sorted`: same indptr, each
// row ascending by id).  node2vec: one search in prev's row per trial, O(log deg(prev)).  node2vec_plus: one search in
// the row of every earlier node, O(t log d) per trial at step t -- the walk's own output row is its history.
#include <math.h>

#include "common.cuh"

namespace pglb {

// A node2vec step takes the exact fallback after max(WALK_TRIALS, deg) rejected trials: by then rejection has cost as
// much as the scan, so no step costs more than O(deg log d), and a hub row (where a scan is expensive) practically never
// reaches it.
constexpr int WALK_TRIALS = 16;
enum { WALK_UNIFORM = 0, WALK_NODE2VEC = 1, WALK_NODE2VEC_PLUS = 2 };

struct WalkRule {
    uint64_t seed;
    uint64_t thr[3];  // class c (0 return, 1 near, 2 far) accepted iff word2 < thr[c]; thr[c] in [0, 2^32]
    double w[3];      // 1/p, 1, 1/q: the fallback's weights
    // selects instead of a dynamic index, which would put the rule in local memory
    __host__ __device__ __forceinline__ uint64_t thr_of(int c) const {
        return c == 0 ? thr[0] : c == 1 ? thr[1] : thr[2];
    }
    __host__ __device__ __forceinline__ double w_of(int c) const { return c == 0 ? w[0] : c == 1 ? w[1] : w[2]; }
};

struct WalkStats {
    unsigned long long trials;     // candidate draws
    unsigned long long fallbacks;  // steps that took the exact fallback
};

// p and q as the entries check them: positive, finite, with finite reciprocals (NaN fails)
inline bool walk_pq_ok(double p, double q) {
    return p > 0.0 && q > 0.0 && isfinite(p) && isfinite(q) && isfinite(1.0 / p) && isfinite(1.0 / q);
}

inline WalkRule walk_rule_of(double p, double q, uint64_t seed) {
    WalkRule r;
    r.seed = seed;
    r.w[0] = 1.0 / p;
    r.w[1] = 1.0;
    r.w[2] = 1.0 / q;
    const double wmax = fmax(r.w[0], fmax(r.w[1], r.w[2]));
    for (int c = 0; c < 3; ++c) r.thr[c] = (uint64_t)floor(r.w[c] / wmax * 4294967296.0);
    return r;
}

__host__ __device__ __forceinline__ int64_t walk_ld(const int64_t *p) {
#ifdef __CUDA_ARCH__
    return __ldg(reinterpret_cast<const long long *>(p));
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ uint64_t walk_mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

__host__ __device__ __forceinline__ uint4 walk_draw(uint64_t seed, uint64_t walker, uint32_t step, uint32_t trial) {
    return philox4x32_10(make_uint4((uint32_t)walker, (uint32_t)(walker >> 32), step, trial), (uint32_t)seed,
                         (uint32_t)(seed >> 32));
}

__host__ __device__ __forceinline__ uint64_t walk_r64(uint4 d) { return ((uint64_t)d.y << 32) | d.x; }

// is x in u's row of the row-sorted columns?
__host__ __device__ __forceinline__ bool walk_row_has(const int64_t *indptr, const int64_t *sorted, int64_t u,
                                                      int64_t x) {
    int64_t lo = walk_ld(indptr + u);
    const int64_t end = walk_ld(indptr + u + 1);
    int64_t hi = end;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (walk_ld(sorted + mid) < x) lo = mid + 1;
        else hi = mid;
    }
    return lo < end && walk_ld(sorted + lo) == x;
}

// class of candidate x at step t (t >= 1): 0 return, 1 near, 2 far.  hist[k] = v_k of this walk, k <= t.
template <int MODE>
__host__ __device__ __forceinline__ int walk_class(const int64_t *indptr, const int64_t *sorted, const int64_t *hist,
                                                   uint32_t t, int64_t prev, int64_t x) {
    if (x == prev) return 0;
    if constexpr (MODE == WALK_NODE2VEC) {
        return walk_row_has(indptr, sorted, prev, x) ? 1 : 2;
    } else {
        for (uint32_t k = 0; k < t; ++k)
            if (walk_row_has(indptr, sorted, hist[k], x)) return 1;
        return 2;
    }
}

// the uniform slot of trial 0: a random_walk step, and the first step of a node2vec walk
__host__ __device__ __forceinline__ int64_t walk_uniform(uint64_t seed, const int64_t *cols, uint32_t t,
                                                         uint64_t walker, int64_t b, int64_t deg, WalkStats &st) {
    st.trials += 1;
    return walk_ld(cols + b + (int64_t)walk_mulhi64(walk_r64(walk_draw(seed, walker, t, 0)), (uint64_t)deg));
}

// Step t of walker `walker` from the row [b, b + deg) (deg > 0) of cur = hist[t], prev = hist[t - 1]: the next node.
template <int MODE>
__host__ __device__ __forceinline__ int64_t walk_step(const WalkRule &r, const int64_t *indptr, const int64_t *cols,
                                                      const int64_t *sorted, const int64_t *hist, uint32_t t,
                                                      uint64_t walker, int64_t b, int64_t deg, int64_t prev,
                                                      WalkStats &st) {
    if constexpr (MODE == WALK_UNIFORM) return walk_uniform(r.seed, cols, t, walker, b, deg, st);
    if (t == 0) return walk_uniform(r.seed, cols, t, walker, b, deg, st);
    const int64_t cap = deg > WALK_TRIALS ? deg : WALK_TRIALS;
    for (int64_t k = 0; k < cap; ++k) {
        const uint4 d = walk_draw(r.seed, walker, t, (uint32_t)k);
        const int64_t x = walk_ld(cols + b + (int64_t)walk_mulhi64(walk_r64(d), (uint64_t)deg));
        st.trials += 1;
        if ((uint64_t)d.z < r.thr_of(walk_class<MODE>(indptr, sorted, hist, t, prev, x))) return x;
    }
    // exact fallback: P(slot s) = w(s) / W over the row, in slot order
    st.fallbacks += 1;
    double W = 0.0;
    for (int64_t s = 0; s < deg; ++s)
        W += r.w_of(walk_class<MODE>(indptr, sorted, hist, t, prev, walk_ld(cols + b + s)));
    const double u = (double)(walk_r64(walk_draw(r.seed, walker, t, (uint32_t)cap)) >> 11) * 0x1p-53;
    const double target = u * W;
    double acc = 0.0;
    int64_t x = -1;
    for (int64_t s = 0; s < deg; ++s) {
        x = walk_ld(cols + b + s);
        acc += r.w_of(walk_class<MODE>(indptr, sorted, hist, t, prev, x));
        if (target < acc) break;
    }
    return x;
}

// The whole walk of one walker into out[0, L): start, then up to `steps` steps, then -1 padding.  A start outside
// [0, num_nodes) gives a row of -1 (the Python layer refuses such starts before any launch).
template <int MODE>
__host__ __device__ __forceinline__ void walk_one(const WalkRule &r, const int64_t *indptr, const int64_t *cols,
                                                  const int64_t *sorted, int64_t num_nodes, int64_t start,
                                                  uint64_t walker, int64_t steps, int64_t *out, int64_t L,
                                                  WalkStats &st) {
    int64_t k = 0;
    if (start >= 0 && start < num_nodes) {
        int64_t cur = start, prev = -1;
        out[k++] = cur;
        for (int64_t t = 0; t < steps; ++t) {
            const int64_t b = walk_ld(indptr + cur);
            const int64_t deg = walk_ld(indptr + cur + 1) - b;
            if (deg == 0) break;
            const int64_t nxt = walk_step<MODE>(r, indptr, cols, sorted, out, (uint32_t)t, walker, b, deg, prev, st);
            out[k++] = nxt;
            prev = cur;
            cur = nxt;
        }
    }
    for (; k < L; ++k) out[k] = -1;
}

template <int MODE>
__global__ void __launch_bounds__(256) walk_kernel(const int64_t *__restrict__ indptr,
                                                   const int64_t *__restrict__ cols,
                                                   const int64_t *__restrict__ sorted, int64_t num_nodes,
                                                   const int64_t *__restrict__ nodes, int64_t n, int64_t steps,
                                                   WalkRule r, int64_t *__restrict__ out, int64_t L,
                                                   unsigned long long *__restrict__ stats) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    WalkStats st{0, 0};
    if (i < n) walk_one<MODE>(r, indptr, cols, sorted, num_nodes, __ldg(reinterpret_cast<const long long *>(nodes + i)),
                              (uint64_t)i, steps, out + i * L, L, st);
    if (stats) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            st.trials += __shfl_down_sync(0xffffffffu, st.trials, o);
            st.fallbacks += __shfl_down_sync(0xffffffffu, st.fallbacks, o);
        }
        if ((threadIdx.x & 31) == 0) {
            atomicAdd(stats, st.trials);
            atomicAdd(stats + 1, st.fallbacks);
        }
    }
}

// the checks every walk entry makes before anything else
inline int walk_check(const char *name, const int64_t *indptr, const int64_t *cols, const int64_t *sorted,
                      int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t max_depth, const int64_t *out,
                      bool node2vec, double p, double q) {
    PGLB_CHECK_ARG(n >= 0 && num_nodes >= 0, PGLB_EINVAL, "%s: negative size", name);
    PGLB_CHECK_ARG(max_depth >= 1 && max_depth < INT32_MAX, PGLB_EINVAL, "%s: max_depth must lie in [1, 2^31 - 1)",
                   name);
    if (node2vec) PGLB_CHECK_ARG(walk_pq_ok(p, q), PGLB_EINVAL, "%s: p and q must be positive and finite", name);
    PGLB_CHECK_ARG(n == 0 || (indptr && cols && nodes && out && (sorted || !node2vec)), PGLB_EINVAL,
                   "%s: NULL pointer", name);
    return PGLB_OK;
}

template <int MODE>
int walk_launch(const char *name, const int64_t *indptr, const int64_t *cols, const int64_t *sorted,
                int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t steps, const WalkRule &r, int64_t *out,
                int64_t L, unsigned long long *stats, void *stream) {
    const unsigned grid = (unsigned)((n + 255) / 256);
    walk_kernel<MODE><<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(indptr, cols, sorted, num_nodes, nodes,
                                                                                 n, steps, r, out, L, stats);
    PGLB_LAUNCH_CHECK(name);
    return PGLB_OK;
}

// A metapath's relations travel into the kernel by value, as one __grid_constant__ parameter of about 1 KB: a step
// reads its (indptr, cols) pair from the parameter bank with a dynamic index (a constant-memory load, no local copy),
// so it costs what a random_walk step costs.
constexpr int METAPATH_MAX = 64;

struct MetapathRule {
    uint64_t seed;
    int m;  // 1 <= m <= METAPATH_MAX
    const int64_t *indptr[METAPATH_MAX];
    const int64_t *cols[METAPATH_MAX];
};

// The whole metapath walk of one walker into out[0, L): start, then up to L - 1 steps, then -1 padding.  A start
// outside [0, num_nodes) gives a row of -1, as in walk_one.
__host__ __device__ __forceinline__ void metapath_one(const MetapathRule &r, int64_t num_nodes, int64_t start,
                                                      uint64_t walker, int64_t *out, int64_t L) {
    WalkStats st{0, 0};  // walk_uniform counts its draws; nothing reads the count here
    int64_t k = 0;
    if (start >= 0 && start < num_nodes) {
        int64_t cur = start;
        out[k++] = cur;
        int pos = 0;  // t % m, kept as a wrapping counter instead of a division
        for (int64_t t = 0; t + 1 < L; ++t) {
            const int64_t *indptr = r.indptr[pos];
            const int64_t b = walk_ld(indptr + cur);
            const int64_t deg = walk_ld(indptr + cur + 1) - b;
            if (deg == 0) break;
            cur = walk_uniform(r.seed, r.cols[pos], (uint32_t)t, walker, b, deg, st);
            out[k++] = cur;
            if (++pos == r.m) pos = 0;
        }
    }
    for (; k < L; ++k) out[k] = -1;
}

__global__ void __launch_bounds__(256) metapath_walk_kernel(const __grid_constant__ MetapathRule r, int64_t num_nodes,
                                                            const int64_t *__restrict__ nodes, int64_t n,
                                                            int64_t *__restrict__ out, int64_t L) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        metapath_one(r, num_nodes, __ldg(reinterpret_cast<const long long *>(nodes + i)), (uint64_t)i, out + i * L, L);
}

// the checks of both metapath entries, before anything else; walk_check's on every relation
inline int metapath_check(const char *name, const int64_t *const *indptrs, const int64_t *const *cols, int m,
                          int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t walk_length, const int64_t *out) {
    PGLB_CHECK_ARG(m >= 1 && m <= METAPATH_MAX, PGLB_EINVAL, "%s: m must lie in [1, %d], got %d", name, METAPATH_MAX,
                   m);
    PGLB_CHECK_ARG(walk_length >= 1 && walk_length < INT32_MAX, PGLB_EINVAL,
                   "%s: walk_length must lie in [1, 2^31 - 1)", name);
    PGLB_CHECK_ARG(n <= 0 || (indptrs && cols), PGLB_EINVAL, "%s: NULL pointer", name);
    for (int k = 0; k < m; ++k)
        if (const int rc = walk_check(name, n > 0 ? indptrs[k] : nullptr, n > 0 ? cols[k] : nullptr, nullptr,
                                      num_nodes, nodes, n, walk_length, out, false, 1, 1))
            return rc;
    return PGLB_OK;
}

inline MetapathRule metapath_rule_of(const int64_t *const *indptrs, const int64_t *const *cols, int m,
                                     uint64_t seed) {
    MetapathRule r{};
    r.seed = seed;
    r.m = m;
    for (int k = 0; k < m; ++k) {
        r.indptr[k] = indptrs[k];
        r.cols[k] = cols[k];
    }
    return r;
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_random_walk(const int64_t *indptr, const int64_t *cols, int64_t num_nodes, const int64_t *nodes,
                                int64_t n, int64_t max_depth, uint64_t seed, int64_t *out, void *stream) {
    const char *name = "pglb_random_walk";
    if (const int rc = walk_check(name, indptr, cols, nullptr, num_nodes, nodes, n, max_depth, out, false, 1, 1))
        return rc;
    if (n == 0) return PGLB_OK;
    const WalkRule r = walk_rule_of(1.0, 1.0, seed);
    return walk_launch<WALK_UNIFORM>("walk_kernel<uniform>", indptr, cols, nullptr, num_nodes, nodes, n, max_depth - 1,
                                     r, out, max_depth, nullptr, stream);
}

extern "C" int pglb_node2vec_walk(const int64_t *indptr, const int64_t *cols, const int64_t *sorted_cols,
                                  int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t max_depth, double p,
                                  double q, int plus, uint64_t seed, int64_t *out, uint64_t *stats, void *stream) {
    const char *name = "pglb_node2vec_walk";
    if (const int rc = walk_check(name, indptr, cols, sorted_cols, num_nodes, nodes, n, max_depth, out, true, p, q))
        return rc;
    if (n == 0) return PGLB_OK;
    const WalkRule r = walk_rule_of(p, q, seed);
    unsigned long long *st = reinterpret_cast<unsigned long long *>(stats);
    if (plus)
        return walk_launch<WALK_NODE2VEC_PLUS>("walk_kernel<node2vec_plus>", indptr, cols, sorted_cols, num_nodes,
                                               nodes, n, max_depth, r, out, max_depth + 1, st, stream);
    return walk_launch<WALK_NODE2VEC>("walk_kernel<node2vec>", indptr, cols, sorted_cols, num_nodes, nodes, n,
                                      max_depth, r, out, max_depth + 1, st, stream);
}

// The same walks on the host, one walker after another, through the kernels' walk_one (include/pglb.h).
extern "C" int pglb_walk_host(const int64_t *indptr, const int64_t *cols, const int64_t *sorted_cols,
                              int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t max_depth, double p,
                              double q, int mode, uint64_t seed, int64_t *out, uint64_t *stats) {
    const char *name = "pglb_walk_host";
    PGLB_CHECK_ARG(mode == WALK_UNIFORM || mode == WALK_NODE2VEC || mode == WALK_NODE2VEC_PLUS, PGLB_EINVAL,
                   "%s: unknown mode %d", name, mode);
    const bool n2v = mode != WALK_UNIFORM;
    if (const int rc = walk_check(name, indptr, cols, sorted_cols, num_nodes, nodes, n, max_depth, out, n2v, p, q))
        return rc;
    const WalkRule r = n2v ? walk_rule_of(p, q, seed) : walk_rule_of(1.0, 1.0, seed);
    const int64_t steps = n2v ? max_depth : max_depth - 1, L = n2v ? max_depth + 1 : max_depth;
    WalkStats st{0, 0};
    for (int64_t i = 0; i < n; ++i) {
        if (mode == WALK_UNIFORM)
            walk_one<WALK_UNIFORM>(r, indptr, cols, sorted_cols, num_nodes, nodes[i], (uint64_t)i, steps, out + i * L,
                                   L, st);
        else if (mode == WALK_NODE2VEC)
            walk_one<WALK_NODE2VEC>(r, indptr, cols, sorted_cols, num_nodes, nodes[i], (uint64_t)i, steps,
                                    out + i * L, L, st);
        else
            walk_one<WALK_NODE2VEC_PLUS>(r, indptr, cols, sorted_cols, num_nodes, nodes[i], (uint64_t)i, steps,
                                         out + i * L, L, st);
    }
    if (stats) {
        stats[0] = st.trials;
        stats[1] = st.fallbacks;
    }
    return PGLB_OK;
}

extern "C" int pglb_metapath_walk(const int64_t *const *indptrs, const int64_t *const *cols, int m, int64_t num_nodes,
                                  const int64_t *nodes, int64_t n, int64_t walk_length, uint64_t seed, int64_t *out,
                                  void *stream) {
    const char *name = "pglb_metapath_walk";
    if (const int rc = metapath_check(name, indptrs, cols, m, num_nodes, nodes, n, walk_length, out)) return rc;
    if (n == 0) return PGLB_OK;
    const MetapathRule r = metapath_rule_of(indptrs, cols, m, seed);
    const unsigned grid = (unsigned)((n + 255) / 256);
    metapath_walk_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(r, num_nodes, nodes, n, out,
                                                                                    walk_length);
    PGLB_LAUNCH_CHECK("metapath_walk_kernel");
    return PGLB_OK;
}

// The same walks on the host, one walker after another, through the kernel's metapath_one (include/pglb.h).
extern "C" int pglb_metapath_walk_host(const int64_t *const *indptrs, const int64_t *const *cols, int m,
                                       int64_t num_nodes, const int64_t *nodes, int64_t n, int64_t walk_length,
                                       uint64_t seed, int64_t *out) {
    const char *name = "pglb_metapath_walk_host";
    if (const int rc = metapath_check(name, indptrs, cols, m, num_nodes, nodes, n, walk_length, out)) return rc;
    if (n == 0) return PGLB_OK;
    const MetapathRule r = metapath_rule_of(indptrs, cols, m, seed);
    for (int64_t i = 0; i < n; ++i)
        metapath_one(r, num_nodes, nodes[i], (uint64_t)i, out + i * walk_length, walk_length);
    return PGLB_OK;
}
