// sgns.cu -- the skip-gram negative-sampling loss of the reference's walk models (examples/deepwalk/model.py and
// examples/metapath2vec/model.py: SkipGramModel.forward), fused into one pass over the rows a batch touches.
//
// The rule (include/pglb.h).  For pair p with centre src[p] and targets dsts[p, 0..K] (0: the positive):
//   s[p, j] = <emb[src[p]], ctx[dsts[p, j]]>
//   loss    = ( mean_p softplus(-s[p, 0]) + mean_{p, k >= 1} softplus(s[p, k]) ) / 2
//   c[p, 0] = -sigmoid(-s[p, 0]) / (2P),  c[p, k] = sigmoid(s[p, k]) / (2PK)      (d loss / d s)
//   w[p]    = sum_j c[p, j] ctx[dsts[p, j]]                                     (d loss / d emb[src[p]], pair p's part)
// softplus(x) = max(x, 0) + log1p(exp(-|x|)) and sigmoid in the form that never divides by an overflowed exp, so
// saturated logits give finite values.
//
// Work layout.  A group of G lanes owns a pair.  It loads the centre row once into registers (NV chunks of VEC floats
// per lane, element (s G + lane) VEC + v), then walks the 1 + K context rows SGNS_U at a time: the U rows' loads are
// all issued before the first reduction, each dot is reduced by the same xor butterfly (fixed order), and the epilogue
// turns it into a loss term and c.  The training kernel folds c_j x_j into w while row j is still in registers, so
// the rows are read from memory once and w costs no second pass.  VEC = 4 needs 16-byte rows (D % 4 == 0, aligned
// tables and ld % 4 == 0); D above the register layout's reach (512 vectorised, 256 scalar) takes the wide kernel, a
// warp per pair that re-reads each row from L1 for w.
//
// The loss is deterministic: each block adds its pairs' terms in a fixed order into one double partial, and a
// one-block launch sums the partials in index order.  The grid is capped at SGNS_MAX_BLOCKS blocks, independent of
// the device, so the pair-to-block assignment depends on P only.
#include "common.cuh"

namespace pglb {

constexpr int SGNS_THREADS = 256;
constexpr int SGNS_MAX_BLOCKS = 4096;
constexpr int SGNS_U = 4;

struct SgnsArgs {
    const float *emb;
    const float *ctx;
    const int64_t *src;
    const int64_t *dsts;
    float *c;
    float *w;
    double *part;
    int64_t ld_emb, ld_ctx, ldw;
    int64_t P, K, D;
};

__device__ __forceinline__ float sgns_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

__device__ __forceinline__ float sgns_sigmoid(float x) {
    const float e = expf(-fabsf(x));  // in (0, 1]: never overflows
    return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

template <int VEC>
__device__ __forceinline__ void sgns_ld(const float *p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
    } else {
        v[0] = __ldg(p);
    }
}

template <int VEC>
__device__ __forceinline__ void sgns_st(float *p, const float (&v)[VEC]) {
    if constexpr (VEC == 4)
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else
        p[0] = v[0];
}

// the pair's loss term lp + ln / K of target j's logit d, and its coefficient c
__device__ __forceinline__ float sgns_epilogue(float d, int64_t j, const SgnsArgs &a, float &lp, float &ln) {
    if (j == 0) {
        lp = sgns_softplus(-d);
        return -sgns_sigmoid(-d) / (float)(2 * a.P);
    }
    ln += sgns_softplus(d);
    return sgns_sigmoid(d) / (float)(2 * a.P * a.K);
}

// acc of every thread, summed in a fixed order, into a.part[blockIdx.x]
__device__ __forceinline__ void sgns_block_sum(double acc, double *part) {
    __shared__ double sh[SGNS_THREADS / 32];
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < SGNS_THREADS / 32; ++i) t += sh[i];
        part[blockIdx.x] = t;
    }
}

// Two resident blocks per SM (up to 128 registers per lane): with no minimum, ptxas spilled the loss-only D <= 256
// layout at 40 registers.  Every layout now compiles without spills.
template <int G, int VEC, int NV, bool TRAIN>
__global__ void __launch_bounds__(SGNS_THREADS, 2) sgns_fwd_kernel(const SgnsArgs a) {
    constexpr int GPB = SGNS_THREADS / G;
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & (G - 1);
    const int grp = threadIdx.x / G;
    const int64_t J = a.K + 1;
    double acc = 0.0;
    // the loop bounds are block-uniform, so every lane reaches every shuffle; lanes of a group past P load nothing
    for (int64_t base = (int64_t)blockIdx.x * GPB; base < a.P; base += (int64_t)gridDim.x * GPB) {
        const int64_t p = base + grp;
        const bool valid = p < a.P;
        float e[NV][VEC], w[NV][VEC];
        const float *er = a.emb + (valid ? __ldg(reinterpret_cast<const long long *>(a.src + p)) : 0) * a.ld_emb;
#pragma unroll
        for (int s = 0; s < NV; ++s) {
            const int64_t col = (int64_t)(s * G + lane) * VEC;
#pragma unroll
            for (int v = 0; v < VEC; ++v) e[s][v] = w[s][v] = 0.f;
            if (valid && col < a.D) sgns_ld<VEC>(er + col, e[s]);
        }
        float lp = 0.f, ln = 0.f;
        const int64_t *dr = a.dsts + (valid ? p : 0) * J;
        for (int64_t j0 = 0; j0 < J; j0 += SGNS_U) {
            float x[SGNS_U][NV][VEC];
#pragma unroll
            for (int u = 0; u < SGNS_U; ++u) {
                const bool ok = valid && j0 + u < J;
                const float *xr = a.ctx + (ok ? __ldg(reinterpret_cast<const long long *>(dr + j0 + u)) : 0) * a.ld_ctx;
#pragma unroll
                for (int s = 0; s < NV; ++s) {
                    const int64_t col = (int64_t)(s * G + lane) * VEC;
#pragma unroll
                    for (int v = 0; v < VEC; ++v) x[u][s][v] = 0.f;
                    if (ok && col < a.D) sgns_ld<VEC>(xr + col, x[u][s]);
                }
            }
            float d[SGNS_U];
#pragma unroll
            for (int u = 0; u < SGNS_U; ++u) {
                d[u] = 0.f;
#pragma unroll
                for (int s = 0; s < NV; ++s)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) d[u] = fmaf(e[s][v], x[u][s][v], d[u]);
            }
#pragma unroll
            for (int off = G / 2; off > 0; off >>= 1)
#pragma unroll
                for (int u = 0; u < SGNS_U; ++u) d[u] += __shfl_xor_sync(full, d[u], off);
#pragma unroll
            for (int u = 0; u < SGNS_U; ++u) {
                const int64_t j = j0 + u;
                if (j < J) {
                    const float c = sgns_epilogue(d[u], j, a, lp, ln);
                    if (TRAIN) {
                        if (valid && lane == 0) a.c[p * J + j] = c;
#pragma unroll
                        for (int s = 0; s < NV; ++s)
#pragma unroll
                            for (int v = 0; v < VEC; ++v) w[s][v] = fmaf(c, x[u][s][v], w[s][v]);
                    }
                }
            }
        }
        if (TRAIN && valid) {
#pragma unroll
            for (int s = 0; s < NV; ++s) {
                const int64_t col = (int64_t)(s * G + lane) * VEC;
                if (col < a.D) sgns_st<VEC>(a.w + p * a.ldw + col, w[s]);
            }
        }
        if (valid && lane == 0) acc += (double)lp + (double)ln / (double)a.K;
    }
    sgns_block_sum(acc, a.part);
}

// D beyond the register layouts: a warp per pair, the centre and context rows streamed in 32-column strips; w is
// accumulated in place in the output row (each column by the lane that owns it, in j order, as the kernel above).
template <bool TRAIN>
__global__ void __launch_bounds__(SGNS_THREADS) sgns_fwd_wide_kernel(const SgnsArgs a) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int64_t J = a.K + 1;
    double acc = 0.0;
    for (int64_t base = (int64_t)blockIdx.x * (SGNS_THREADS / 32); base < a.P;
         base += (int64_t)gridDim.x * (SGNS_THREADS / 32)) {
        const int64_t p = base + (threadIdx.x >> 5);
        if (p >= a.P) continue;  // warp-uniform
        const float *er = a.emb + a.src[p] * a.ld_emb;
        float *wr = a.w + p * a.ldw;
        float lp = 0.f, ln = 0.f;
        for (int64_t j = 0; j < J; ++j) {
            const float *xr = a.ctx + a.dsts[p * J + j] * a.ld_ctx;
            float d = 0.f;
            for (int64_t col = lane; col < a.D; col += 32) d = fmaf(__ldg(er + col), __ldg(xr + col), d);
            for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(full, d, off);
            const float c = sgns_epilogue(d, j, a, lp, ln);
            if (TRAIN) {
                if (lane == 0) a.c[p * J + j] = c;
                for (int64_t col = lane; col < a.D; col += 32)
                    wr[col] = j == 0 ? c * __ldg(xr + col) : fmaf(c, __ldg(xr + col), wr[col]);
            }
        }
        if (lane == 0) acc += (double)lp + (double)ln / (double)a.K;
    }
    sgns_block_sum(acc, a.part);
}

// loss = (sum of the block partials, in index order) / (2P)
__global__ void __launch_bounds__(SGNS_THREADS) sgns_loss_kernel(const double *__restrict__ part, int n, int64_t P,
                                                                 float *__restrict__ loss) {
    __shared__ double sh[SGNS_THREADS];
    double t = 0.0;
    for (int i = threadIdx.x; i < n; i += SGNS_THREADS) t += part[i];
    sh[threadIdx.x] = t;
    __syncthreads();
    for (int h = SGNS_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) sh[threadIdx.x] += sh[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = (float)(sh[0] / (2.0 * (double)P));
}

inline unsigned sgns_grid(int64_t P, int pairs_per_block) {
    const int64_t want = (P + pairs_per_block - 1) / pairs_per_block;
    return (unsigned)(want < SGNS_MAX_BLOCKS ? want : SGNS_MAX_BLOCKS);
}

// the forward kernel of layout (G, VEC, NV); returns its grid size
template <int G, int VEC, int NV>
inline unsigned sgns_launch(const SgnsArgs &a, bool train, cudaStream_t s) {
    const unsigned grid = sgns_grid(a.P, SGNS_THREADS / G);
    if (train)
        sgns_fwd_kernel<G, VEC, NV, true><<<grid, SGNS_THREADS, 0, s>>>(a);
    else
        sgns_fwd_kernel<G, VEC, NV, false><<<grid, SGNS_THREADS, 0, s>>>(a);
    return grid;
}

inline bool sgns_a16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// do the byte ranges [a, a + na) and [b, b + nb) meet?
inline bool sgns_overlap(const void *a, size_t na, const void *b, size_t nb) {
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return a && b && na && nb && x < y + nb && y < x + na;
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_sgns_fwd_ws(int64_t P, size_t *ws_bytes) {
    PGLB_CHECK_ARG(P >= 1 && ws_bytes, PGLB_EINVAL, "pglb_sgns_fwd_ws: bad args");
    *ws_bytes = SGNS_MAX_BLOCKS * sizeof(double);
    return PGLB_OK;
}

extern "C" int pglb_sgns_fwd_f32(const float *emb, int64_t n_emb, int64_t ld_emb, const float *ctx, int64_t n_ctx,
                                 int64_t ld_ctx, const int64_t *src, const int64_t *dsts, int64_t P, int64_t K,
                                 int64_t D, float *loss, float *c, float *w, int64_t ldw, void *ws, size_t ws_bytes,
                                 void *stream) {
    const char *name = "pglb_sgns_fwd_f32";
    PGLB_CHECK_ARG(emb && ctx && src && dsts && loss, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(P >= 1 && K >= 1 && D >= 1 && n_emb >= 1 && n_ctx >= 1, PGLB_EINVAL,
                   "%s: P, K, D, n_emb and n_ctx must be >= 1 (P=%lld K=%lld D=%lld)", name, (long long)P,
                   (long long)K, (long long)D);
    PGLB_CHECK_ARG(P < (1LL << 40) && K < (1LL << 20) && D < (1LL << 31), PGLB_ESHAPE, "%s: sizes too large", name);
    PGLB_CHECK_ARG(ld_emb >= D && ld_ctx >= D, PGLB_ESHAPE, "%s: leading dimension smaller than D", name);
    PGLB_CHECK_ARG(!c == !w, PGLB_EINVAL, "%s: c and w are given together (training) or not at all", name);
    const bool train = c != nullptr;
    PGLB_CHECK_ARG(!train || ldw >= D, PGLB_ESHAPE, "%s: ldw smaller than D", name);
    const int64_t J = K + 1;
    const size_t b_emb = (size_t)((n_emb - 1) * ld_emb + D) * 4, b_ctx = (size_t)((n_ctx - 1) * ld_ctx + D) * 4;
    const size_t b_src = (size_t)P * 8, b_dsts = (size_t)(P * J) * 8, b_c = (size_t)(P * J) * 4;
    const size_t b_w = train ? (size_t)((P - 1) * ldw + D) * 4 : 0;
    const void *in[4] = {emb, ctx, src, dsts};
    const size_t nin[4] = {b_emb, b_ctx, b_src, b_dsts};
    for (int i = 0; i < 4; ++i)
        PGLB_CHECK_ARG(!sgns_overlap(loss, 4, in[i], nin[i]) && !sgns_overlap(c, b_c, in[i], nin[i]) &&
                           !sgns_overlap(w, b_w, in[i], nin[i]),
                       PGLB_EINVAL, "%s: an output overlaps an input", name);
    PGLB_CHECK_ARG(!sgns_overlap(loss, 4, c, b_c) && !sgns_overlap(loss, 4, w, b_w) && !sgns_overlap(c, b_c, w, b_w),
                   PGLB_EINVAL, "%s: the outputs overlap", name);
    PGLB_CHECK_ARG(ws && ws_bytes >= SGNS_MAX_BLOCKS * sizeof(double) && (reinterpret_cast<uintptr_t>(ws) & 7u) == 0,
                   PGLB_EWORKSPACE, "%s: workspace too small or misaligned", name);

    SgnsArgs a{emb, ctx, src, dsts, c, w, static_cast<double *>(ws), ld_emb, ld_ctx, ldw, P, K, D};
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const bool vec = D % 4 == 0 && ld_emb % 4 == 0 && ld_ctx % 4 == 0 && sgns_a16(emb) && sgns_a16(ctx) &&
                     (!train || (ldw % 4 == 0 && sgns_a16(w)));
    unsigned grid;
    if (vec && D <= 16) grid = sgns_launch<4, 4, 1>(a, train, s);
    else if (vec && D <= 32) grid = sgns_launch<8, 4, 1>(a, train, s);
    else if (vec && D <= 64) grid = sgns_launch<16, 4, 1>(a, train, s);
    else if (vec && D <= 128) grid = sgns_launch<32, 4, 1>(a, train, s);
    else if (vec && D <= 256) grid = sgns_launch<32, 4, 2>(a, train, s);
    else if (vec && D <= 512) grid = sgns_launch<32, 4, 4>(a, train, s);
    else if (!vec && D <= 4) grid = sgns_launch<4, 1, 1>(a, train, s);
    else if (!vec && D <= 8) grid = sgns_launch<8, 1, 1>(a, train, s);
    else if (!vec && D <= 16) grid = sgns_launch<16, 1, 1>(a, train, s);
    else if (!vec && D <= 32) grid = sgns_launch<32, 1, 1>(a, train, s);
    else if (!vec && D <= 64) grid = sgns_launch<32, 1, 2>(a, train, s);
    else if (!vec && D <= 128) grid = sgns_launch<32, 1, 4>(a, train, s);
    else if (!vec && D <= 256) grid = sgns_launch<32, 1, 8>(a, train, s);
    else {
        grid = sgns_grid(P, SGNS_THREADS / 32);
        if (train)
            sgns_fwd_wide_kernel<true><<<grid, SGNS_THREADS, 0, s>>>(a);
        else
            sgns_fwd_wide_kernel<false><<<grid, SGNS_THREADS, 0, s>>>(a);
    }
    PGLB_LAUNCH_CHECK("sgns_fwd_kernel");
    sgns_loss_kernel<<<1, SGNS_THREADS, 0, s>>>(a.part, (int)grid, P, loss);
    PGLB_LAUNCH_CHECK("sgns_loss_kernel");
    return PGLB_OK;
}
