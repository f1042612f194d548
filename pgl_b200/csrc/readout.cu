// readout.cu -- graph-level readouts keyed by a segment CSR indptr[B + 1]: segment g is the contiguous rows
// indptr[g] .. indptr[g + 1] (a batched graph's _graph_node_index).
//   - fused attention readout (GlobalAttention / Set2Set): out[g] = sum_i softmax_g(s)_i x_i, s from a per-node gate
//     or from <x_i, q_g>, one pass over x with an online max and sum, and its backward;
//   - segmented top-k (SAGPool / segment_topk): k_g per segment, then the first k_g ranks of every segment;
//   - dense batching (to_dense_batch / segment_padding): [N, D] <-> [B, max_len, D] copies by element size.
// Every output element has exactly one writer and there are no atomics: results do not depend on the launch, and a
// segment's result does not depend on where it sits in the batch.
#include <algorithm>

#include "common.cuh"

namespace pglb {

// ---- attention readout --------------------------------------------------------------------------------------------
// A work item is one chunk of RO_CHUNK rows of one segment (a segment of n rows has max(1, ceil(n / RO_CHUNK))
// chunks, so the boundaries depend on n only).  One CTA per item; thread t owns the columns t, t + nt, ... of its
// accumulators (shared memory, touched by that thread only).  Rows are taken RO_R at a time: RO_R scores, one max
// update, RO_R weighted rows.  A single-chunk segment is finished by its item; a longer one writes a partial
// (m, s, v[D]) and ro_merge_kernel combines the partials in chunk order.
constexpr int RO_CHUNK = 2048;
constexpr int RO_R = 8;
constexpr int RO_MAX_D = 16384;  // shared memory: up to 3 D-float arrays per CTA (backward, query given)

static int ro_threads(int64_t D) {
    const int64_t per = (D + 255) / 256;  // columns per thread at 256 threads
    const int64_t nt = ((D + per - 1) / per + 31) / 32 * 32;
    return (int)std::max<int64_t>(32, std::min<int64_t>(256, nt));
}

static int64_t ro_items_bound(int64_t B, int64_t N) {
    // sum over segments of max(1, ceil(n / C)) <= B + sum over long segments of (n / C + 1) <= B + 2 N / C
    return B + 2 * ((N + RO_CHUNK - 1) / RO_CHUNK);
}

// sum of v[k] over the CTA, the totals in every thread; lanes by butterfly, then warps in order (deterministic)
template <int K>
__device__ __forceinline__ void block_sum(float (&v)[K], float *red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) red[w * K + k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float t = 0.0f;
        for (int j = 0; j < nw; ++j) t += red[j * K + k];
        v[k] = t;
    }
    __syncthreads();
}

// item w -> (segment g, chunk c, chunks of g).  off == nullptr: one item per segment.  Returns false past the end.
__device__ __forceinline__ bool ro_item(const int64_t *off, int64_t B, int64_t w, int64_t &g, int64_t &c,
                                        int64_t &nch) {
    if (!off) {
        g = w;
        c = 0;
        nch = 1;
        return w < B;
    }
    if (w >= off[B]) return false;
    int64_t lo = 0, hi = B;  // last g with off[g] <= w (off strictly increasing)
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= w) lo = mid;
        else hi = mid;
    }
    g = lo;
    c = w - off[g];
    nch = off[g + 1] - off[g];
    return true;
}

// end of item (g, c): the chunk's last row + 1.  Without item offsets (max_len <= RO_CHUNK) an item is the whole
// segment, so a max_len below the true longest segment still covers every row (that segment is read as one chunk).
__device__ __forceinline__ int64_t ro_chunk_end(const int64_t *off, int64_t s0, int64_t n, int64_t b) {
    return off ? std::min<int64_t>(s0 + n, b + RO_CHUNK) : s0 + n;
}

struct RoFwd {
    const float *x;
    const int64_t *indptr;
    const float *gate;
    const float *query;
    int64_t B, D;
    float *out, *lse;
    const int64_t *off;
    float *part;  // [items][D + 2]: m, s, v[D]
};

template <bool QUERY>
__global__ void __launch_bounds__(256) attn_readout_kernel(RoFwd a) {
    extern __shared__ float ro_smem[];
    __shared__ float red[8 * RO_R];
    int64_t g, c, nch;
    const int64_t w = blockIdx.x;
    if (!ro_item(a.off, a.B, w, g, c, nch)) return;
    const int64_t D = a.D, nt = blockDim.x;
    const int64_t s0 = a.indptr[g], n = a.indptr[g + 1] - s0;
    const int64_t b = s0 + c * RO_CHUNK, e = ro_chunk_end(a.off, s0, n, b);
    float *acc = ro_smem, *q = ro_smem + D;
    for (int64_t col = threadIdx.x; col < D; col += nt) {
        acc[col] = 0.0f;
        if (QUERY) q[col] = a.query[g * D + col];
    }
    float m = -INFINITY, ssum = 0.0f;
    for (int64_t i0 = b; i0 < e; i0 += RO_R) {
        float s[RO_R];
        if (QUERY) {
#pragma unroll
            for (int r = 0; r < RO_R; ++r) s[r] = 0.0f;
            for (int64_t col = threadIdx.x; col < D; col += nt) {
                const float qc = q[col];
#pragma unroll
                for (int r = 0; r < RO_R; ++r)
                    if (i0 + r < e) s[r] = fmaf(__ldg(a.x + (i0 + r) * D + col), qc, s[r]);
            }
            block_sum<RO_R>(s, red);
#pragma unroll
            for (int r = 0; r < RO_R; ++r)
                if (i0 + r >= e) s[r] = -INFINITY;
        } else {
#pragma unroll
            for (int r = 0; r < RO_R; ++r) s[r] = i0 + r < e ? __ldg(a.gate + i0 + r) : -INFINITY;
        }
        float mn = m;
#pragma unroll
        for (int r = 0; r < RO_R; ++r) mn = fmaxf(mn, s[r]);
        const float sc = mn == m ? 1.0f : expf(m - mn);
        float wr[RO_R];
        ssum *= sc;
#pragma unroll
        for (int r = 0; r < RO_R; ++r) {
            wr[r] = s[r] == -INFINITY ? 0.0f : expf(s[r] - mn);
            ssum += wr[r];
        }
        for (int64_t col = threadIdx.x; col < D; col += nt) {
            float v = acc[col] * sc;
#pragma unroll
            for (int r = 0; r < RO_R; ++r)
                if (i0 + r < e) v = fmaf(wr[r], __ldg(a.x + (i0 + r) * D + col), v);
            acc[col] = v;
        }
        m = mn;
    }
    if (nch == 1) {
        for (int64_t col = threadIdx.x; col < D; col += nt) a.out[g * D + col] = n ? __fdiv_rn(acc[col], ssum) : 0.0f;
        if (threadIdx.x == 0) a.lse[g] = n ? m + logf(ssum) : -INFINITY;
    } else {
        float *p = a.part + w * (D + 2);
        if (threadIdx.x == 0) {
            p[0] = m;
            p[1] = ssum;
        }
        for (int64_t col = threadIdx.x; col < D; col += nt) p[2 + col] = acc[col];
    }
}

// the first item of every multi-chunk segment combines that segment's partials, in chunk order
__global__ void __launch_bounds__(256) ro_merge_kernel(const int64_t *off, int64_t B, int64_t D,
                                                       const float *__restrict__ part, float *__restrict__ out,
                                                       float *__restrict__ lse) {
    int64_t g, c, nch;
    if (!ro_item(off, B, blockIdx.x, g, c, nch) || c != 0 || nch == 1) return;
    const float *p0 = part + (int64_t)blockIdx.x * (D + 2);
    float M = -INFINITY;
    for (int64_t k = 0; k < nch; ++k) M = fmaxf(M, p0[k * (D + 2)]);
    float S = 0.0f;
    for (int64_t k = 0; k < nch; ++k) {
        const float mk = p0[k * (D + 2)];
        S += p0[k * (D + 2) + 1] * (mk == M ? 1.0f : expf(mk - M));
    }
    for (int64_t col = threadIdx.x; col < D; col += blockDim.x) {
        float v = 0.0f;
        for (int64_t k = 0; k < nch; ++k) {
            const float mk = p0[k * (D + 2)];
            v = fmaf(p0[k * (D + 2) + 2 + col], mk == M ? 1.0f : expf(mk - M), v);
        }
        out[g * D + col] = __fdiv_rn(v, S);
    }
    if (threadIdx.x == 0) lse[g] = M + logf(S);
}

struct RoBwd {
    const float *x;
    const int64_t *indptr;
    const float *gate;
    const float *query;
    const float *r;  // forward output
    const float *lse;
    const float *gout;
    int64_t B, D;
    float *gx, *ggate, *gq;
    const int64_t *off;
    float *part;  // [items][D]: partial grad_q
};

// a_i = exp(s_i - lse_g), ds_i = a_i (<x_i, gout_g> - <r_g, gout_g>), grad_x_i = a_i gout_g (+ ds_i q_g),
// grad_gate_i = ds_i, grad_q_g = sum_i ds_i x_i
template <bool QUERY>
__global__ void __launch_bounds__(256) attn_readout_bwd_kernel(RoBwd a) {
    extern __shared__ float ro_smem[];
    constexpr int K = QUERY ? 2 * RO_R : RO_R;
    __shared__ float red[8 * K];
    int64_t g, c, nch;
    const int64_t w = blockIdx.x;
    if (!ro_item(a.off, a.B, w, g, c, nch)) return;
    const int64_t D = a.D, nt = blockDim.x;
    const int64_t s0 = a.indptr[g], n = a.indptr[g + 1] - s0;
    const int64_t b = s0 + c * RO_CHUNK, e = ro_chunk_end(a.off, s0, n, b);
    float *go = ro_smem, *q = ro_smem + D, *gq = ro_smem + 2 * D;
    float cg[1] = {0.0f};
    for (int64_t col = threadIdx.x; col < D; col += nt) {
        go[col] = a.gout[g * D + col];
        cg[0] = fmaf(a.r[g * D + col], go[col], cg[0]);
        if (QUERY) {
            q[col] = a.query[g * D + col];
            gq[col] = 0.0f;
        }
    }
    block_sum<1>(cg, red);
    const float L = n ? a.lse[g] : 0.0f;
    for (int64_t i0 = b; i0 < e; i0 += RO_R) {
        float v[K];  // <x_i, gout_g> for the RO_R rows, then (query) <x_i, q_g>
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = 0.0f;
        for (int64_t col = threadIdx.x; col < D; col += nt) {
            const float gc = go[col];
            const float qc = QUERY ? q[col] : 0.0f;
#pragma unroll
            for (int r = 0; r < RO_R; ++r) {
                if (i0 + r < e) {
                    const float xv = __ldg(a.x + (i0 + r) * D + col);
                    v[r] = fmaf(xv, gc, v[r]);
                    if (QUERY) v[RO_R + r] = fmaf(xv, qc, v[RO_R + r]);
                }
            }
        }
        block_sum<K>(v, red);
        float al[RO_R], ds[RO_R];
#pragma unroll
        for (int r = 0; r < RO_R; ++r) {
            al[r] = ds[r] = 0.0f;
            if (i0 + r < e) {
                const float s = QUERY ? v[RO_R + r] : __ldg(a.gate + i0 + r);
                al[r] = expf(s - L);
                ds[r] = al[r] * (v[r] - cg[0]);
                if (a.ggate && threadIdx.x == 0) a.ggate[i0 + r] = ds[r];
            }
        }
        for (int64_t col = threadIdx.x; col < D; col += nt) {
            const float gc = go[col];
            const float qc = QUERY ? q[col] : 0.0f;
            float acc = QUERY ? gq[col] : 0.0f;
#pragma unroll
            for (int r = 0; r < RO_R; ++r) {
                if (i0 + r < e) {
                    float gxv = al[r] * gc;
                    if (QUERY) {
                        gxv = fmaf(ds[r], qc, gxv);
                        acc = fmaf(ds[r], __ldg(a.x + (i0 + r) * D + col), acc);
                    }
                    a.gx[(i0 + r) * D + col] = gxv;
                }
            }
            if (QUERY) gq[col] = acc;
        }
    }
    if (QUERY) {
        float *dst = nch == 1 ? a.gq + g * D : a.part + w * D;
        for (int64_t col = threadIdx.x; col < D; col += nt) dst[col] = gq[col];
    }
}

__global__ void __launch_bounds__(256) ro_merge_gq_kernel(const int64_t *off, int64_t B, int64_t D,
                                                          const float *__restrict__ part, float *__restrict__ gq) {
    int64_t g, c, nch;
    if (!ro_item(off, B, blockIdx.x, g, c, nch) || c != 0 || nch == 1) return;
    const float *p0 = part + (int64_t)blockIdx.x * D;
    for (int64_t col = threadIdx.x; col < D; col += blockDim.x) {
        float v = 0.0f;
        for (int64_t k = 0; k < nch; ++k) v += p0[k * D + col];
        gq[g * D + col] = v;
    }
}

// cnt[g] = chunks of segment g, cnt[B] = 0 (exclusive-scanned in place into the item offsets)
__global__ void __launch_bounds__(256) ro_count_kernel(const int64_t *indptr, int64_t B, int64_t *cnt) {
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= B; g += (int64_t)gridDim.x * blockDim.x) {
        if (g == B) {
            cnt[g] = 0;
            continue;
        }
        const int64_t n = indptr[g + 1] - indptr[g];
        cnt[g] = n <= RO_CHUNK ? 1 : (n + RO_CHUNK - 1) / RO_CHUNK;
    }
}

struct RoPlan {
    size_t off, scan, part, total;
};

static RoPlan ro_plan(int64_t B, int64_t N, int64_t D) {
    RoPlan p;
    p.off = 0;
    p.scan = align_up(sizeof(int64_t) * (size_t)(B + 1), 256);
    p.part = p.scan + scan_i64_ws_bytes(B + 1);
    p.total = p.part + align_up(sizeof(float) * (size_t)ro_items_bound(B, N) * (size_t)(D + 2), 256);
    return p;
}

// chunked mode: item offsets into the workspace; returns the grid (an upper bound on the items)
static int ro_chunk_offsets(const int64_t *indptr, int64_t B, int64_t N, const RoPlan &p, char *ws,
                            cudaStream_t stream, int64_t *&off, int64_t &grid) {
    off = reinterpret_cast<int64_t *>(ws + p.off);
    ro_count_kernel<<<(unsigned)std::min<int64_t>((B + 256) / 256, (int64_t)sm_count() * 16), 256, 0, stream>>>(
        indptr, B, off);
    PGLB_LAUNCH_CHECK("ro_count_kernel");
    const int rc = scan_i64(off, off, B + 1, /*inclusive=*/0, ws + p.scan, stream);
    if (rc) return rc;
    grid = ro_items_bound(B, N);
    return PGLB_OK;
}

static int ro_check(const char *name, int64_t N, int64_t D, const int64_t *indptr, int64_t B, const float *gate,
                    const float *query) {
    PGLB_CHECK_ARG(N >= 0 && B >= 0 && D >= 1, PGLB_EINVAL, "%s: negative size or D < 1", name);
    PGLB_CHECK_ARG((gate == nullptr) != (query == nullptr), PGLB_EINVAL, "%s: pass exactly one of gate and query",
                   name);
    PGLB_CHECK_ARG(D <= RO_MAX_D, PGLB_EUNSUPPORTED, "%s: D must be at most %d", name, RO_MAX_D);
    PGLB_CHECK_ARG(B == 0 || indptr != nullptr, PGLB_EINVAL, "%s: indptr is NULL", name);
    return PGLB_OK;
}

static std::atomic<unsigned long long> g_ro_smem_done[4];

template <typename K>
static int ro_opt_in(K kernel, size_t bytes, int which) {
    if (bytes > 48 * 1024) PGLB_CUDA(ensure_dyn_smem(kernel, (int)bytes, g_ro_smem_done[which]));
    return PGLB_OK;
}

// ---- segmented top-k ----------------------------------------------------------------------------------------------
constexpr int TOPK_SMEM_MAX = 2048;  // longest segment ranked inside one CTA
constexpr int TOPK_T = 1024;

// order key of a score: larger key = earlier rank.  -0.0 == +0.0; NaN below every number (-inf included).
__device__ __forceinline__ uint32_t topk_key(float f) {
    if (f != f) return 0u;
    if (f == 0.0f) f = 0.0f;
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// one CTA: k_g, the exclusive prefix off[0 .. B] and info = {off[B], longest segment}
__global__ void __launch_bounds__(TOPK_T) topk_count_kernel(const int64_t *__restrict__ indptr, int64_t B,
                                                            float ratio, int64_t kint, int64_t *__restrict__ off,
                                                            int64_t *__restrict__ info) {
    __shared__ int64_t wsum[TOPK_T / 32];
    __shared__ int64_t wmax[TOPK_T / 32];
    __shared__ int64_t carry;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    int64_t mx = 0;
    __syncthreads();
    for (int64_t g0 = 0; g0 < B; g0 += TOPK_T) {
        const int64_t g = g0 + threadIdx.x;
        int64_t k = 0;
        if (g < B) {
            const int64_t n = indptr[g + 1] - indptr[g];
            mx = max(mx, n);
            k = kint > 0 ? min(kint, n) : min((int64_t)ceilf(ratio * (float)n), n);
        }
        int64_t incl = k;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[wid] = incl;
        __syncthreads();
        int64_t base = carry, tot = 0;
        for (int j = 0; j < TOPK_T / 32; ++j) {
            if (j < wid) base += wsum[j];
            tot += wsum[j];
        }
        if (g < B) off[g] = base + incl - k;
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) wmax[wid] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t m = 0;
        for (int j = 0; j < TOPK_T / 32; ++j) m = max(m, wmax[j]);
        off[B] = carry;
        info[0] = carry;
        info[1] = m;
    }
}

// one CTA per segment of at most TOPK_SMEM_MAX nodes: rank = number of nodes that come before in the total order
__global__ void __launch_bounds__(256) topk_smem_kernel(const float *__restrict__ scores,
                                                        const int64_t *__restrict__ indptr,
                                                        const int64_t *__restrict__ off, int64_t *__restrict__ perm) {
    __shared__ uint32_t key[TOPK_SMEM_MAX];
    const int64_t g = blockIdx.x;
    const int64_t s0 = indptr[g];
    const int64_t n = indptr[g + 1] - s0;
    const int64_t o = off[g];
    const int64_t k = off[g + 1] - o;
    if (k == 0) return;
    // a segment longer than the shared array (a max_len below the true longest segment) is ranked from global memory:
    // the same ranks, only slower
    const bool staged = n <= TOPK_SMEM_MAX;
    if (staged)
        for (int i = threadIdx.x; i < n; i += blockDim.x) key[i] = topk_key(__ldg(scores + s0 + i));
    __syncthreads();
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t ki = staged ? key[i] : topk_key(__ldg(scores + s0 + i));
        int64_t r = 0;
        for (int64_t j = 0; j < n; ++j) {
            const uint32_t kj = staged ? key[j] : topk_key(__ldg(scores + s0 + j));
            r += (kj > ki) | ((kj == ki) & (j < i));
        }
        if (r < k) perm[o + r] = s0 + i;
    }
}

// long path: sort (segment << 32 | ~key) ascending, stable, with the node id as the value.  Nodes outside
// [indptr[0], indptr[B]) belong to no segment, as on the shared-memory path: those before take the low word 0 in
// segment 0 and those after take 0xffffffff in segment B - 1 (no score maps there: ~key >= 0x007fffff, NaN ties and
// loses on the node id), so every segment's members keep the sorted positions [indptr[g], indptr[g + 1]).
__global__ void __launch_bounds__(256) topk_pack_kernel(const float *__restrict__ scores, int64_t N,
                                                        const int64_t *__restrict__ indptr, int64_t B,
                                                        uint64_t *__restrict__ keys, uint64_t *__restrict__ vals) {
    const int64_t first = __ldg((const long long *)indptr), last = __ldg((const long long *)indptr + B);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = B;  // last g with indptr[g] <= i
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg((const long long *)indptr + mid) <= i) lo = mid;
            else hi = mid;
        }
        const uint32_t low = i < first ? 0u : i >= last ? 0xffffffffu : ~topk_key(__ldg(scores + i));
        keys[i] = ((uint64_t)lo << 32) | (uint64_t)low;
        vals[i] = (uint64_t)i;
    }
}

__global__ void __launch_bounds__(256) topk_emit_kernel(const uint64_t *__restrict__ keys,
                                                        const uint64_t *__restrict__ vals, int64_t N,
                                                        const int64_t *__restrict__ indptr,
                                                        const int64_t *__restrict__ off, int64_t *__restrict__ perm) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = (int64_t)(keys[p] >> 32);
        const int64_t r = p - indptr[g];  // < 0 before indptr[0], >= the segment's length after indptr[B]
        if (r >= 0 && r < off[g + 1] - off[g]) perm[off[g] + r] = (int64_t)vals[p];
    }
}

static int key_bits_of(int64_t n) {
    int b = 1;
    while (b < 62 && ((int64_t)1 << b) < n) ++b;
    return b;
}

struct TopkPlan {
    size_t ka, kb, va, vb, sort, total;
};

static TopkPlan topk_plan(int64_t N, int64_t max_len) {
    TopkPlan p{};
    if (max_len <= TOPK_SMEM_MAX) return p;
    const size_t a = align_up(sizeof(uint64_t) * (size_t)std::max<int64_t>(N, 1), 256);
    p.ka = 0;
    p.kb = a;
    p.va = 2 * a;
    p.vb = 3 * a;
    p.sort = 4 * a;
    p.total = p.sort + radix_sort_u64_ws_bytes(N);
    return p;
}

// ---- dense batching -----------------------------------------------------------------------------------------------
// pad: one warp per output row (b, p) of [B, L, D]; unpad: one warp per node row i
template <typename T>
__global__ void __launch_bounds__(256) segment_pad_kernel(const T *__restrict__ x, int64_t D,
                                                          const int64_t *__restrict__ indptr, int64_t B, int64_t L,
                                                          T fill, T *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < B * L; row += nw) {
        const int64_t b = row / L, p = row - b * L;
        const int64_t s0 = indptr[b];
        T *o = out + row * D;
        if (p < indptr[b + 1] - s0) {
            const T *src = x + (s0 + p) * D;
            for (int64_t j = lane; j < D; j += 32) o[j] = src[j];
        } else {
            for (int64_t j = lane; j < D; j += 32) o[j] = fill;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) segment_unpad_kernel(const T *__restrict__ padded, int64_t D,
                                                            const int64_t *__restrict__ indptr, int64_t B, int64_t L,
                                                            int64_t N, T *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < N; i += nw) {
        int64_t lo = 0, hi = B;  // last b with indptr[b] <= i
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg((const long long *)indptr + mid) <= i) lo = mid;
            else hi = mid;
        }
        const int64_t p = i - indptr[lo];
        T *o = out + i * D;
        if (p < L) {
            const T *src = padded + (lo * L + p) * D;
            for (int64_t j = lane; j < D; j += 32) o[j] = src[j];
        } else {
            for (int64_t j = lane; j < D; j += 32) o[j] = T(0);
        }
    }
}

static unsigned warp_grid(int64_t rows) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 7) / 8, (int64_t)sm_count() * 32));
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_attn_readout_ws(int64_t B, int64_t N, int64_t D, int64_t max_len, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr, PGLB_EINVAL, "pglb_attn_readout_ws: ws_bytes is NULL");
    PGLB_CHECK_ARG(B >= 0 && N >= 0 && D >= 1 && max_len >= 0, PGLB_EINVAL,
                   "pglb_attn_readout_ws: negative size or D < 1");
    *ws_bytes = max_len <= RO_CHUNK ? 0 : ro_plan(B, N, D).total;
    return PGLB_OK;
}

extern "C" int pglb_attn_readout_f32(const float *x, int64_t N, int64_t D, const int64_t *indptr, int64_t B,
                                     int64_t max_len, const float *gate, const float *query, float *out, float *lse,
                                     void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_attn_readout_f32";
    if (const int rc = ro_check(name, N, D, indptr, B, gate, query)) return rc;
    PGLB_CHECK_ARG(max_len >= 0, PGLB_EINVAL, "%s: negative max_len", name);
    PGLB_CHECK_ARG(B == 0 || (out && lse), PGLB_EINVAL, "%s: NULL output", name);
    PGLB_CHECK_ARG(N == 0 || x, PGLB_EINVAL, "%s: x is NULL", name);
    size_t need = 0;
    pglb_attn_readout_ws(B, N, D, max_len, &need);
    PGLB_CHECK_ARG(need == 0 || (ws && ws_bytes >= need && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0),
                   PGLB_EWORKSPACE, "%s: workspace of %zu bytes needed (got %zu)", name, need, ws_bytes);
    if (B == 0) return PGLB_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    RoFwd a{x, indptr, gate, query, B, D, out, lse, nullptr, nullptr};
    int64_t grid = B;
    RoPlan p{};
    if (need) {
        p = ro_plan(B, N, D);
        int64_t *off;
        if (const int rc = ro_chunk_offsets(indptr, B, N, p, reinterpret_cast<char *>(ws), stream, off, grid))
            return rc;
        a.off = off;
        a.part = reinterpret_cast<float *>(reinterpret_cast<char *>(ws) + p.part);
    }
    const int nt = ro_threads(D);
    const size_t smem = sizeof(float) * (size_t)D * (query ? 2 : 1);
    if (query) {
        if (const int rc = ro_opt_in(attn_readout_kernel<true>, smem, 0)) return rc;
        attn_readout_kernel<true><<<(unsigned)grid, nt, smem, stream>>>(a);
    } else {
        if (const int rc = ro_opt_in(attn_readout_kernel<false>, smem, 1)) return rc;
        attn_readout_kernel<false><<<(unsigned)grid, nt, smem, stream>>>(a);
    }
    PGLB_LAUNCH_CHECK("attn_readout_kernel");
    if (need) {
        ro_merge_kernel<<<(unsigned)grid, nt, 0, stream>>>(a.off, B, D, a.part, out, lse);
        PGLB_LAUNCH_CHECK("ro_merge_kernel");
    }
    return PGLB_OK;
}

extern "C" int pglb_attn_readout_bwd_f32(const float *x, int64_t N, int64_t D, const int64_t *indptr, int64_t B,
                                         int64_t max_len, const float *gate, const float *query, const float *out,
                                         const float *lse, const float *grad_out, float *grad_x, float *grad_gate,
                                         float *grad_query, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_attn_readout_bwd_f32";
    if (const int rc = ro_check(name, N, D, indptr, B, gate, query)) return rc;
    PGLB_CHECK_ARG(max_len >= 0, PGLB_EINVAL, "%s: negative max_len", name);
    PGLB_CHECK_ARG(B == 0 || (out && lse && grad_out && (query == nullptr || grad_query)), PGLB_EINVAL,
                   "%s: NULL pointer", name);
    PGLB_CHECK_ARG(N == 0 || (x && grad_x), PGLB_EINVAL, "%s: x or grad_x is NULL", name);
    size_t need = 0;
    pglb_attn_readout_ws(B, N, D, max_len, &need);
    PGLB_CHECK_ARG(need == 0 || (ws && ws_bytes >= need && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0),
                   PGLB_EWORKSPACE, "%s: workspace of %zu bytes needed (got %zu)", name, need, ws_bytes);
    if (B == 0) return PGLB_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    RoBwd a{x, indptr, gate, query, out, lse, grad_out, B, D, grad_x, grad_gate, grad_query, nullptr, nullptr};
    int64_t grid = B;
    if (need) {
        const RoPlan p = ro_plan(B, N, D);
        int64_t *off;
        if (const int rc = ro_chunk_offsets(indptr, B, N, p, reinterpret_cast<char *>(ws), stream, off, grid))
            return rc;
        a.off = off;
        a.part = reinterpret_cast<float *>(reinterpret_cast<char *>(ws) + p.part);
    }
    const int nt = ro_threads(D);
    const size_t smem = sizeof(float) * (size_t)D * (query ? 3 : 1);
    if (query) {
        if (const int rc = ro_opt_in(attn_readout_bwd_kernel<true>, smem, 2)) return rc;
        attn_readout_bwd_kernel<true><<<(unsigned)grid, nt, smem, stream>>>(a);
    } else {
        if (const int rc = ro_opt_in(attn_readout_bwd_kernel<false>, smem, 3)) return rc;
        attn_readout_bwd_kernel<false><<<(unsigned)grid, nt, smem, stream>>>(a);
    }
    PGLB_LAUNCH_CHECK("attn_readout_bwd_kernel");
    if (need && query) {
        ro_merge_gq_kernel<<<(unsigned)grid, nt, 0, stream>>>(a.off, B, D, a.part, grad_query);
        PGLB_LAUNCH_CHECK("ro_merge_gq_kernel");
    }
    return PGLB_OK;
}

extern "C" int pglb_segment_topk_count(const int64_t *indptr, int64_t B, float ratio, int64_t k, int64_t *offsets,
                                       int64_t *info, void *stream) {
    const char *name = "pglb_segment_topk_count";
    PGLB_CHECK_ARG(B >= 0 && k >= 0, PGLB_EINVAL, "%s: negative size or k", name);
    PGLB_CHECK_ARG(k > 0 || (ratio > 0.0f && ratio <= 1.0f), PGLB_EINVAL, "%s: a float ratio must lie in (0, 1]",
                   name);
    PGLB_CHECK_ARG(offsets && info && (B == 0 || indptr), PGLB_EINVAL, "%s: NULL pointer", name);
    topk_count_kernel<<<1, TOPK_T, 0, reinterpret_cast<cudaStream_t>(stream)>>>(indptr, B, ratio, k, offsets, info);
    PGLB_LAUNCH_CHECK("topk_count_kernel");
    return PGLB_OK;
}

extern "C" int pglb_segment_topk_ws(int64_t B, int64_t N, int64_t max_len, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr, PGLB_EINVAL, "pglb_segment_topk_ws: ws_bytes is NULL");
    PGLB_CHECK_ARG(B >= 0 && N >= 0 && max_len >= 0, PGLB_EINVAL, "pglb_segment_topk_ws: negative size");
    *ws_bytes = topk_plan(N, max_len).total;
    return PGLB_OK;
}

extern "C" int pglb_segment_topk_fill(const float *scores, int64_t N, const int64_t *indptr, int64_t B,
                                      const int64_t *offsets, int64_t max_len, int64_t *perm, void *ws,
                                      size_t ws_bytes, void *stream_) {
    const char *name = "pglb_segment_topk_fill";
    PGLB_CHECK_ARG(B >= 0 && N >= 0 && max_len >= 0 && max_len <= N, PGLB_EINVAL, "%s: bad size", name);
    PGLB_CHECK_ARG(B == 0 || (indptr && offsets), PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(N == 0 || (scores && perm), PGLB_EINVAL, "%s: NULL pointer", name);
    const TopkPlan p = topk_plan(N, max_len);
    PGLB_CHECK_ARG(p.total == 0 || (ws && ws_bytes >= p.total && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0),
                   PGLB_EWORKSPACE, "%s: workspace of %zu bytes needed (got %zu)", name, p.total, ws_bytes);
    if (B == 0 || N == 0) return PGLB_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (max_len <= TOPK_SMEM_MAX) {
        topk_smem_kernel<<<(unsigned)B, 256, 0, stream>>>(scores, indptr, offsets, perm);
        PGLB_LAUNCH_CHECK("topk_smem_kernel");
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(B < ((int64_t)1 << 30), PGLB_EUNSUPPORTED, "%s: at most 2^30 segments on the sort path", name);
    char *base = reinterpret_cast<char *>(ws);
    uint64_t *ka = reinterpret_cast<uint64_t *>(base + p.ka), *kb = reinterpret_cast<uint64_t *>(base + p.kb);
    uint64_t *va = reinterpret_cast<uint64_t *>(base + p.va), *vb = reinterpret_cast<uint64_t *>(base + p.vb);
    const unsigned grid = (unsigned)std::min<int64_t>((N + 255) / 256, (int64_t)sm_count() * 16);
    topk_pack_kernel<<<grid, 256, 0, stream>>>(scores, N, indptr, B, ka, va);
    PGLB_LAUNCH_CHECK("topk_pack_kernel");
    int in_alt = 0;
    if (const int rc = radix_sort_u64(ka, va, kb, vb, N, 32 + key_bits_of(B), base + p.sort, stream, &in_alt))
        return rc;
    topk_emit_kernel<<<grid, 256, 0, stream>>>(in_alt ? kb : ka, in_alt ? vb : va, N, indptr, offsets, perm);
    PGLB_LAUNCH_CHECK("topk_emit_kernel");
    return PGLB_OK;
}

static int pad_check(const char *name, int64_t N, int64_t D, int elem_size, const int64_t *indptr, int64_t B,
                     int64_t L) {
    PGLB_CHECK_ARG(N >= 0 && D >= 0 && B >= 0 && L >= 0, PGLB_EINVAL, "%s: negative size", name);
    PGLB_CHECK_ARG(elem_size == 2 || elem_size == 4 || elem_size == 8, PGLB_EINVAL,
                   "%s: element size must be 2, 4 or 8 bytes", name);
    PGLB_CHECK_ARG(B == 0 || indptr, PGLB_EINVAL, "%s: indptr is NULL", name);
    return PGLB_OK;
}

extern "C" int pglb_segment_pad(const void *x, int64_t N, int64_t D, int elem_size, const int64_t *indptr, int64_t B,
                                int64_t max_len, uint64_t fill_bits, void *out, void *stream_) {
    const char *name = "pglb_segment_pad";
    if (const int rc = pad_check(name, N, D, elem_size, indptr, B, max_len)) return rc;
    PGLB_CHECK_ARG((N == 0 || x) && (B * max_len == 0 || out), PGLB_EINVAL, "%s: NULL pointer", name);
    const int64_t rows = B * max_len;
    if (rows == 0 || D == 0) return PGLB_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const unsigned grid = warp_grid(rows);
    if (elem_size == 2)
        segment_pad_kernel<uint16_t><<<grid, 256, 0, stream>>>(static_cast<const uint16_t *>(x), D, indptr, B, max_len,
                                                               (uint16_t)fill_bits, static_cast<uint16_t *>(out));
    else if (elem_size == 4)
        segment_pad_kernel<uint32_t><<<grid, 256, 0, stream>>>(static_cast<const uint32_t *>(x), D, indptr, B, max_len,
                                                               (uint32_t)fill_bits, static_cast<uint32_t *>(out));
    else
        segment_pad_kernel<uint64_t><<<grid, 256, 0, stream>>>(static_cast<const uint64_t *>(x), D, indptr, B, max_len,
                                                               (uint64_t)fill_bits, static_cast<uint64_t *>(out));
    PGLB_LAUNCH_CHECK("segment_pad_kernel");
    return PGLB_OK;
}

extern "C" int pglb_segment_unpad(const void *padded, int64_t B, int64_t max_len, int64_t D, int elem_size,
                                  const int64_t *indptr, int64_t N, void *out, void *stream_) {
    const char *name = "pglb_segment_unpad";
    if (const int rc = pad_check(name, N, D, elem_size, indptr, B, max_len)) return rc;
    PGLB_CHECK_ARG(N == 0 || (out && B > 0 && (max_len == 0 || padded)), PGLB_EINVAL, "%s: NULL pointer or no segment",
                   name);
    if (N == 0 || D == 0) return PGLB_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const unsigned grid = warp_grid(N);
    if (elem_size == 2)
        segment_unpad_kernel<uint16_t><<<grid, 256, 0, stream>>>(static_cast<const uint16_t *>(padded), D, indptr, B,
                                                                 max_len, N, static_cast<uint16_t *>(out));
    else if (elem_size == 4)
        segment_unpad_kernel<uint32_t><<<grid, 256, 0, stream>>>(static_cast<const uint32_t *>(padded), D, indptr, B,
                                                                 max_len, N, static_cast<uint32_t *>(out));
    else
        segment_unpad_kernel<uint64_t><<<grid, 256, 0, stream>>>(static_cast<const uint64_t *>(padded), D, indptr, B,
                                                                 max_len, N, static_cast<uint64_t *>(out));
    PGLB_LAUNCH_CHECK("segment_unpad_kernel");
    return PGLB_OK;
}
