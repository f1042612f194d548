// csr_build.cu -- device CSR/CSC construction, bit-identical to the reference's stable
// counting sort (pgl/graph_kernel.pyx:59-88): degree histogram, exclusive scan, and a
// STABLE key sort of (u, edge id) so that every bucket keeps ascending edge id.
//
// Everything here is hand-written (no CUB / Thrust): a three-kernel multi-block int64 scan and an
// LSD radix sort of (key, value) pairs, 8 bits per pass.  A pass is (1) per-block digit histograms,
// (2) one scan of the digit-major [256 x blocks] table, (3) a scatter in which every warp ranks its
// contiguous sub-tile in order (__match_any_sync + popc, so equal digits keep their order), the
// block stages the tile in shared memory grouped by digit and writes each digit run coalesced.
// Order inside a digit is preserved at every level (lane, warp, block, grid) => the sort is stable
// => sorted_eid is ascending inside every row, exactly like the reference's counting sort.
// One-off index preparation, cached on the EdgeIndex; the per-layer hot loop never calls it.
#include <algorithm>

#include "common.cuh"

namespace pglb {

// ---- multi-block scan of int64 ---------------------------------------------------------------
constexpr int SCAN_T = 256;
constexpr int SCAN_IPT = 8;
constexpr int SCAN_TILE = SCAN_T * SCAN_IPT;

__device__ __forceinline__ int64_t block_exclusive_scan_256(int64_t v, int64_t *total) {
    // exclusive prefix of v over the 256 threads of the block
    __shared__ int64_t wsum[8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();  // protects wsum against the previous use
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    int64_t base = 0, tot = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j < w) base += wsum[j];
        tot += wsum[j];
    }
    if (total) *total = tot;
    return base + incl - v;
}

__global__ void __launch_bounds__(SCAN_T) scan_tile_sums_kernel(const int64_t *__restrict__ in, int64_t n,
                                                                int64_t *__restrict__ sums) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    int64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int64_t i = base + k * SCAN_T + threadIdx.x;
        if (i < n) s += in[i];
    }
    int64_t tot;
    block_exclusive_scan_256(s, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

// one block: sums[] -> exclusive prefix in place
__global__ void __launch_bounds__(SCAN_T) scan_sums_kernel(int64_t *sums, int64_t nb) {
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < nb; b0 += SCAN_T) {
        const int64_t i = b0 + threadIdx.x;
        const int64_t v = i < nb ? sums[i] : 0;
        int64_t tot;
        const int64_t ex = block_exclusive_scan_256(v, &tot);
        const int64_t c = carry;
        if (i < nb) sums[i] = c + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry = c + tot;
        __syncthreads();
    }
}

// out[i] = (inclusive ? in[i] : 0) + sum_{j<i} in[j]; thread t owns SCAN_IPT consecutive items
__global__ void __launch_bounds__(SCAN_T) scan_apply_kernel(const int64_t *__restrict__ in,
                                                            int64_t *__restrict__ out, int64_t n,
                                                            const int64_t *__restrict__ sums,
                                                            int inclusive) {
    __shared__ int64_t tile[SCAN_TILE];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int64_t i = base + k * SCAN_T + threadIdx.x;
        tile[k * SCAN_T + threadIdx.x] = i < n ? in[i] : 0;
    }
    __syncthreads();
    int64_t loc[SCAN_IPT];
    int64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        loc[k] = tile[threadIdx.x * SCAN_IPT + k];
        s += loc[k];
    }
    int64_t run = sums[blockIdx.x] + block_exclusive_scan_256(s, nullptr);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int64_t ex = run;
        run += loc[k];
        tile[threadIdx.x * SCAN_IPT + k] = inclusive ? run : ex;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int64_t i = base + k * SCAN_T + threadIdx.x;
        if (i < n) out[i] = tile[k * SCAN_T + threadIdx.x];
    }
}

static inline int64_t scan_blocks(int64_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }
static inline size_t scan_ws_bytes(int64_t n) { return align_up(sizeof(int64_t) * (size_t)std::max<int64_t>(scan_blocks(n), 1), 256); }
size_t scan_i64_ws_bytes(int64_t n) { return scan_ws_bytes(n); }

// in and out may alias.  tmp: scan_ws_bytes(n).  (also used by localgraph.cu)
int scan_i64(const int64_t *in, int64_t *out, int64_t n, int inclusive, void *tmp,
                    cudaStream_t stream) {
    if (n <= 0) return PGLB_OK;
    const int64_t nb = scan_blocks(n);
    int64_t *sums = reinterpret_cast<int64_t *>(tmp);
    scan_tile_sums_kernel<<<(unsigned)nb, SCAN_T, 0, stream>>>(in, n, sums);
    PGLB_LAUNCH_CHECK("scan_tile_sums_kernel");
    scan_sums_kernel<<<1, SCAN_T, 0, stream>>>(sums, nb);
    PGLB_LAUNCH_CHECK("scan_sums_kernel");
    scan_apply_kernel<<<(unsigned)nb, SCAN_T, 0, stream>>>(in, out, n, sums, inclusive);
    PGLB_LAUNCH_CHECK("scan_apply_kernel");
    return PGLB_OK;
}

// ---- key packing / result emission -----------------------------------------------------------
template <typename KeyT, typename ValT>
__global__ void __launch_bounds__(256) pack_keys_kernel(const int64_t *u, int64_t u_stride,
                                                        int64_t E, int64_t N, KeyT *keys, ValT *vals,
                                                        unsigned long long *degree, int *bad) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = u[i * u_stride];
        if ((unsigned long long)k >= (unsigned long long)N) {  // id outside [0, N): report, never index with it
            *bad = 1;
            keys[i] = (KeyT)0;
            vals[i] = (ValT)i;
            continue;
        }
        keys[i] = (KeyT)k;
        vals[i] = (ValT)i;
        atomicAdd(degree + k, 1ull);
    }
}

template <typename KeyT, typename ValT>
__global__ void __launch_bounds__(256) emit_sorted_kernel(const KeyT *keys, const ValT *vals,
                                                          const int64_t *v, int64_t v_stride,
                                                          int64_t E, int64_t *sorted_u,
                                                          int64_t *sorted_v,
                                                          int64_t *sorted_eid) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = (int64_t)vals[i];
        sorted_u[i] = (int64_t)keys[i];
        sorted_eid[i] = e;
        sorted_v[i] = v[e * v_stride];
    }
}

__global__ void set_first_kernel(int64_t *indptr) { indptr[0] = 0; }

static int key_bits(int64_t n) {
    int b = 1;
    while (b < 63 && ((int64_t)1 << b) < n) ++b;
    return b;
}

// ---- stable LSD radix sort of pairs, 8 bits per pass -------------------------------------------
template <typename KeyT>
__device__ __forceinline__ unsigned digit_of(KeyT k, int shift) {
    return (unsigned)((k >> shift) & 0xff);
}

// table[d * nb + b] = number of keys of block b's tile whose current digit is d
template <typename KeyT, int IPW>
__global__ void __launch_bounds__(256) rs_hist_kernel(const KeyT *__restrict__ keys, int64_t n, int shift,
                                                      int64_t nb, int64_t *__restrict__ table) {
    constexpr int TILE = 8 * IPW;
    __shared__ unsigned hist[256];
    hist[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * TILE;
    for (int i = threadIdx.x; i < TILE; i += 256) {
        const int64_t g = base + i;
        if (g < n) atomicAdd(&hist[digit_of(keys[g], shift)], 1u);
    }
    __syncthreads();
    table[(int64_t)threadIdx.x * nb + blockIdx.x] = hist[threadIdx.x];
}

// table has been exclusive-scanned in digit-major order: table[d*nb+b] = first output slot of the
// run of digit d contributed by block b
template <typename KeyT, typename ValT, int IPW>
__global__ void __launch_bounds__(256) rs_scatter_kernel(const KeyT *__restrict__ kin,
                                                         const ValT *__restrict__ vin,
                                                         KeyT *__restrict__ kout, ValT *__restrict__ vout,
                                                         int64_t n, int shift, int64_t nb,
                                                         const int64_t *__restrict__ table) {
    constexpr int TILE = 8 * IPW;
    __shared__ unsigned whist[8][256];  // per-warp digit counts, then running local bases
    __shared__ unsigned bpre[256];      // local position where the block's run of digit d starts
    __shared__ unsigned wsum[8];
    __shared__ int64_t goff[256];
    __shared__ KeyT skey[TILE];
    __shared__ ValT sval[TILE];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int64_t base = (int64_t)blockIdx.x * TILE;
    const int64_t rem = n - base;
    const int cnt = rem < TILE ? (int)rem : TILE;

    for (int i = tid; i < 8 * 256; i += 256) (&whist[0][0])[i] = 0;
    __syncthreads();
    // (a) warp w owns the contiguous items [w*IPW, (w+1)*IPW)
    for (int c = 0; c < IPW; c += 32) {
        const int i = w * IPW + c + lane;
        if (i < cnt) atomicAdd(&whist[w][digit_of(kin[base + i], shift)], 1u);
    }
    __syncthreads();
    // (b) thread d: exclusive prefix over the warps for digit d, then over the digits for the block
    {
        const int d = tid;
        unsigned tot = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned c = whist[j][d];
            whist[j][d] = tot;
            tot += c;
        }
        unsigned incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[w] = incl;
        __syncthreads();
        unsigned wb = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < w) wb += wsum[j];
        bpre[d] = wb + incl - tot;
        goff[d] = table[(int64_t)d * nb + blockIdx.x];
    }
    __syncthreads();
    // (c) every warp walks its sub-tile in order; equal digits inside a 32-item chunk are ranked by
    //     lane, chunks are sequential => stable.  Items land in shared memory grouped by digit.
    for (int c = 0; c < IPW; c += 32) {
        const int i = w * IPW + c + lane;
        const bool valid = i < cnt;
        KeyT k = 0;
        ValT v = 0;
        unsigned d = 0;
        if (valid) {
            k = kin[base + i];
            v = vin[base + i];
            d = digit_of(k, shift);
        }
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const unsigned m = __match_any_sync(act, d);
            const unsigned r = __popc(m & ((1u << lane) - 1u));
            const unsigned lp = bpre[d] + whist[w][d] + r;
            skey[lp] = k;
            sval[lp] = v;
            __syncwarp(act);  // every lane has read whist[w][d] before its leader bumps it
            if (r == 0) whist[w][d] += __popc(m);
        }
        __syncwarp();
    }
    __syncthreads();
    // (d) write out: consecutive local positions of one digit are consecutive global slots
    for (int lp = tid; lp < cnt; lp += 256) {
        const KeyT k = skey[lp];
        const unsigned d = digit_of(k, shift);
        const int64_t g = goff[d] + (int64_t)(lp - bpre[d]);
        kout[g] = k;
        vout[g] = sval[lp];
    }
}

template <typename KeyT>
struct SortGeo {
    static constexpr int kIpw = sizeof(KeyT) == 4 ? 512 : 256;  // tile = 4096 (32-bit) / 2048 (64-bit) pairs
    static constexpr int kTile = 8 * kIpw;
};

struct SortPlan {
    size_t keys_a, keys_b, vals_a, vals_b, table, scan_tmp, bad, total;
    int64_t nb;
};

// The stable LSD pass loop over key bits [0, bits): one histogram, one scan of the digit-major table and one scatter
// per 8-bit digit, ping-ponging between (ka, va) and (kb, vb).  On return ka / va name the buffers holding the result.
// table: 256 * nb int64 with nb = ceil(n / SortGeo<KeyT>::kTile); scan_tmp: scan_ws_bytes(256 * nb).
template <typename KeyT, typename ValT>
static int sort_passes(KeyT *&ka, ValT *&va, KeyT *&kb, ValT *&vb, int64_t n, int64_t nb, int bits, int64_t *table,
                       void *scan_tmp, cudaStream_t stream) {
    constexpr int IPW = SortGeo<KeyT>::kIpw;
    for (int shift = 0; shift < bits; shift += 8) {
        rs_hist_kernel<KeyT, IPW><<<(unsigned)nb, 256, 0, stream>>>(ka, n, shift, nb, table);
        PGLB_LAUNCH_CHECK("rs_hist_kernel");
        const int rc = scan_i64(table, table, 256 * nb, /*inclusive=*/0, scan_tmp, stream);
        if (rc) return rc;
        rs_scatter_kernel<KeyT, ValT, IPW><<<(unsigned)nb, 256, 0, stream>>>(ka, va, kb, vb, n, shift, nb, table);
        PGLB_LAUNCH_CHECK("rs_scatter_kernel");
        std::swap(ka, kb);
        std::swap(va, vb);
    }
    return PGLB_OK;
}

static int64_t sort_blocks_u64(int64_t n) { return (n + SortGeo<uint64_t>::kTile - 1) / SortGeo<uint64_t>::kTile; }

size_t radix_sort_u64_ws_bytes(int64_t n) {
    const int64_t nb = std::max<int64_t>(sort_blocks_u64(n), 1);
    return align_up(sizeof(int64_t) * 256 * (size_t)nb, 256) + scan_ws_bytes(256 * nb);
}

int radix_sort_u64(uint64_t *keys, uint64_t *vals, uint64_t *keys_alt, uint64_t *vals_alt, int64_t n, int bits,
                   void *tmp, cudaStream_t stream, int *result_in_alt) {
    *result_in_alt = 0;
    if (n <= 0) return PGLB_OK;
    const int64_t nb = sort_blocks_u64(n);
    int64_t *table = reinterpret_cast<int64_t *>(tmp);
    void *scan_tmp = reinterpret_cast<char *>(tmp) + align_up(sizeof(int64_t) * 256 * (size_t)nb, 256);
    uint64_t *ka = keys, *va = vals, *kb = keys_alt, *vb = vals_alt;
    const int rc = sort_passes<uint64_t, uint64_t>(ka, va, kb, vb, n, nb, bits, table, scan_tmp, stream);
    *result_in_alt = ka != keys;
    return rc;
}

template <typename KeyT, typename ValT>
static SortPlan plan(int64_t E, int64_t N) {
    SortPlan pl;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t r = off;
        off += align_up(bytes ? bytes : 1, 256);
        return r;
    };
    pl.nb = (E + SortGeo<KeyT>::kTile - 1) / SortGeo<KeyT>::kTile;
    pl.keys_a = take(sizeof(KeyT) * E);
    pl.keys_b = take(sizeof(KeyT) * E);
    pl.vals_a = take(sizeof(ValT) * E);
    pl.vals_b = take(sizeof(ValT) * E);
    pl.table = take(sizeof(int64_t) * 256 * (size_t)std::max<int64_t>(pl.nb, 1));
    const int64_t longest = std::max<int64_t>(256 * std::max<int64_t>(pl.nb, 1), N);
    pl.scan_tmp = take(scan_ws_bytes(longest));
    pl.bad = take(sizeof(int));
    pl.total = off;
    return pl;
}

template <typename KeyT, typename ValT>
static int run(const int64_t *u, int64_t us, const int64_t *v, int64_t vs, int64_t E, int64_t N,
               int64_t *degree, int64_t *indptr, int64_t *su, int64_t *sv, int64_t *se, void *ws,
               size_t ws_bytes, cudaStream_t stream) {
    const SortPlan pl = plan<KeyT, ValT>(E, N);
    PGLB_CHECK_ARG(ws_bytes >= pl.total, PGLB_EWORKSPACE,
                   "pglb_csr_build: workspace of %zu bytes needed (got %zu)", pl.total, ws_bytes);
    char *base = reinterpret_cast<char *>(ws);
    KeyT *ka = reinterpret_cast<KeyT *>(base + pl.keys_a);
    KeyT *kb = reinterpret_cast<KeyT *>(base + pl.keys_b);
    ValT *va = reinterpret_cast<ValT *>(base + pl.vals_a);
    ValT *vb = reinterpret_cast<ValT *>(base + pl.vals_b);
    int64_t *table = reinterpret_cast<int64_t *>(base + pl.table);
    void *scan_tmp = base + pl.scan_tmp;

    PGLB_CUDA(cudaMemsetAsync(degree, 0, sizeof(int64_t) * N, stream));
    const int blocks = (int)std::min<int64_t>((E + 255) / 256, (int64_t)sm_count() * 16);
    if (E > 0) {
        int *bad = reinterpret_cast<int *>(base + pl.bad);
        PGLB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), stream));
        pack_keys_kernel<KeyT, ValT><<<blocks, 256, 0, stream>>>(
            u, us, E, N, ka, va, reinterpret_cast<unsigned long long *>(degree), bad);
        PGLB_LAUNCH_CHECK("pack_keys_kernel");
        // the build is graph preparation (one-off): read the range-check flag back before sorting garbage,
        // and answer like the host twin pglb_build_index_host does (ADVICE r1)
        int bad_h = 0;
        PGLB_CUDA(cudaMemcpyAsync(&bad_h, bad, sizeof(int), cudaMemcpyDeviceToHost, stream));
        PGLB_CUDA(cudaStreamSynchronize(stream));
        PGLB_CHECK_ARG(bad_h == 0, PGLB_ESHAPE, "pglb_csr_build: a node id lies outside [0, %lld)", (long long)N);
    }
    set_first_kernel<<<1, 1, 0, stream>>>(indptr);
    PGLB_LAUNCH_CHECK("set_first_kernel");
    if (N > 0) {
        const int rc = scan_i64(degree, indptr + 1, N, /*inclusive=*/1, scan_tmp, stream);
        if (rc) return rc;
    }
    if (E > 0) {
        const int rc = sort_passes<KeyT, ValT>(ka, va, kb, vb, E, pl.nb, key_bits(N), table, scan_tmp, stream);
        if (rc) return rc;
        emit_sorted_kernel<KeyT, ValT><<<blocks, 256, 0, stream>>>(ka, va, v, vs, E, su, sv, se);
        PGLB_LAUNCH_CHECK("emit_sorted_kernel");
    }
    return PGLB_OK;
}

// ---- segment ids ------------------------------------------------------------------------

// flag[r] = degree(r) > 0 ; then uniq = compaction of rows, seg id of slot j = rank(row(j))
__global__ void __launch_bounds__(256) nonempty_flag_kernel(const int64_t *indptr, int64_t N,
                                                            int64_t *flag) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < N;
         r += (int64_t)gridDim.x * blockDim.x)
        flag[r] = (indptr[r + 1] > indptr[r]) ? 1 : 0;
}

// rank[] is the EXCLUSIVE prefix sum of flag[]
__global__ void __launch_bounds__(256) emit_segments_kernel(const int64_t *indptr,
                                                            const int64_t *rank, int64_t N,
                                                            int64_t *uniq, int64_t *seg,
                                                            int64_t *num_uniq) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < N; r += nwarps) {
        const int64_t b = indptr[r], e = indptr[r + 1];
        if (e > b) {
            const int64_t k = rank[r];
            if (lane == 0) uniq[k] = r;
            for (int64_t j = b + lane; j < e; j += 32) seg[j] = k;
        }
        if (r == N - 1 && lane == 0) *num_uniq = rank[r] + (e > b ? 1 : 0);
    }
}

// sorted ids -> indptr[K+1]: indptr[k] = first slot whose id >= k
__global__ void __launch_bounds__(256) segment_indptr_kernel(const int64_t *ids, int64_t E,
                                                             int64_t K, int64_t *indptr) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= E;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t prev = (i == 0) ? -1 : ids[i - 1];
        const int64_t cur = (i == E) ? K : ids[i];
        for (int64_t k = prev + 1; k <= cur && k <= K; ++k) indptr[k] = i;
    }
}


// ---- plan of the narrow-row aggregation (csrc/spmm_narrow2.inl) ----------------------------------------------
// plan[j] = cols[j] | (slot j starts a row) << 30 ; nz_row[k] = id of the k-th non-empty row (padded with two
// copies of the last one) ; blk_k[b] = k of the row that owns slot 32 b - 1 (-1 for b = 0).
__global__ void __launch_bounds__(256) plan_cols_kernel(const int64_t *__restrict__ cols,
                                                        const uint32_t *__restrict__ packed, int64_t E,
                                                        uint32_t *__restrict__ plan) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    // packed (optional, from pglb_pack_cols): same id with the L2 residency hint in bit 31
    if (j < E) plan[j] = packed ? (packed[j] & 0xbfffffffu) : (uint32_t)cols[j];
}
__global__ void __launch_bounds__(256) plan_rows_kernel(const int64_t *__restrict__ indptr, int64_t N,
                                                        const int64_t *__restrict__ rank,
                                                        uint32_t *__restrict__ plan, int32_t *__restrict__ nz_row) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const int64_t b = indptr[r], e = indptr[r + 1];
    if (e > b) {
        nz_row[rank[r]] = (int32_t)r;
        plan[b] |= 0x40000000u;
    }
    if (r == N - 1) {  // pad: the kernel reads nz_row[k + 1] one row ahead
        const int64_t K = rank[r] + (e > b ? 1 : 0);
        // the last non-empty row is the one that owns the last slot; with K == 0 there is nothing to read
        int64_t last = 0;
        if (K > 0) {
            int64_t lo = 0, hi = N;  // upper_bound(indptr, E - 1) - 1
            const int64_t v = indptr[N] - 1;
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (indptr[mid] > v) hi = mid;
                else lo = mid + 1;
            }
            last = lo - 1;
        }
        nz_row[K] = (int32_t)last;
        nz_row[K + 1] = (int32_t)last;
    }
}
__global__ void __launch_bounds__(256) plan_blocks_kernel(const int64_t *__restrict__ indptr, int64_t N,
                                                          const int64_t *__restrict__ rank, int64_t nblk,
                                                          int32_t *__restrict__ blk_k) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblk) return;
    if (b == 0) {
        blk_k[0] = -1;
        return;
    }
    const int64_t v = b * 32 - 1;  // the slot just before the block: which row owns it?
    int64_t lo = 0, hi = N;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg((const long long *)indptr + mid) > v) hi = mid;
        else lo = mid + 1;
    }
    blk_k[b] = (int32_t)rank[lo - 1];
}

}  // namespace pglb

using namespace pglb;

static bool use_small(int64_t E, int64_t N) { return E < 0xffffffffLL && N < 0xffffffffLL; }

extern "C" int pglb_csr_build_ws(int64_t E, int64_t N, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr, PGLB_EINVAL, "pglb_csr_build_ws: ws_bytes is NULL");
    PGLB_CHECK_ARG(E >= 0 && N >= 0, PGLB_EINVAL, "pglb_csr_build_ws: negative size");
    *ws_bytes = use_small(E, N) ? plan<uint32_t, uint32_t>(E, N).total
                                : plan<uint64_t, uint64_t>(E, N).total;
    return PGLB_OK;
}

extern "C" int pglb_csr_build(const int64_t *u, int64_t u_stride, const int64_t *v,
                              int64_t v_stride, int64_t E, int64_t N, int64_t *degree,
                              int64_t *indptr, int64_t *sorted_u, int64_t *sorted_v,
                              int64_t *sorted_eid, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(E >= 0 && N >= 0, PGLB_EINVAL, "pglb_csr_build: negative size");
    PGLB_CHECK_ARG(indptr != nullptr, PGLB_EINVAL, "pglb_csr_build: indptr is NULL");
    PGLB_CHECK_ARG(N == 0 || degree != nullptr, PGLB_EINVAL, "pglb_csr_build: degree is NULL");
    PGLB_CHECK_ARG(E == 0 || (u && v && sorted_u && sorted_v && sorted_eid), PGLB_EINVAL,
                   "pglb_csr_build: NULL edge pointer");
    PGLB_CHECK_ARG(E == 0 || N > 0, PGLB_ESHAPE, "pglb_csr_build: edges but no nodes");
    PGLB_CHECK_ARG(u_stride >= 1 && v_stride >= 1, PGLB_EINVAL, "pglb_csr_build: bad stride");
    PGLB_CHECK_ARG(ws != nullptr && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0,
                   PGLB_EWORKSPACE, "pglb_csr_build: workspace NULL or not 256-byte aligned");
    if (use_small(E, N))
        return run<uint32_t, uint32_t>(u, u_stride, v, v_stride, E, N, degree, indptr, sorted_u,
                                       sorted_v, sorted_eid, ws, ws_bytes, stream);
    return run<uint64_t, uint64_t>(u, u_stride, v, v_stride, E, N, degree, indptr, sorted_u,
                                   sorted_v, sorted_eid, ws, ws_bytes, stream);
}

extern "C" int pglb_segment_ids_ws(int64_t N, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr && N >= 0, PGLB_EINVAL, "pglb_segment_ids_ws: bad args");
    *ws_bytes = align_up(sizeof(int64_t) * (N ? N : 1), 256) * 2 + scan_ws_bytes(N);
    return PGLB_OK;
}

extern "C" int pglb_segment_ids(const int64_t *indptr, int64_t N, int64_t E, int64_t *uniq_ind,
                                int64_t *segment_ids, int64_t *num_uniq, void *ws,
                                size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(N >= 0 && E >= 0 && num_uniq != nullptr, PGLB_EINVAL,
                   "pglb_segment_ids: bad args");
    if (N == 0) {
        PGLB_CUDA(cudaMemsetAsync(num_uniq, 0, sizeof(int64_t), stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(indptr && uniq_ind && (E == 0 || segment_ids), PGLB_EINVAL,
                   "pglb_segment_ids: NULL pointer");
    size_t need = 0;
    int rc = pglb_segment_ids_ws(N, &need);
    if (rc) return rc;
    PGLB_CHECK_ARG(ws && ws_bytes >= need, PGLB_EWORKSPACE,
                   "pglb_segment_ids: workspace of %zu bytes needed (got %zu)", need, ws_bytes);
    char *base = reinterpret_cast<char *>(ws);
    const size_t a = align_up(sizeof(int64_t) * N, 256);
    int64_t *flag = reinterpret_cast<int64_t *>(base);
    int64_t *rank = reinterpret_cast<int64_t *>(base + a);
    void *tmp = base + 2 * a;
    const int blocks = (int)std::min<int64_t>((N + 255) / 256, (int64_t)sm_count() * 16);
    nonempty_flag_kernel<<<blocks, 256, 0, stream>>>(indptr, N, flag);
    PGLB_LAUNCH_CHECK("nonempty_flag_kernel");
    {
        const int rc2 = scan_i64(flag, rank, N, /*inclusive=*/0, tmp, stream);
        if (rc2) return rc2;
    }
    const int wblocks = (int)std::min<int64_t>((N + 7) / 8, (int64_t)sm_count() * 16);
    emit_segments_kernel<<<wblocks, 256, 0, stream>>>(indptr, rank, N, uniq_ind, segment_ids,
                                                      num_uniq);
    PGLB_LAUNCH_CHECK("emit_segments_kernel");
    return PGLB_OK;
}

extern "C" int pglb_segment_indptr(const int64_t *segment_ids, int64_t E, int64_t K,
                                   int64_t *indptr, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(E >= 0 && K >= 0 && indptr != nullptr, PGLB_EINVAL,
                   "pglb_segment_indptr: bad args");
    PGLB_CHECK_ARG(E == 0 || segment_ids != nullptr, PGLB_EINVAL,
                   "pglb_segment_indptr: segment_ids is NULL");
    const int blocks = (int)std::min<int64_t>((E + 256) / 256, (int64_t)sm_count() * 16);
    segment_indptr_kernel<<<blocks, 256, 0, stream>>>(segment_ids, E, K, indptr);
    PGLB_LAUNCH_CHECK("segment_indptr_kernel");
    return PGLB_OK;
}


extern "C" int pglb_narrow_plan_ws(int64_t N, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes && N >= 0, PGLB_EINVAL, "pglb_narrow_plan_ws: bad argument");
    *ws_bytes = align_up(sizeof(int64_t) * (N ? N : 1), 256) * 2 + scan_ws_bytes(N);
    return PGLB_OK;
}

extern "C" int pglb_narrow_plan(const int64_t *indptr, const int64_t *cols, const uint32_t *cols_packed, int64_t N,
                                int64_t n_src, int64_t E, uint32_t *plan, int32_t *nz_row, int32_t *blk_k, void *ws,
                                size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(N > 0 && E > 0, PGLB_EINVAL, "pglb_narrow_plan: needs at least one row and one slot");
    PGLB_CHECK_ARG(N < 0x7fffffffLL && n_src < 0x40000000LL, PGLB_ESHAPE,
                   "pglb_narrow_plan: needs n_dst < 2^31 and n_src < 2^30");
    PGLB_CHECK_ARG(indptr && cols && plan && nz_row && blk_k, PGLB_EINVAL, "pglb_narrow_plan: NULL pointer");
    size_t need = 0;
    pglb_narrow_plan_ws(N, &need);
    PGLB_CHECK_ARG(ws && ws_bytes >= need, PGLB_EWORKSPACE, "pglb_narrow_plan: workspace of %zu bytes needed (got %zu)",
                   need, ws_bytes);
    char *base = reinterpret_cast<char *>(ws);
    const size_t vec = align_up(sizeof(int64_t) * (size_t)N, 256);
    int64_t *flag = reinterpret_cast<int64_t *>(base);
    int64_t *rank = reinterpret_cast<int64_t *>(base + vec);
    void *tmp = base + 2 * vec;
    nonempty_flag_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(indptr, N, flag);
    PGLB_LAUNCH_CHECK("nonempty_flag_kernel");
    const int rc = scan_i64(flag, rank, N, /*inclusive=*/0, tmp, stream);
    if (rc) return rc;
    plan_cols_kernel<<<(unsigned)((E + 255) / 256), 256, 0, stream>>>(cols, cols_packed, E, plan);
    PGLB_LAUNCH_CHECK("plan_cols_kernel");
    plan_rows_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(indptr, N, rank, plan, nz_row);
    PGLB_LAUNCH_CHECK("plan_rows_kernel");
    const int64_t nblk = (E + 31) / 32;
    plan_blocks_kernel<<<(unsigned)((nblk + 255) / 256), 256, 0, stream>>>(indptr, N, rank, nblk, blk_k);
    PGLB_LAUNCH_CHECK("plan_blocks_kernel");
    return PGLB_OK;
}
