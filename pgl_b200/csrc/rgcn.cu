// rgcn.cu -- RGCNConv's relation-typed aggregation (reference pgl/nn/conv.py:998-1024,
//     out = sum_r mean_r(x W_r)   reassociated as   out[d] = sum_r A_r[d] W_r,
//     A_r[d] = mean over the r-run of row d of x[src]  (0 when the run is empty))
// on a typed CSR: the slots of every row are grouped by relation in ascending relation id (ascending eid inside a
// group), so a row's r-run is one contiguous slot range.
//
// rgcn_agg_kernel: a persistent CTA per 64-row tile.  For every relation present in the tile it gathers each row's
// run into a shared [64, K] A tile (a warp per row, slots in order), stages W_r [K, N] in shared memory, and adds
// A W_r into register accumulators with 3xTF32 products (linear_tc.cu's accuracy contract); [64, N] is written once.
// Relations absent from the tile cost nothing: the next relation is the least relation id at the rows' cursors.
// With per-slot weights the same kernel is grad x on the typed src-CSR: gx[s] = sum_r (sum_j w_j g[dst_j]) W_r^T.
//
// rgcn_wgrad_kernel: gW_r = sum over the runs p of r of A_p^T g[row_p], over the run list sorted by relation.  A run
// list chunk of one relation is one work item; each item writes its own fp32 [D, O] partial, and rgcn_wsum_kernel
// adds a relation's partials in item order.  No floating-point atomics anywhere: results are bit-identical run to run.
#include <limits.h>

#include <algorithm>

#include "common.cuh"

namespace pglb {

constexpr int RG_ROWS = 64;          // rows per tile: 4 row blocks of 16
constexpr int RG_WARPS = 8;          // 4 row blocks x 2 column groups
constexpr int RG_THREADS = RG_WARPS * 32;
constexpr int RG_KMAX = 128;
constexpr int RG_AS = RG_KMAX + 4;   // A tile stride (floats): 132 = 4 mod 32 -> conflict-free A fragment loads
constexpr int RG_RUNS = 64;          // runs per k-step of the weight gradient

// sum over slots [j0, j1) of w_j x[cols[j]] in slot order (w_j = 1 without slot_w); the lane owns float4 column
// `lane` (lane < kq).  Four rows are loaded before they are added, in order.
__device__ __forceinline__ float4 run_sum(const int64_t *__restrict__ cols, const float *__restrict__ slot_w,
                                          const float *__restrict__ x, int64_t ldx, int64_t j0, int64_t j1, int lane,
                                          int kq) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t base = j0; base < j1; base += 32) {
        const int n = (int)min((int64_t)32, j1 - base);
        int64_t c = 0;
        float w = 1.f;
        if (lane < n) {
            c = __ldg((const long long *)cols + base + lane);
            if (slot_w) w = __ldg(slot_w + base + lane);
        }
        int i = 0;
        for (; i + 4 <= n; i += 4) {
            float4 v[4];
            float wi[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int64_t ci = __shfl_sync(0xffffffffu, c, i + u);
                wi[u] = __shfl_sync(0xffffffffu, w, i + u);
                v[u] = lane < kq ? __ldg(reinterpret_cast<const float4 *>(x + ci * ldx) + lane)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                acc.x = fmaf(wi[u], v[u].x, acc.x);
                acc.y = fmaf(wi[u], v[u].y, acc.y);
                acc.z = fmaf(wi[u], v[u].z, acc.z);
                acc.w = fmaf(wi[u], v[u].w, acc.w);
            }
        }
        for (; i < n; ++i) {
            const int64_t ci = __shfl_sync(0xffffffffu, c, i);
            const float wi = __shfl_sync(0xffffffffu, w, i);
            if (lane < kq) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(x + ci * ldx) + lane);
                acc.x = fmaf(wi, v.x, acc.x);
                acc.y = fmaf(wi, v.y, acc.y);
                acc.z = fmaf(wi, v.z, acc.z);
                acc.w = fmaf(wi, v.w, acc.w);
            }
        }
    }
    return acc;
}

__device__ __forceinline__ float4 div4(float4 a, float d) {
    return make_float4(a.x / d, a.y / d, a.z / d, a.w / d);
}

// acc[16 x 8 NT] += A[16 x K8] B[K8 x 8 NT], 3xTF32.  A(m, k) = A[m * am + k * ak], B(k, n) = B[k * bk + n];
// fragments as linear_tc.cu (a: rows g, g+8 x cols t, t+4; b: rows t, t+4 x col g).
template <int NT>
__device__ __forceinline__ void mma3_block(float (&acc)[NT][4], const float *A, int am, int ak, const float *B, int bk,
                                           int K8, int g, int t) {
    for (int k0 = 0; k0 < K8; k0 += 8) {
        float af[4];
        af[0] = A[g * am + (k0 + t) * ak];
        af[1] = A[(g + 8) * am + (k0 + t) * ak];
        af[2] = A[g * am + (k0 + t + 4) * ak];
        af[3] = A[(g + 8) * am + (k0 + t + 4) * ak];
        uint32_t ahi[4], alo[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            ahi[i] = to_tf32(af[i]);
            alo[i] = to_tf32(af[i] - __uint_as_float(ahi[i]));
        }
        const float *b0p = B + (k0 + t) * bk + g;
        const float *b1p = b0p + 4 * bk;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const float f0 = b0p[j * 8], f1 = b1p[j * 8];
            const uint32_t h0 = to_tf32(f0), h1 = to_tf32(f1);
            const uint32_t l0 = to_tf32(f0 - __uint_as_float(h0)), l1 = to_tf32(f1 - __uint_as_float(h1));
            mma_tf32(acc[j], alo, h0, h1);
            mma_tf32(acc[j], ahi, l0, l1);
            mma_tf32(acc[j], ahi, h0, h1);
        }
    }
}

// NP: output width padded to 32, 64 or 128.  Dynamic shared memory: Ws [RG_KMAX][NP + 8] fp32 (rows >= K and
// columns >= N zero), As [RG_ROWS][RG_AS] fp32 (columns >= K zero).
template <int NP>
__global__ void __launch_bounds__(RG_THREADS, 2)
rgcn_agg_kernel(const int64_t *__restrict__ indptr, const int64_t *__restrict__ cols, const int16_t *__restrict__ rel,
                const float *__restrict__ slot_w, const float *__restrict__ x, int64_t ldx,
                const float *__restrict__ w, int K, int N, float *__restrict__ out, int64_t ldo, int64_t n_rows) {
    constexpr int WS = NP + 8;       // = 8 mod 32 -> conflict-free B fragment loads
    constexpr int NT = NP / 16;      // 8-wide column tiles per warp (2 column groups)
    extern __shared__ __align__(16) float rg_smem[];
    float *Ws = rg_smem;
    float *As = rg_smem + RG_KMAX * WS;
    __shared__ int64_t s_cur[RG_ROWS], s_end[RG_ROWS];
    __shared__ int s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int K8 = (K + 7) & ~7, kq = K >> 2;
    for (int i = tid; i < RG_KMAX * WS; i += RG_THREADS) Ws[i] = 0.f;
    for (int i = tid; i < RG_ROWS * RG_AS; i += RG_THREADS) As[i] = 0.f;

    const int64_t tiles = (n_rows + RG_ROWS - 1) / RG_ROWS;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t r0 = tile * RG_ROWS;
        for (int i = tid; i < RG_ROWS; i += RG_THREADS) {
            const int64_t row = r0 + i;
            s_cur[i] = row < n_rows ? indptr[row] : 0;
            s_end[i] = row < n_rows ? indptr[row + 1] : 0;
        }
        float acc[NT][4];
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        __syncthreads();
        for (;;) {
            if (tid == 0) s_next = INT_MAX;
            __syncthreads();
            for (int i = tid; i < RG_ROWS; i += RG_THREADS)
                if (s_cur[i] < s_end[i]) atomicMin(&s_next, (int)rel[s_cur[i]]);
            __syncthreads();
            const int r = s_next;
            if (r == INT_MAX) break;
            for (int i = warp; i < RG_ROWS; i += RG_WARPS) {
                const int64_t j0 = s_cur[i], e = s_end[i];
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                if (j0 < e && rel[j0] == r) {
                    int64_t j1 = j0;
                    for (;;) {   // end of the r-run: rel is ascending inside the row
                        const int64_t idx = j1 + lane;
                        const unsigned in = __ballot_sync(0xffffffffu, idx < e && rel[idx] == r);
                        if (in != 0xffffffffu) {
                            j1 += __ffs(~in) - 1;
                            break;
                        }
                        j1 += 32;
                    }
                    a = run_sum(cols, slot_w, x, ldx, j0, j1, lane, kq);
                    if (!slot_w) a = div4(a, (float)(j1 - j0));
                    __syncwarp();
                    if (lane == 0) s_cur[i] = j1;
                }
                if (lane < kq) *reinterpret_cast<float4 *>(As + i * RG_AS + 4 * lane) = a;
            }
            const float *wr = w + (int64_t)r * K * N;
            for (int i = tid; i < K * N; i += RG_THREADS) {
                const int k = i / N, n = i - k * N;
                Ws[k * WS + n] = __ldg(wr + i);
            }
            __syncthreads();
            mma3_block<NT>(acc, As + wm * 16 * RG_AS, RG_AS, 1, Ws + wn * (NP / 2), WS, K8, g, t);
            __syncthreads();
        }
        // c0, c1 -> (row g, cols 2t, 2t+1); c2, c3 -> row g + 8
        const int64_t row0 = r0 + wm * 16 + g;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int col = wn * (NP / 2) + j * 8 + 2 * t;
            if (col < N) {   // N % 4 == 0: col < N implies col + 1 < N
                if (row0 < n_rows) *reinterpret_cast<float2 *>(out + row0 * ldo + col) = make_float2(acc[j][0], acc[j][1]);
                if (row0 + 8 < n_rows)
                    *reinterpret_cast<float2 *>(out + (row0 + 8) * ldo + col) = make_float2(acc[j][2], acc[j][3]);
            }
        }
    }
}

// DP: D padded to 64 or 128 (rows of gW), NP: O padded to 32, 64 or 128.  Warp (wm, wn) owns rows
// [wm DP/4, (wm+1) DP/4) and columns [wn NP/2, (wn+1) NP/2).  Dynamic shared memory: As [RG_RUNS][DP + 8] (A_p^T
// stored run-major: A(m, k) = As[k][m]) and Gs [RG_RUNS][NP + 8], both zero outside the live runs / columns.
template <int DP, int NP>
__global__ void __launch_bounds__(RG_THREADS, 2)
rgcn_wgrad_kernel(const int64_t *__restrict__ run_row, const int64_t *__restrict__ run_beg,
                  const int64_t *__restrict__ run_end, const int64_t *__restrict__ run_off,
                  const int64_t *__restrict__ item_off, int R, int64_t n_items, int64_t chunk,
                  const int64_t *__restrict__ cols, const float *__restrict__ x, int64_t ldx,
                  const float *__restrict__ gr, int64_t ldg, int D, int O, float *__restrict__ partial) {
    constexpr int SA = DP + 8, SB = NP + 8;   // = 8 mod 32: conflict-free fragment loads
    constexpr int MT = DP / 64, NT = NP / 16;
    extern __shared__ __align__(16) float rg_smem[];
    float *As = rg_smem;
    float *Gs = rg_smem + RG_RUNS * SA;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int dq = D >> 2, oq = O >> 2;
    for (int i = tid; i < RG_RUNS * SA; i += RG_THREADS) As[i] = 0.f;
    for (int i = tid; i < RG_RUNS * SB; i += RG_THREADS) Gs[i] = 0.f;
    __syncthreads();

    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        int lo = 0, hi = R;   // the relation r with item_off[r] <= item < item_off[r + 1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (item_off[mid] <= item) lo = mid;
            else hi = mid;
        }
        const int64_t k0 = run_off[lo] + (item - item_off[lo]) * chunk;
        const int64_t k1 = min(k0 + chunk, run_off[lo + 1]);
        float acc[MT][NT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int j = 0; j < NT; ++j) acc[m][j][0] = acc[m][j][1] = acc[m][j][2] = acc[m][j][3] = 0.f;
        for (int64_t kb = k0; kb < k1; kb += RG_RUNS) {
            const int nk = (int)min((int64_t)RG_RUNS, k1 - kb);
            for (int i = warp; i < RG_RUNS; i += RG_WARPS) {
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f), gv = a;
                if (i < nk) {
                    const int64_t p = kb + i;
                    const int64_t j0 = run_beg[p], j1 = run_end[p];
                    a = div4(run_sum(cols, nullptr, x, ldx, j0, j1, lane, dq), (float)(j1 - j0));
                    if (lane < oq) gv = __ldg(reinterpret_cast<const float4 *>(gr + run_row[p] * ldg) + lane);
                }
                if (lane < dq) *reinterpret_cast<float4 *>(As + i * SA + 4 * lane) = a;
                if (lane < oq) *reinterpret_cast<float4 *>(Gs + i * SB + 4 * lane) = gv;
            }
            __syncthreads();
#pragma unroll
            for (int m = 0; m < MT; ++m)
                mma3_block<NT>(acc[m], As + wm * (DP / 4) + m * 16, 1, SA, Gs + wn * (NP / 2), SB, RG_RUNS, g, t);
            __syncthreads();
        }
        float *pt = partial + item * (int64_t)D * O;
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const int row0 = wm * (DP / 4) + m * 16 + g;
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const int col = wn * (NP / 2) + j * 8 + 2 * t;
                if (col < O) {
                    if (row0 < D) *reinterpret_cast<float2 *>(pt + (int64_t)row0 * O + col) = make_float2(acc[m][j][0], acc[m][j][1]);
                    if (row0 + 8 < D)
                        *reinterpret_cast<float2 *>(pt + (int64_t)(row0 + 8) * O + col) = make_float2(acc[m][j][2], acc[m][j][3]);
                }
            }
        }
    }
}

// gW[r] = sum of relation r's partials in item order (0 for a relation without runs)
__global__ void rgcn_wsum_kernel(const float *__restrict__ partial, const int64_t *__restrict__ item_off, int R,
                                 int64_t DO, float *__restrict__ gw) {
    const int64_t total = (int64_t)R * DO;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / DO, e = i - r * DO;
        float s = 0.f;
        for (int64_t p = item_off[r]; p < item_off[r + 1]; ++p) s += partial[p * DO + e];
        gw[i] = s;
    }
}

static int pad_width(int n) { return n <= 32 ? 32 : n <= 64 ? 64 : 128; }

template <int NP>
static int agg_launch(const int64_t *indptr, const int64_t *cols, const int16_t *rel, const float *slot_w,
                      const float *x, int64_t ldx, const float *w, int K, int N, float *out, int64_t ldo,
                      int64_t n_rows, cudaStream_t s) {
    const size_t smem = sizeof(float) * ((size_t)RG_KMAX * (NP + 8) + (size_t)RG_ROWS * RG_AS);
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(rgcn_agg_kernel<NP>, (int)smem, attr_done));
    const int64_t tiles = (n_rows + RG_ROWS - 1) / RG_ROWS;
    const unsigned grid = (unsigned)std::min<int64_t>(tiles, 2 * (int64_t)sm_count());
    rgcn_agg_kernel<NP><<<grid, RG_THREADS, smem, s>>>(indptr, cols, rel, slot_w, x, ldx, w, K, N, out, ldo, n_rows);
    PGLB_LAUNCH_CHECK("rgcn_agg_kernel");
    return PGLB_OK;
}

template <int DP, int NP>
static int wgrad_launch(const int64_t *run_row, const int64_t *run_beg, const int64_t *run_end,
                        const int64_t *run_off, const int64_t *item_off, int R, int64_t n_items, int64_t chunk,
                        const int64_t *cols, const float *x, int64_t ldx, const float *gr, int64_t ldg, int D, int O,
                        float *partial, cudaStream_t s) {
    const size_t smem = sizeof(float) * (size_t)RG_RUNS * ((DP + 8) + (NP + 8));
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(rgcn_wgrad_kernel<DP, NP>, (int)smem, attr_done));
    const unsigned grid = (unsigned)std::min<int64_t>(n_items, 2 * (int64_t)sm_count());
    rgcn_wgrad_kernel<DP, NP><<<grid, RG_THREADS, smem, s>>>(run_row, run_beg, run_end, run_off, item_off, R, n_items,
                                                             chunk, cols, x, ldx, gr, ldg, D, O, partial);
    PGLB_LAUNCH_CHECK("rgcn_wgrad_kernel");
    return PGLB_OK;
}

static bool width_ok(int64_t v) { return v >= 4 && v <= RG_KMAX && v % 4 == 0; }

}  // namespace pglb

extern "C" int pglb_rgcn_agg_f32(const int64_t *indptr, const int64_t *cols, const int16_t *rel, const float *slot_w,
                                 const float *x, int64_t ldx, const float *weight, int64_t num_rels, int64_t K,
                                 int64_t N, float *out, int64_t ldo, int64_t n_rows, void *stream) {
    using namespace pglb;
    PGLB_CHECK_ARG(n_rows >= 0 && num_rels >= 1 && num_rels <= 32767, PGLB_EINVAL,
                   "pglb_rgcn_agg_f32: n_rows must be >= 0 and num_rels in [1, 32767]");
    PGLB_CHECK_ARG(width_ok(K) && width_ok(N), PGLB_EINVAL,
                   "pglb_rgcn_agg_f32: K and N must be multiples of 4 in [4, 128] (got %lld, %lld)", (long long)K,
                   (long long)N);
    PGLB_CHECK_ARG(ldx >= K && ldx % 4 == 0 && ldo >= N && ldo % 2 == 0, PGLB_EINVAL,
                   "pglb_rgcn_agg_f32: ldx must be >= K and a multiple of 4, ldo >= N and even");
    if (n_rows == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && cols && rel && x && weight && out, PGLB_EINVAL, "pglb_rgcn_agg_f32: NULL pointer");
    PGLB_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 8) == 0 && ((uintptr_t)weight % 4) == 0,
                   PGLB_EINVAL, "pglb_rgcn_agg_f32: x must be 16-byte and out 8-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int k = (int)K, n = (int)N;
    switch (pad_width(n)) {
        case 32: return agg_launch<32>(indptr, cols, rel, slot_w, x, ldx, weight, k, n, out, ldo, n_rows, s);
        case 64: return agg_launch<64>(indptr, cols, rel, slot_w, x, ldx, weight, k, n, out, ldo, n_rows, s);
        default: return agg_launch<128>(indptr, cols, rel, slot_w, x, ldx, weight, k, n, out, ldo, n_rows, s);
    }
}

extern "C" int pglb_rgcn_wgrad_ws(int64_t n_items, int64_t D, int64_t O, size_t *ws_bytes) {
    using namespace pglb;
    PGLB_CHECK_ARG(ws_bytes && n_items >= 0 && width_ok(D) && width_ok(O), PGLB_EINVAL,
                   "pglb_rgcn_wgrad_ws: bad arguments");
    *ws_bytes = align_up(sizeof(float) * (size_t)n_items * (size_t)D * (size_t)O, 256);
    return PGLB_OK;
}

extern "C" int pglb_rgcn_wgrad_f32(const int64_t *run_row, const int64_t *run_beg, const int64_t *run_end,
                                   const int64_t *run_off, const int64_t *item_off, int64_t num_rels, int64_t n_items,
                                   int64_t chunk, const int64_t *cols, const float *x, int64_t ldx,
                                   const float *grad_out, int64_t ldg, int64_t D, int64_t O, float *grad_weight,
                                   void *ws, size_t ws_bytes, void *stream) {
    using namespace pglb;
    PGLB_CHECK_ARG(num_rels >= 1 && num_rels <= 32767 && n_items >= 0 && chunk >= 1, PGLB_EINVAL,
                   "pglb_rgcn_wgrad_f32: num_rels must lie in [1, 32767], n_items >= 0, chunk >= 1");
    PGLB_CHECK_ARG(width_ok(D) && width_ok(O), PGLB_EINVAL,
                   "pglb_rgcn_wgrad_f32: D and O must be multiples of 4 in [4, 128] (got %lld, %lld)", (long long)D,
                   (long long)O);
    PGLB_CHECK_ARG(ldx >= D && ldx % 4 == 0 && ldg >= O && ldg % 4 == 0, PGLB_EINVAL,
                   "pglb_rgcn_wgrad_f32: ldx must be >= D, ldg >= O, both multiples of 4");
    PGLB_CHECK_ARG(run_off && item_off && grad_weight, PGLB_EINVAL, "pglb_rgcn_wgrad_f32: NULL pointer");
    PGLB_CHECK_ARG(n_items == 0 || (run_row && run_beg && run_end && cols && x && grad_out), PGLB_EINVAL,
                   "pglb_rgcn_wgrad_f32: NULL pointer");
    PGLB_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)grad_out % 16) == 0 && ((uintptr_t)grad_weight % 4) == 0,
                   PGLB_EINVAL, "pglb_rgcn_wgrad_f32: x and grad_out must be 16-byte aligned");
    const size_t need = sizeof(float) * (size_t)n_items * (size_t)D * (size_t)O;
    PGLB_CHECK_ARG(n_items == 0 || (ws && ws_bytes >= need && ((uintptr_t)ws % 16) == 0), PGLB_EINVAL,
                   "pglb_rgcn_wgrad_f32: workspace smaller than pglb_rgcn_wgrad_ws or not 16-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    float *partial = static_cast<float *>(ws);
    const int d = (int)D, o = (int)O, r = (int)num_rels;
    if (n_items > 0) {
        int rc;
        const int dp = d <= 64 ? 64 : 128, np = pad_width(o);
#define PGLB_WG(DP_, NP_)                                                                                           \
    rc = wgrad_launch<DP_, NP_>(run_row, run_beg, run_end, run_off, item_off, r, n_items, chunk, cols, x, ldx, grad_out, \
                                ldg, d, o, partial, s)
        if (dp == 64) {
            if (np == 32) PGLB_WG(64, 32);
            else if (np == 64) PGLB_WG(64, 64);
            else PGLB_WG(64, 128);
        } else {
            if (np == 32) PGLB_WG(128, 32);
            else if (np == 64) PGLB_WG(128, 64);
            else PGLB_WG(128, 128);
        }
#undef PGLB_WG
        if (rc != PGLB_OK) return rc;
    }
    const int64_t total = (int64_t)r * d * o;
    const unsigned grid = (unsigned)std::min<int64_t>((total + 255) / 256, 8 * (int64_t)sm_count());
    rgcn_wsum_kernel<<<grid, 256, 0, s>>>(partial, item_off, r, (int64_t)d * o, grad_weight);
    PGLB_LAUNCH_CHECK("rgcn_wsum_kernel");
    return PGLB_OK;
}
