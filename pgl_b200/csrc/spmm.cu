// spmm.cu -- node-parallel CSR aggregation for sm_90a (K1 send_u_recv, K2 send_ue_recv,
// K4 segment_* of SURVEY.md section 2.2).
//
// Design (DESIGN.md section 4.2):
//  * a "group" of G lanes (G = 4..32, one float4 or float per lane per iteration) owns a
//    task of `rpg` consecutive dst rows; the rows' slots are one contiguous range of the CSR,
//    so column indices are fetched G at a time with one coalesced streaming load and
//    broadcast by shuffle; U independent feature-row loads (U*ITERS = 8 x 16 B per lane)
//    are issued before the first add, so every group keeps >= 4 KB of gathers in flight
//    regardless of how short the individual rows are.
//  * accumulation is strictly sequential in slot order (= ascending edge id inside a row,
//    the order of the reference's CPU loop), with __fadd_rn/__fmul_rn so that no FMA
//    contraction changes the rounding: results are bit-identical to the sequential
//    restatement for every row below the hub threshold.
//  * rows longer than HUB_T slots ("hubs": ~4k rows holding ~18 % of the edges of the
//    10M/100M power-law graph) are not processed by the row's owner: they are appended to a
//    device-side list, cut into CH-slot chunks by a one-block planning kernel, and the SAME
//    kernel is re-launched twice over "virtual rows" (chunk -> partial, partials -> row).
//    No atomics on feature data, fixed chunking => deterministic run to run.
#include <cfloat>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "common.cuh"

namespace pglb {

constexpr int64_t HUB_T = 1024;  // rows with more slots than this take the hub path
constexpr int64_t HUB_CH = 1024; // slots per hub chunk
constexpr int kThreads = 256;

struct SpmmP {
    const int64_t *rbeg;  // row r covers slots [rbeg[r], rend[r])
    const int64_t *rend;
    const int64_t *cols;  // nullable: identity
    const int64_t *eid;   // nullable: identity (only read when y != nullptr)
    const float *x;
    int64_t ldx;
    const float *y;
    int64_t ldy;
    int y_bcast;
    float *out;
    int64_t ldo;
    int64_t n_rows;
    const int64_t *n_rows_dev;  // nullable: overrides n_rows (hub passes)
    int D;
    int head_dim;
    int msg_op;
    int reduce_op;
    const float *scale_src;
    const float *scale_dst;
    const int64_t *row_map;      // nullable: out row = row_map[row]
    const int64_t *mean_indptr;  // nullable: MEAN divides by mean_indptr[o+1]-mean_indptr[o]
    int rpg;                     // rows per group task
    int contig;                  // 1: rows of a task are contiguous in slot space
    int64_t hub_threshold;
    unsigned long long *hub_count;
    int64_t *hub_rows;
    int accumulate;  // SUM only: add the previous contents of out before the row epilogue
    PropEpi epi;     // PROP kernels only (copy sum, float32)
};

template <int VEC>
struct VecIO;
template <>
struct VecIO<4> {
    static __device__ __forceinline__ void ld(const float *p, float (&v)[4]) {
        float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void st(float *p, const float (&v)[4]) {
        __stcs(reinterpret_cast<float4 *>(p), make_float4(v[0], v[1], v[2], v[3]));
    }
    // 16-bit elements: 8 bytes per lane
    template <typename T>
    static __device__ __forceinline__ void ld(const T *p, float (&v)[4]) {
        const float4 t = widen4<T>(__ldg(reinterpret_cast<const uint2 *>(p)));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    template <typename T>
    static __device__ __forceinline__ void st(T *p, const float (&v)[4]) {
        __stcs(reinterpret_cast<uint2 *>(p), round4<T>(make_float4(v[0], v[1], v[2], v[3])));
    }
};
template <>
struct VecIO<1> {
    static __device__ __forceinline__ void ld(const float *p, float (&v)[1]) { v[0] = __ldg(p); }
    static __device__ __forceinline__ void st(float *p, const float (&v)[1]) { __stcs(p, v[0]); }
    template <typename T>
    static __device__ __forceinline__ void ld(const T *p, float (&v)[1]) {
        v[0] = X16<T>::widen(__ldg(reinterpret_cast<const unsigned short *>(p)));
    }
    template <typename T>
    static __device__ __forceinline__ void st(T *p, const float (&v)[1]) {
        __stcs(reinterpret_cast<unsigned short *>(p), X16<T>::round(v[0]));
    }
};

__device__ __forceinline__ float apply_msg(int op, float a, float b) {
    switch (op) {
        case PGLB_MSG_ADD: return __fadd_rn(a, b);
        case PGLB_MSG_SUB: return __fsub_rn(a, b);
        case PGLB_MSG_MUL: return __fmul_rn(a, b);
        case PGLB_MSG_DIV: return __fdiv_rn(a, b);
        default: return a;
    }
}

// MODE 0: msg = x[col] (* scale_src);  MODE 1: msg = (x[col] (* scale_src)) op y[eid]
// RK 0: sum / mean;  RK 1: max / min
// TI / TO: element type of p.x / p.out (float, or the 16-bit type of pglb_spmm_csr_x16; its hub pass 1 writes fp32
// partials and pass 2 reads them).  Messages are widened to fp32 on load, and each output is rounded once on store.
// PROP (TI = TO = float, copy sum): the row closes with p.epi's epilogue (pglb_propagate_f32).
template <typename TI, typename TO, int VEC, int G, int ITERS, int MODE, int RK, bool PROP = false>
__device__ __forceinline__ void spmm_csr_body(const SpmmP &p) {
    constexpr int U = (8 / ITERS) < G ? (8 / ITERS) : G;
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
    const int64_t groups_per_block = kThreads / G;
    const int64_t gid = (int64_t)blockIdx.x * groups_per_block + threadIdx.x / G;
    const int64_t ngroups = (int64_t)gridDim.x * groups_per_block;
    const int64_t n_rows = p.n_rows_dev ? *p.n_rows_dev : p.n_rows;
    const int col_tile = blockIdx.y * (G * VEC * ITERS);
    const bool is_max = (p.reduce_op == PGLB_REDUCE_MAX);
    const float ident = (RK == 0) ? 0.0f : (is_max ? -INFINITY : INFINITY);

    int col[ITERS];
    bool act[ITERS];
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        col[it] = col_tile + (it * G + gl) * VEC;
        act[it] = col[it] < p.D;
    }

    for (int64_t task = gid; task * p.rpg < n_rows; task += ngroups) {
        int64_t row = task * p.rpg;
        int64_t row_end = row + p.rpg;
        if (row_end > n_rows) row_end = n_rows;
        const int64_t task_end = p.contig ? ld_ro(p.rend + row_end - 1) : 0;

        float acc[ITERS][VEC];
        int64_t pos = 0, cur_beg = 0, cur_end = 0;
        bool hub = false;

        auto open_row = [&]() {
            cur_beg = ld_ro(p.rbeg + row);
            cur_end = ld_ro(p.rend + row);
            pos = cur_beg;
            hub = (cur_end - cur_beg) > p.hub_threshold;
            if (hub && gl == 0 && blockIdx.y == 0) {
                unsigned long long s = atomicAdd(p.hub_count, 1ull);
                p.hub_rows[s] = row;
            }
#pragma unroll
            for (int it = 0; it < ITERS; ++it)
#pragma unroll
                for (int j = 0; j < VEC; ++j) acc[it][j] = ident;
        };
        auto close_row = [&]() {
            if (hub) return;
            const int64_t orow = p.row_map ? ld_ro(p.row_map + row) : row;
            const int64_t deg = cur_end - cur_beg;
            float inv_cnt = 1.0f;
            if (p.reduce_op == PGLB_REDUCE_MEAN) {
                int64_t cnt = p.mean_indptr
                                  ? (ld_ro(p.mean_indptr + orow + 1) - ld_ro(p.mean_indptr + orow))
                                  : deg;
                inv_cnt = (float)cnt;
            }
            const float sd = p.scale_dst ? __ldg(p.scale_dst + orow) : 1.0f;
            if constexpr (PROP) {
                const float cc = prop_c(p.epi);
#pragma unroll
                for (int it = 0; it < ITERS; ++it) {
                    if (!act[it]) continue;
                    float t[VEC], hv[VEC], y[VEC];
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        float a = acc[it][j];
                        if (deg == 0) a = 0.0f;
                        if (p.scale_dst) a = __fmul_rn(a, sd);
                        t[j] = a;
                        hv[j] = a;
                    }
                    if (p.epi.h) VecIO<VEC>::ld(p.epi.h + orow * p.epi.ldh + col[it], hv);
#pragma unroll
                    for (int j = 0; j < VEC; ++j) y[j] = prop_y(p.epi, t[j], hv[j]);
                    VecIO<VEC>::st(p.out + orow * p.ldo + col[it], y);
                    if (p.epi.acc_out) {
                        // plain loads: in place, acc_in is the row this thread is about to overwrite
                        const float *ai = p.epi.acc_in + orow * p.epi.ld_acc_in + col[it];
                        float ao[VEC];
                        if constexpr (VEC == 4) {
                            const float4 v = *reinterpret_cast<const float4 *>(ai);
                            ao[0] = v.x; ao[1] = v.y; ao[2] = v.z; ao[3] = v.w;
                        } else {
                            ao[0] = *ai;
                        }
#pragma unroll
                        for (int j = 0; j < VEC; ++j) ao[j] = __fadd_rn(ao[j], __fmul_rn(cc, y[j]));
                        VecIO<VEC>::st(p.epi.acc_out + orow * p.epi.ld_acc_out + col[it], ao);
                    }
                }
            } else {
#pragma unroll
                for (int it = 0; it < ITERS; ++it) {
                    if (!act[it]) continue;
                    float v[VEC];
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        float a = acc[it][j];
                        if (deg == 0) a = 0.0f;
                        if (sizeof(TO) == 4 && p.accumulate) a = __fadd_rn(p.out[orow * p.ldo + col[it] + j], a);
                        if (p.reduce_op == PGLB_REDUCE_MEAN && deg != 0) a = __fdiv_rn(a, inv_cnt);
                        if (p.scale_dst) a = __fmul_rn(a, sd);
                        v[j] = a;
                    }
                    VecIO<VEC>::st(reinterpret_cast<TO *>(p.out) + orow * p.ldo + col[it], v);
                }
            }
        };

        open_row();
        for (;;) {
            if (hub || pos == cur_end) {
                close_row();
                ++row;
                if (row == row_end) break;
                open_row();
                continue;
            }
            const int64_t lim = p.contig ? task_end : cur_end;
            const int64_t rem = lim - pos;
            const int nb = rem < (int64_t)G ? (int)rem : G;
            int64_t my_col = 0, my_e = 0;
            if (gl < nb) {
                my_col = p.cols ? ld_stream(p.cols + pos + gl) : (pos + gl);
                if (MODE == 1) my_e = p.eid ? ld_stream(p.eid + pos + gl) : (pos + gl);
            }
            bool abandon = false;
            for (int k0 = 0; k0 < nb && !abandon; k0 += U) {
                float xv[U][ITERS][VEC];
                float yv[MODE == 1 ? U : 1][ITERS][VEC];
                float sv[U];
                // ---- phase A: issue every load of this sub-batch ----
#pragma unroll
                for (int k = 0; k < U; ++k) {
                    const int64_t c = __shfl_sync(gmask, my_col, k0 + k, G);
                    int64_t e = 0;
                    if (MODE == 1) e = __shfl_sync(gmask, my_e, k0 + k, G);
                    if (k0 + k < nb) {
                        const TI *xr = reinterpret_cast<const TI *>(p.x) + c * p.ldx;
#pragma unroll
                        for (int it = 0; it < ITERS; ++it) {
                            if (act[it]) VecIO<VEC>::ld(xr + col[it], xv[k][it]);
                        }
                        if (p.scale_src) sv[k] = __ldg(p.scale_src + c);
                        if (MODE == 1) {
                            const float *yr = p.y + e * p.ldy;
#pragma unroll
                            for (int it = 0; it < ITERS; ++it) {
                                if (!act[it]) continue;
                                if (p.y_bcast == PGLB_BCAST_FULL) {
                                    VecIO<VEC>::ld(yr + col[it], yv[k][it]);
                                } else if (p.y_bcast == PGLB_BCAST_HEAD) {
#pragma unroll
                                    for (int j = 0; j < VEC; ++j)
                                        yv[k][it][j] = __ldg(yr + (col[it] + j) / p.head_dim);
                                } else {
                                    const float s = __ldg(yr);
#pragma unroll
                                    for (int j = 0; j < VEC; ++j) yv[k][it][j] = s;
                                }
                            }
                        }
                    }
                }
                // ---- phase B: consume in slot order, closing rows on the way ----
#pragma unroll
                for (int k = 0; k < U; ++k) {
                    if (k0 + k < nb && !abandon) {
                        while (pos == cur_end) {
                            close_row();
                            ++row;
                            open_row();
                            if (hub) break;
                        }
                        if (hub) {
                            abandon = true;
                        } else {
#pragma unroll
                            for (int it = 0; it < ITERS; ++it) {
                                if (!act[it]) continue;
#pragma unroll
                                for (int j = 0; j < VEC; ++j) {
                                    float m = xv[k][it][j];
                                    if (p.scale_src) m = __fmul_rn(m, sv[k]);
                                    if (MODE == 1) m = apply_msg(p.msg_op, m, yv[k][it][j]);
                                    if (RK == 0) {
                                        acc[it][j] = __fadd_rn(acc[it][j], m);
                                    } else {
                                        acc[it][j] = is_max ? fmaxf(acc[it][j], m)
                                                            : fminf(acc[it][j], m);
                                    }
                                }
                            }
                            ++pos;
                        }
                    }
                }
            }
        }
    }
}

template <typename TI, typename TO, int VEC, int G, int ITERS, int MODE, int RK, bool PROP = false>
__global__ void __launch_bounds__(kThreads) spmm_csr_kernel(const SpmmP p) {
    spmm_csr_body<TI, TO, VEC, G, ITERS, MODE, RK, PROP>(p);
}
// 4 elements per lane with 2 column iterations (129 <= D <= 256): under __launch_bounds__(kThreads)
// ptxas holds these at 80 registers and spills 16-32 bytes; a cap of 96 registers instead removes the spills and ran
// 11 % faster on an H100.  One element per lane (odd D, unaligned rows) also spills 8-24 bytes under the launch bound,
// but capped it ran 17-26 % slower (more registers, fewer resident blocks), so it keeps the launch bound and its
// spills, like the fp32 kernel of the same shape.
template <typename TI, typename TO, int VEC, int G, int ITERS, int RK>
__global__ void __maxnreg__(96) spmm_csr_capped_kernel(const SpmmP p) {
    spmm_csr_body<TI, TO, VEC, G, ITERS, 0, RK>(p);
}

// One block: turn the hub list into chunk tables.
//   chunk_off[h]   exclusive prefix of ceil(deg_h / CH); chunk_off[n] = total
//   vbeg/vend[c]   slot range of chunk c
__global__ void __launch_bounds__(1024) hub_plan_kernel(const int64_t *indptr,
                                                        const unsigned long long *hub_count,
                                                        const int64_t *hub_rows,
                                                        int64_t *chunk_off, int64_t *vbeg,
                                                        int64_t *vend, int64_t *total_chunks,
                                                        int64_t *n_hubs_out) {
    __shared__ int64_t warp_sums[32];
    __shared__ int64_t running;
    const int tid = threadIdx.x;
    const int lane = tid & 31, wid = tid >> 5;
    const int64_t n = (int64_t)*hub_count;
    if (tid == 0) running = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += blockDim.x) {
        const int64_t h = base + tid;
        int64_t b = 0, e = 0, nch = 0;
        if (h < n) {
            const int64_t r = hub_rows[h];
            b = indptr[r];
            e = indptr[r + 1];
            nch = (e - b + HUB_CH - 1) / HUB_CH;
        }
        // block exclusive scan of nch
        int64_t incl = nch;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_sums[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int64_t w = (lane < (int)(blockDim.x >> 5)) ? warp_sums[lane] : 0;
            int64_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int64_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_sums[lane] = wi - w;  // exclusive
            if (lane == 31) warp_sums[31] = wi - w;
        }
        __syncthreads();
        const int64_t off = running + warp_sums[wid] + (incl - nch);
        if (h < n) {
            chunk_off[h] = off;
            for (int64_t c = 0; c < nch; ++c) {
                vbeg[off + c] = b + c * HUB_CH;
                const int64_t ce = b + (c + 1) * HUB_CH;
                vend[off + c] = ce < e ? ce : e;
            }
        }
        __syncthreads();
        if (tid == blockDim.x - 1) running = off + nch;
        __syncthreads();
    }
    if (tid == 0) {
        chunk_off[n] = running;
        *total_chunks = running;
        *n_hubs_out = n;
    }
}

// ---- host side dispatch ----------------------------------------------------------------

struct Shape {
    int vec, g, iters, tiles;
};

static Shape pick_shape(int64_t D, bool vec4) {
    Shape s;
    s.vec = vec4 ? 4 : 1;
    const int64_t cv = D / s.vec;
    s.iters = 1;
    s.tiles = 1;
    if (cv <= 4) s.g = 4;
    else if (cv <= 8) s.g = 8;
    else if (cv <= 16) s.g = 16;
    else {
        s.g = 32;
        if (cv <= 32) s.iters = 1;
        else if (cv <= 64) s.iters = 2;
        else s.iters = 4;
        s.tiles = (int)((cv + 32 * s.iters - 1) / (32 * s.iters));
    }
    return s;
}

typedef void (*SpmmKernel)(const SpmmP);

// TI / TO: element types of the kernel's x / out.  A 16-bit type on either side takes the capped kernel at 4 elements
// per lane and two column iterations for copy messages.  MODE 1 (an edge operand) exists for float32, and for 16-bit x
// (pglb_spmm_csr_ue_x16: fp32 y, sum, 4 elements per lane -- the main pass and hub pass 1) with RK 0 only.
template <typename TI, typename TO, int VEC, int G, int ITERS>
static SpmmKernel pick_mode(int mode, int rk) {
    if constexpr (sizeof(TI) == 4 && sizeof(TO) == 4) {
        if (mode == 1)
            return rk == 0 ? spmm_csr_kernel<TI, TO, VEC, G, ITERS, 1, 0>
                           : spmm_csr_kernel<TI, TO, VEC, G, ITERS, 1, 1>;
        return rk == 0 ? spmm_csr_kernel<TI, TO, VEC, G, ITERS, 0, 0> : spmm_csr_kernel<TI, TO, VEC, G, ITERS, 0, 1>;
    } else {
        if constexpr (sizeof(TI) == 2 && VEC == 4) {
            if (mode == 1) return spmm_csr_kernel<TI, TO, VEC, G, ITERS, 1, 0>;
        }
        if constexpr (VEC == 4 && ITERS == 2) {
            return rk == 0 ? spmm_csr_capped_kernel<TI, TO, VEC, G, ITERS, 0>
                           : spmm_csr_capped_kernel<TI, TO, VEC, G, ITERS, 1>;
        } else {
            return rk == 0 ? spmm_csr_kernel<TI, TO, VEC, G, ITERS, 0, 0>
                           : spmm_csr_kernel<TI, TO, VEC, G, ITERS, 0, 1>;
        }
    }
}

template <typename TI, typename TO, int VEC>
static SpmmKernel pick_kernel_v(const Shape &s, int mode, int rk) {
    switch (s.g) {
        case 4: return pick_mode<TI, TO, VEC, 4, 1>(mode, rk);
        case 8: return pick_mode<TI, TO, VEC, 8, 1>(mode, rk);
        case 16: return pick_mode<TI, TO, VEC, 16, 1>(mode, rk);
        default:
            if (s.iters == 1) return pick_mode<TI, TO, VEC, 32, 1>(mode, rk);
            if (s.iters == 2) return pick_mode<TI, TO, VEC, 32, 2>(mode, rk);
            return pick_mode<TI, TO, VEC, 32, 4>(mode, rk);
    }
}

template <typename TI, typename TO>
static SpmmKernel pick_kernel(const Shape &s, int mode, int rk) {
    return s.vec == 4 ? pick_kernel_v<TI, TO, 4>(s, mode, rk) : pick_kernel_v<TI, TO, 1>(s, mode, rk);
}

// the float32 copy-sum kernel of shape s with pglb_propagate_f32's row epilogue
template <int VEC>
static SpmmKernel pick_prop_kernel_v(const Shape &s) {
    switch (s.g) {
        case 4: return spmm_csr_kernel<float, float, VEC, 4, 1, 0, 0, true>;
        case 8: return spmm_csr_kernel<float, float, VEC, 8, 1, 0, 0, true>;
        case 16: return spmm_csr_kernel<float, float, VEC, 16, 1, 0, 0, true>;
        default:
            if (s.iters == 1) return spmm_csr_kernel<float, float, VEC, 32, 1, 0, 0, true>;
            if (s.iters == 2) return spmm_csr_kernel<float, float, VEC, 32, 2, 0, 0, true>;
            return spmm_csr_kernel<float, float, VEC, 32, 4, 0, 0, true>;
    }
}
static SpmmKernel pick_prop_kernel(const Shape &s) {
    return s.vec == 4 ? pick_prop_kernel_v<4>(s) : pick_prop_kernel_v<1>(s);
}

struct HubWs {
    unsigned long long *hub_count;  // [1]
    int64_t *total_chunks;          // [1]
    int64_t *n_hubs;                // [1]
    int64_t *hub_rows;              // [hub_cap]
    int64_t *chunk_off;             // [hub_cap + 1]
    int64_t *vbeg;                  // [chunk_cap]
    int64_t *vend;                  // [chunk_cap]
    float *partial;                 // [chunk_cap * dpad]
    int64_t hub_cap, chunk_cap, dpad;
    size_t bytes;
};

static HubWs layout_ws(void *ws, int64_t E, int64_t D) {
    HubWs h;
    h.hub_cap = E / (HUB_T + 1) + 1;
    h.chunk_cap = E / HUB_CH + h.hub_cap + 1;
    h.dpad = (D + 3) / 4 * 4;
    char *p = reinterpret_cast<char *>(ws);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char *r = p ? p + off : nullptr;
        off += align_up(bytes, 256);
        return r;
    };
    h.hub_count = reinterpret_cast<unsigned long long *>(take(8));
    h.total_chunks = reinterpret_cast<int64_t *>(take(8));
    h.n_hubs = reinterpret_cast<int64_t *>(take(8));
    h.hub_rows = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * h.hub_cap));
    h.chunk_off = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * (h.hub_cap + 1)));
    h.vbeg = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * h.chunk_cap));
    h.vend = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * h.chunk_cap));
    h.partial = reinterpret_cast<float *>(take(sizeof(float) * h.chunk_cap * h.dpad));
    h.bytes = off;
    return h;
}

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// spmm_stream.cu
size_t stream_ws_bytes(int64_t E, int64_t D);
int spmm_stream_run(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx,
                    float *out, int64_t ldo, int64_t n_dst, int64_t n_src, int64_t E, int64_t D,
                    int reduce_op, const float *scale_src, const float *scale_dst,
                    const uint32_t *cols32, int l2_hints, int accumulate, const int64_t *eid,
                    const float *y, int64_t ldy, int y_bcast, int head_dim, int msg_op, void *ws,
                    size_t ws_bytes, cudaStream_t stream);

// the fused GAT aggregation over f / out of element type T (float, __nv_bfloat16 or __half); gat5_takes: whether its
// TMA kernel takes a call (16-bit calls must be such calls)
template <typename T>
int gat_fused_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, void *out,
                  int64_t ldo, int64_t n_dst, int64_t n_src, int64_t E, int64_t D, int64_t H,
                  const float *attn_src, const float *attn_dst, float slope, float *lse, const AttnDrop *drop, void *ws,
                  size_t ws_bytes, cudaStream_t stream);
template <typename T>
bool gat5_takes(int64_t D, float slope, const void *f, int64_t ldf, const float *attn_src, int64_t H, int64_t n_src);
// the fused dot-product attention (TransformerConv) over q / k / v / out of element type T, with edge features e
// (nullable, through eid), and whether it takes a call
template <typename T>
int dot_attn_run(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq, const void *k, int64_t ldk,
                 const void *v, int64_t ldv, const int64_t *eid, const void *e, int64_t lde, void *out, int64_t ldo,
                 float *lse, int64_t n_dst, int64_t E, int64_t H, int64_t head_dim, const AttnDrop *drop, void *ws,
                 size_t ws_bytes, cudaStream_t stream);
template <typename T>
bool dot_attn_takes(int64_t D, int64_t head_dim, const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v,
                    int64_t ldv, const void *e, int64_t lde, int64_t n_src);

// the fused GATv2 attention (GATv2Conv) over f / out of element type T, and whether it takes a call
template <typename T>
int gatv2_attn_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *attn,
                   float slope, void *out, int64_t ldo, float *lse, int64_t n, int64_t E, int64_t H, int64_t head_dim,
                   const AttnDrop *drop, void *ws, size_t ws_bytes, cudaStream_t stream);
template <typename T>
bool gatv2_attn_takes(int64_t D, int64_t head_dim, float slope, const void *f, int64_t ldf, const float *attn,
                      int64_t n_src);

// the fused FAConv aggregation over f / out of element type T, and whether it takes a call
template <typename T>
int fa_attn_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *rec, void *out,
                int64_t ldo, int64_t n, int64_t E, int64_t D, const AttnDrop *drop, void *ws, size_t ws_bytes,
                cudaStream_t stream);
template <typename T>
bool fa_attn_takes(int64_t D, const void *f, int64_t ldf, const float *rec, int64_t n);

// spmm_v5_kernel over rows of element type T (float, __nv_bfloat16 or __half): whether it takes a call, and the run
template <typename T>
bool v5_eligible(const int64_t *cols, const uint32_t *cols32, const void *x, int64_t ldx, const void *out, int64_t ldo,
                 int64_t n_src, int64_t E, int64_t D, int reduce_op);
template <typename T>
int spmm_v5_run(const int64_t *indptr, const int64_t *cols, const void *x, int64_t ldx, void *out, int64_t ldo,
                int64_t n_dst, int64_t E, int64_t D, int reduce_op, const float *scale_src, const float *scale_slot,
                const float *scale_dst, const uint32_t *cols32, int l2_hints, int accumulate, void *ws,
                size_t ws_bytes, cudaStream_t stream);
int propagate_v5_run(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx, float *out, int64_t ldo,
                     int64_t n_dst, int64_t E, int64_t D, const float *scale_src, const float *scale_slot,
                     const float *scale_dst, const uint32_t *cols32, int l2_hints, const PropEpi &epi, void *ws,
                     size_t ws_bytes, cudaStream_t stream);

// The node-parallel launch sequence behind both entries: spmm_csr kernel over all rows, then, when some row is longer
// than HUB_T slots, the hub plan and the two hub passes.  E is the element type of x and out.  The main pass reads E
// and writes E, hub pass 1 turns chunks into fp32 partials, and pass 2 reduces a hub's partials into its E row.
template <typename E>
static int spmm_generic_run(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *x,
                            int64_t ldx, const float *y, int64_t ldy, int y_bcast, void *out, int64_t ldo,
                            int64_t n_dst, int64_t num_edges, int64_t D, int64_t head_dim, int msg_op, int reduce_op,
                            const float *scale_src, const float *scale_dst, int64_t max_degree_hint, int accumulate,
                            bool vec4, void *ws, size_t ws_bytes, cudaStream_t stream,
                            const PropEpi *epi = nullptr) {
    const Shape s = pick_shape(D, vec4);
    const int mode = (msg_op == PGLB_MSG_COPY) ? 0 : 1;
    const int rk = (reduce_op >= PGLB_REDUCE_MAX) ? 1 : 0;
    const bool need_hub = !(max_degree_hint >= 0 && max_degree_hint <= HUB_T) && num_edges > HUB_T;
    HubWs h{};
    if (need_hub) {
        h = layout_ws(ws, num_edges, D);
        PGLB_CHECK_ARG(ws != nullptr && ws_bytes >= h.bytes, PGLB_EWORKSPACE,
                       "pglb_spmm_csr: workspace of %zu bytes needed (got %zu)", h.bytes,
                       ws_bytes);
        PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                       "pglb_spmm_csr: workspace must be 256-byte aligned");
        PGLB_CUDA(cudaMemsetAsync(h.hub_count, 0, 8, stream));
    }

    SpmmP p{};
    p.rbeg = indptr;
    p.rend = indptr + 1;
    p.cols = cols;
    p.eid = eid;
    p.x = reinterpret_cast<const float *>(x);
    p.ldx = ldx;
    p.y = y;
    p.ldy = ldy;
    p.y_bcast = y_bcast;
    p.out = reinterpret_cast<float *>(out);
    p.ldo = ldo;
    p.n_rows = n_dst;
    p.n_rows_dev = nullptr;
    p.D = (int)D;
    p.head_dim = (int)(head_dim > 0 ? head_dim : 1);
    p.msg_op = msg_op;
    p.reduce_op = reduce_op;
    p.scale_src = scale_src;
    p.scale_dst = scale_dst;
    p.row_map = nullptr;
    p.mean_indptr = nullptr;
    p.rpg = 8;
    p.contig = 1;
    p.hub_threshold = need_hub ? HUB_T : INT64_MAX;
    p.hub_count = h.hub_count;
    p.hub_rows = h.hub_rows;
    p.accumulate = accumulate;
    if (epi) p.epi = *epi;

    const int64_t gpb = kThreads / s.g;
    {
        const int64_t tasks = (n_dst + p.rpg - 1) / p.rpg;
        const int64_t blocks = (tasks + gpb - 1) / gpb;
        PGLB_CHECK_ARG(blocks <= 0x7fffffffLL, PGLB_ESHAPE, "pglb_spmm_csr: grid too large");
        dim3 grid((unsigned)blocks, (unsigned)s.tiles);
        (epi ? pick_prop_kernel(s) : pick_kernel<E, E>(s, mode, rk))<<<grid, kThreads, 0, stream>>>(p);
        PGLB_LAUNCH_CHECK("spmm_csr_kernel");
    }
    if (need_hub) {
        hub_plan_kernel<<<1, 1024, 0, stream>>>(indptr, h.hub_count, h.hub_rows, h.chunk_off,
                                                h.vbeg, h.vend, h.total_chunks, h.n_hubs);
        PGLB_LAUNCH_CHECK("hub_plan_kernel");
        const int64_t max_blocks = (int64_t)sm_count() * 8;
        // pass 1: chunk -> partial (same message, SUM/MAX/MIN, no row epilogue)
        SpmmP p1 = p;
        p1.rbeg = h.vbeg;
        p1.rend = h.vend;
        p1.out = h.partial;
        p1.ldo = h.dpad;
        p1.n_rows = 0;
        p1.n_rows_dev = h.total_chunks;
        p1.reduce_op = (reduce_op == PGLB_REDUCE_MEAN) ? PGLB_REDUCE_SUM : reduce_op;
        p1.scale_dst = nullptr;
        p1.rpg = 1;
        p1.contig = 0;
        p1.accumulate = 0;
        p1.hub_threshold = INT64_MAX;
        {
            int64_t blocks = (h.chunk_cap + gpb - 1) / gpb;
            if (blocks > max_blocks) blocks = max_blocks;
            // partial rows are dpad floats, 16-byte aligned => same vector shape is valid
            dim3 grid((unsigned)blocks, (unsigned)s.tiles);
            pick_kernel<E, float>(s, mode, rk)<<<grid, kThreads, 0, stream>>>(p1);
            PGLB_LAUNCH_CHECK("spmm_csr_kernel(hub pass 1)");
        }
        // pass 2: partials of a hub -> its output row
        SpmmP p2 = p;
        p2.rbeg = h.chunk_off;
        p2.rend = h.chunk_off + 1;
        p2.cols = nullptr;
        p2.eid = nullptr;
        p2.x = h.partial;
        p2.ldx = h.dpad;
        p2.y = nullptr;
        p2.msg_op = PGLB_MSG_COPY;
        p2.scale_src = nullptr;
        p2.n_rows = 0;
        p2.n_rows_dev = h.n_hubs;
        p2.row_map = h.hub_rows;
        p2.mean_indptr = indptr;
        p2.rpg = 1;
        p2.contig = 0;
        p2.hub_threshold = INT64_MAX;
        {
            int64_t blocks = (h.hub_cap + gpb - 1) / gpb;
            if (blocks > max_blocks) blocks = max_blocks;
            dim3 grid((unsigned)blocks, (unsigned)s.tiles);
            (epi ? pick_prop_kernel(s) : pick_kernel<float, E>(s, 0, rk))<<<grid, kThreads, 0, stream>>>(p2);
            PGLB_LAUNCH_CHECK("spmm_csr_kernel(hub pass 2)");
        }
    }
    return PGLB_OK;
}

// ---- GATv2 score gradient (pglb_gatv2_score_grad_*) ------------------------------------------------------------------
// gr[r, c] = sum over the slots j of row r of ds[eid_j, h(c)] * a[c] * lrelu'(f[r, c] + f[cols_j, c]),
// lrelu'(x) = 1 if x > 0 else slope (torch's convention at 0).  On the dst-keyed CSR this is the dst term of GATv2's
// grad f, on the src-keyed CSR its src term (z = f[src] + f[dst] either way); the [E, H*Dh] dz is never stored.  A
// group of G lanes owns a row, a lane 4 columns; slots are taken in order, so each row's sum has a fixed order.  Rows
// longer than HUB_T slots go through spmm_generic_run's hub path: the same kernel over HUB_CH-slot chunks into fp32
// partials (chunks = 1: a chunk's own row is found in indptr), then the copy-sum spmm_csr_kernel over a hub's partials
// in chunk order.  No atomics on values: run to run the result is bit-identical.
struct V2GradP {
    const int64_t *rbeg;    // row r covers slots [rbeg[r], rend[r])
    const int64_t *rend;
    const int64_t *indptr;  // chunks: the CSR, to find the row whose slots hold rbeg[r]
    int64_t n_ind;          // its row count
    const int64_t *cols;
    const int64_t *eid;     // nullable: identity
    const void *f;          // [n, D] of T
    int64_t ldf;
    const float *attn;      // [D]
    const float *ds;        // [E, H]
    float slope;
    int H, D, head_dim;
    float *out;
    int64_t ldo;
    int64_t n_rows;
    const int64_t *n_rows_dev;  // nullable: overrides n_rows (chunks)
    int chunks;
    int accumulate;             // add out's previous contents (rows of the main pass)
    int64_t hub_threshold;
    unsigned long long *hub_count;
    int64_t *hub_rows;
};

template <typename T, int G>
__global__ void __launch_bounds__(kThreads) gatv2_score_grad_kernel(const V2GradP p) {
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
    const int64_t gid = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G;
    const int64_t ngroups = (int64_t)gridDim.x * (kThreads / G);
    const int64_t n_rows = p.n_rows_dev ? *p.n_rows_dev : p.n_rows;
    const int c0 = gl * 4;
    const bool act = c0 < p.D;
    const int head = act ? c0 / p.head_dim : 0;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a4 = act ? __ldg(reinterpret_cast<const float4 *>(p.attn) + gl) : zero;
    const T *f = reinterpret_cast<const T *>(p.f);
    const float slope = p.slope;
    for (int64_t r = gid; r < n_rows; r += ngroups) {
        const int64_t beg = ld_ro(p.rbeg + r), end = ld_ro(p.rend + r);
        if (end - beg > p.hub_threshold) {
            if (gl == 0) p.hub_rows[atomicAdd(p.hub_count, 1ull)] = r;
            continue;
        }
        int64_t row = r;
        if (p.chunks) {   // the last row whose first slot is <= beg (rows of a chunk are never empty)
            int64_t lo = 0, hi = p.n_ind;
            while (hi - lo > 1) {
                const int64_t mid = (lo + hi) >> 1;
                if (ld_ro(p.indptr + mid) <= beg) lo = mid;
                else hi = mid;
            }
            row = lo;
        }
        const float4 fr = act ? ldg_row4<T>(f + row * p.ldf + c0) : zero;
        float4 acc = zero;
        for (int64_t pos = beg; pos < end; pos += G) {
            const int nb = (end - pos) < (int64_t)G ? (int)(end - pos) : G;
            int64_t my_col = 0, my_e = 0;
            if (gl < nb) {
                my_col = ld_stream(p.cols + pos + gl);
                my_e = p.eid ? ld_stream(p.eid + pos + gl) : (pos + gl);
            }
            for (int k0 = 0; k0 < nb; k0 += 4) {
                float4 fs[4];
                float dv[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int src = (k0 + u) & (G - 1);
                    const int64_t c = __shfl_sync(gmask, my_col, src, G);
                    const int64_t e = __shfl_sync(gmask, my_e, src, G);
                    fs[u] = zero;
                    dv[u] = 0.f;
                    if (k0 + u < nb && act) {
                        fs[u] = ldg_row4<T>(f + c * p.ldf + c0);
                        dv[u] = __ldg(p.ds + e * p.H + head);
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (k0 + u >= nb) break;
                    // dz = ds * a * lrelu'(z), z = f[row] + f[col] (the forward's f[src] + f[dst], addition commutes)
                    const float zx = fr.x + fs[u].x, zy = fr.y + fs[u].y, zz = fr.z + fs[u].z, zw = fr.w + fs[u].w;
                    const float tx = dv[u] * a4.x, ty = dv[u] * a4.y, tz = dv[u] * a4.z, tw = dv[u] * a4.w;
                    acc.x = __fadd_rn(acc.x, zx > 0.f ? tx : tx * slope);
                    acc.y = __fadd_rn(acc.y, zy > 0.f ? ty : ty * slope);
                    acc.z = __fadd_rn(acc.z, zz > 0.f ? tz : tz * slope);
                    acc.w = __fadd_rn(acc.w, zw > 0.f ? tw : tw * slope);
                }
            }
        }
        if (act) {
            float *o = p.out + r * p.ldo + c0;
            if (p.accumulate) {
                const float4 prev = *reinterpret_cast<const float4 *>(o);
                acc = make_float4(__fadd_rn(prev.x, acc.x), __fadd_rn(prev.y, acc.y), __fadd_rn(prev.z, acc.z),
                                  __fadd_rn(prev.w, acc.w));
            }
            *reinterpret_cast<float4 *>(o) = acc;
        }
    }
}

template <typename T, int G>
static void launch_v2_grad(const V2GradP &p, int64_t blocks, cudaStream_t stream) {
    gatv2_score_grad_kernel<T, G><<<(unsigned)blocks, kThreads, 0, stream>>>(p);
}

// The launch sequence of pglb_gatv2_score_grad_*: main pass over the rows, then the hub plan and the two hub passes
// when some row is longer than HUB_T slots.  out is float32 [n_rows, D]; ws as pglb_spmm_csr_ws(n_rows, E, D).
template <typename T>
static int gatv2_score_grad_run(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *f,
                                int64_t ldf, const float *attn, float slope, const float *ds, float *out, int64_t ldo,
                                int64_t n_rows, int64_t num_edges, int64_t H, int64_t head_dim, int accumulate,
                                void *ws, size_t ws_bytes, cudaStream_t stream) {
    const int64_t D = H * head_dim;
    const Shape s = pick_shape(D, true);   // the copy-sum kernel of hub pass 2; one tile (D <= 128)
    const bool need_hub = num_edges > HUB_T;
    HubWs h{};
    if (need_hub) {
        h = layout_ws(ws, num_edges, D);
        PGLB_CHECK_ARG(ws != nullptr && ws_bytes >= h.bytes, PGLB_EWORKSPACE,
                       "pglb_gatv2_score_grad: workspace of %zu bytes needed (got %zu)", h.bytes, ws_bytes);
        PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                       "pglb_gatv2_score_grad: workspace must be 256-byte aligned");
        PGLB_CUDA(cudaMemsetAsync(h.hub_count, 0, 8, stream));
    }
    V2GradP p{};
    p.rbeg = indptr;
    p.rend = indptr + 1;
    p.indptr = indptr;
    p.n_ind = n_rows;
    p.cols = cols;
    p.eid = eid;
    p.f = f;
    p.ldf = ldf;
    p.attn = attn;
    p.ds = ds;
    p.slope = slope;
    p.H = (int)H;
    p.D = (int)D;
    p.head_dim = (int)head_dim;
    p.out = out;
    p.ldo = ldo;
    p.n_rows = n_rows;
    p.accumulate = accumulate;
    p.hub_threshold = need_hub ? HUB_T : INT64_MAX;
    p.hub_count = h.hub_count;
    p.hub_rows = h.hub_rows;
    const int64_t gpb = kThreads / s.g;
    auto launch = [&](const V2GradP &q, int64_t blocks) {
        switch (s.g) {
            case 4: launch_v2_grad<T, 4>(q, blocks, stream); break;
            case 8: launch_v2_grad<T, 8>(q, blocks, stream); break;
            case 16: launch_v2_grad<T, 16>(q, blocks, stream); break;
            default: launch_v2_grad<T, 32>(q, blocks, stream); break;
        }
    };
    {
        const int64_t blocks = (n_rows + gpb - 1) / gpb;
        PGLB_CHECK_ARG(blocks <= 0x7fffffffLL, PGLB_ESHAPE, "pglb_gatv2_score_grad: grid too large");
        launch(p, blocks);
        PGLB_LAUNCH_CHECK("gatv2_score_grad_kernel");
    }
    if (need_hub) {
        hub_plan_kernel<<<1, 1024, 0, stream>>>(indptr, h.hub_count, h.hub_rows, h.chunk_off, h.vbeg, h.vend,
                                                h.total_chunks, h.n_hubs);
        PGLB_LAUNCH_CHECK("hub_plan_kernel");
        const int64_t max_blocks = (int64_t)sm_count() * 8;
        // pass 1: chunk -> fp32 partial
        V2GradP p1 = p;
        p1.rbeg = h.vbeg;
        p1.rend = h.vend;
        p1.out = h.partial;
        p1.ldo = h.dpad;
        p1.n_rows = 0;
        p1.n_rows_dev = h.total_chunks;
        p1.chunks = 1;
        p1.accumulate = 0;
        p1.hub_threshold = INT64_MAX;
        {
            int64_t blocks = (h.chunk_cap + gpb - 1) / gpb;
            if (blocks > max_blocks) blocks = max_blocks;
            launch(p1, blocks);
            PGLB_LAUNCH_CHECK("gatv2_score_grad_kernel(hub pass 1)");
        }
        // pass 2: the partials of a hub, in chunk order, into its output row
        SpmmP p2{};
        p2.rbeg = h.chunk_off;
        p2.rend = h.chunk_off + 1;
        p2.x = h.partial;
        p2.ldx = h.dpad;
        p2.out = out;
        p2.ldo = ldo;
        p2.n_rows_dev = h.n_hubs;
        p2.D = (int)D;
        p2.head_dim = 1;
        p2.msg_op = PGLB_MSG_COPY;
        p2.reduce_op = PGLB_REDUCE_SUM;
        p2.row_map = h.hub_rows;
        p2.rpg = 1;
        p2.contig = 0;
        p2.hub_threshold = INT64_MAX;
        p2.accumulate = accumulate;
        {
            int64_t blocks = (h.hub_cap + gpb - 1) / gpb;
            if (blocks > max_blocks) blocks = max_blocks;
            dim3 grid((unsigned)blocks, (unsigned)s.tiles);
            pick_kernel<float, float>(s, 0, 0)<<<grid, kThreads, 0, stream>>>(p2);
            PGLB_LAUNCH_CHECK("spmm_csr_kernel(hub pass 2)");
        }
    }
    return PGLB_OK;
}

// [p, p + extent) of an n-row matrix of D floats per row at stride ld
static bool overlaps(const void *p, int64_t n, int64_t ld, const void *q, int64_t m, int64_t ldq, int64_t D) {
    if (!p || !q || n <= 0 || m <= 0) return false;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
    const uintptr_t ae = a + (uintptr_t)(((n - 1) * ld + D) * 4), be = b + (uintptr_t)(((m - 1) * ldq + D) * 4);
    return a < be && b < ae;
}

int prop_check_args(const char *entry, const void *x, int64_t ldx, int64_t n_src, const void *out, int64_t ldo,
                    int64_t n_dst, int64_t D, const float *h, int64_t ldh, const float *acc_in, int64_t ld_acc_in,
                    const float *acc_out, int64_t ld_acc_out, int flags) {
    PGLB_CHECK_ARG(!(flags & PGLB_SPMM_ACCUMULATE), PGLB_EUNSUPPORTED, "%s: PGLB_SPMM_ACCUMULATE is not taken", entry);
    PGLB_CHECK_ARG(!acc_out == !acc_in, PGLB_EINVAL, "%s: acc_in and acc_out come together", entry);
    PGLB_CHECK_ARG((!h || ldh >= D) && (!acc_in || ld_acc_in >= D) && (!acc_out || ld_acc_out >= D), PGLB_ESHAPE,
                   "%s: leading dimension of h / acc smaller than D", entry);
    if (n_dst == 0 || D == 0) return PGLB_OK;
    // rows of out and acc_out are written while x and h are gathered and acc_in is read: only acc_out == acc_in (the
    // same rows at the same stride) may share memory
    PGLB_CHECK_ARG(!overlaps(out, n_dst, ldo, x, n_src, ldx, D) && !overlaps(out, n_dst, ldo, h, n_dst, ldh, D) &&
                       !overlaps(out, n_dst, ldo, acc_in, n_dst, ld_acc_in, D) &&
                       !overlaps(out, n_dst, ldo, acc_out, n_dst, ld_acc_out, D),
                   PGLB_EINVAL, "%s: out overlaps x, h or acc", entry);
    PGLB_CHECK_ARG(!overlaps(acc_out, n_dst, ld_acc_out, x, n_src, ldx, D) &&
                       !overlaps(acc_out, n_dst, ld_acc_out, h, n_dst, ldh, D),
                   PGLB_EINVAL, "%s: acc_out overlaps x or h", entry);
    PGLB_CHECK_ARG(!overlaps(acc_out, n_dst, ld_acc_out, acc_in, n_dst, ld_acc_in, D) ||
                       (acc_out == acc_in && ld_acc_out == ld_acc_in),
                   PGLB_EINVAL, "%s: acc_out overlaps acc_in other than in place", entry);
    return PGLB_OK;
}

// the 16-byte row accesses of the vector kernels' epilogues
bool prop_rows16(const PropEpi &e) {
    return (!e.h || (aligned16(e.h) && e.ldh % 4 == 0)) && (!e.acc_in || (aligned16(e.acc_in) && e.ld_acc_in % 4 == 0)) &&
           (!e.acc_out || (aligned16(e.acc_out) && e.ld_acc_out % 4 == 0));
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_spmm_csr_ws(int64_t n_dst, int64_t num_edges, int64_t D, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr, PGLB_EINVAL, "pglb_spmm_csr_ws: ws_bytes is NULL");
    PGLB_CHECK_ARG(n_dst >= 0 && num_edges >= 0 && D >= 0, PGLB_EINVAL,
                   "pglb_spmm_csr_ws: negative size");
    size_t a = layout_ws(nullptr, num_edges, D).bytes;
    size_t b = stream_ws_bytes(num_edges, D);
    *ws_bytes = a > b ? a : b;
    return PGLB_OK;
}

extern "C" int pglb_spmm_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                 const float *x, int64_t ldx, const float *y, int64_t ldy,
                                 int y_bcast, float *out, int64_t ldo, int64_t n_dst,
                                 int64_t n_src, int64_t num_edges, int64_t D, int64_t head_dim,
                                 int msg_op, int reduce_op, const float *scale_src,
                                 const float *scale_dst, const uint32_t *cols_packed,
                                 int64_t max_degree_hint, int flags, void *ws, size_t ws_bytes,
                                 void *stream_) {
    return pglb_spmm_csr_slot_scale_f32(indptr, cols, eid, x, ldx, y, ldy, y_bcast, out, ldo, n_dst, n_src, num_edges,
                                        D, head_dim, msg_op, reduce_op, scale_src, nullptr, scale_dst, cols_packed,
                                        max_degree_hint, flags, ws, ws_bytes, stream_);
}

// The argument checks both spmm entries make; `entry` names the caller in pglb_last_error().  A call without work
// (n_dst or D is 0) passes without the pointer and shape checks, so the caller's own early-out follows this call.
static int spmm_check_args(const char *entry, const int64_t *indptr, const void *x, int64_t ldx, const void *out,
                           int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, int reduce_op) {
    PGLB_CHECK_ARG(n_dst >= 0 && n_src >= 0 && num_edges >= 0 && D >= 0, PGLB_EINVAL, "%s: negative size", entry);
    PGLB_CHECK_ARG(reduce_op >= PGLB_REDUCE_SUM && reduce_op <= PGLB_REDUCE_MIN, PGLB_EINVAL,
                   "%s: unknown reduce_op %d", entry, reduce_op);
    if (n_dst == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out, PGLB_EINVAL, "%s: indptr/out is NULL", entry);
    PGLB_CHECK_ARG(num_edges == 0 || x, PGLB_EINVAL, "%s: x is NULL", entry);
    PGLB_CHECK_ARG(ldx >= D && ldo >= D, PGLB_ESHAPE, "%s: leading dimension smaller than D", entry);
    PGLB_CHECK_ARG(D <= INT32_MAX, PGLB_ESHAPE, "%s: D too large", entry);
    return PGLB_OK;
}

extern "C" int pglb_spmm_csr_slot_scale_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                            const float *x, int64_t ldx, const float *y, int64_t ldy,
                                            int y_bcast, float *out, int64_t ldo, int64_t n_dst,
                                            int64_t n_src, int64_t num_edges, int64_t D, int64_t head_dim,
                                            int msg_op, int reduce_op, const float *scale_src,
                                            const float *scale_slot, const float *scale_dst,
                                            const uint32_t *cols_packed, int64_t max_degree_hint, int flags,
                                            void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(msg_op >= PGLB_MSG_COPY && msg_op <= PGLB_MSG_DIV, PGLB_EINVAL,
                   "pglb_spmm_csr_f32: unknown msg_op %d", msg_op);
    PGLB_CHECK_ARG(!scale_slot || scale_src, PGLB_EINVAL, "pglb_spmm_csr_slot_scale_f32: scale_slot needs scale_src");
    {
        const int rc = spmm_check_args("pglb_spmm_csr_f32", indptr, x, ldx, out, ldo, n_dst, n_src, num_edges, D,
                                       reduce_op);
        if (rc) return rc;
    }
    if (n_dst == 0 || D == 0) return PGLB_OK;
    const int accumulate = (flags & PGLB_SPMM_ACCUMULATE) ? 1 : 0;
    PGLB_CHECK_ARG(!accumulate || reduce_op == PGLB_REDUCE_SUM, PGLB_EUNSUPPORTED,
                   "pglb_spmm_csr_f32: PGLB_SPMM_ACCUMULATE needs reduce_op SUM");
    const int mode = (msg_op == PGLB_MSG_COPY) ? 0 : 1;
    if (mode == 1) {
        PGLB_CHECK_ARG(y != nullptr, PGLB_EINVAL, "pglb_spmm_csr_f32: msg_op needs y");
        PGLB_CHECK_ARG(y_bcast >= PGLB_BCAST_FULL && y_bcast <= PGLB_BCAST_SCALAR, PGLB_EINVAL,
                       "pglb_spmm_csr_f32: unknown y_bcast %d", y_bcast);
        if (y_bcast == PGLB_BCAST_HEAD)
            PGLB_CHECK_ARG(head_dim > 0 && D % head_dim == 0, PGLB_ESHAPE,
                           "pglb_spmm_csr_f32: head_dim must divide D");
    }
    const bool vec4 = (D % 4 == 0) && (ldx % 4 == 0) && (ldo % 4 == 0) && aligned16(x) &&
                      aligned16(out) &&
                      (mode == 0 || y_bcast != PGLB_BCAST_FULL || ((ldy % 4 == 0) && aligned16(y)));
    // wide rows: the edge-balanced kernels (spmm_stream.cu), spmm_v5_kernel where it applies.  With an edge operand
    // only the GAT shape qualifies: per-head (head_dim % 4 == 0) or scalar y, mul / add, D <= 128.
    const bool ue_fast = mode == 1 && D <= 128 && scale_src == nullptr && num_edges < 0x7fffffffLL &&
                         (msg_op == PGLB_MSG_MUL || msg_op == PGLB_MSG_ADD) &&
                         (y_bcast == PGLB_BCAST_SCALAR || (y_bcast == PGLB_BCAST_HEAD && head_dim % 4 == 0));
    if ((mode == 0 || ue_fast) && vec4 && D > 64 && num_edges > 0) {
        PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                       "pglb_spmm_csr_f32: workspace must be 256-byte aligned");
        const int l2_hints = (flags & PGLB_SPMM_L2_HINTS) ? 1 : 0;
        if (mode == 0 && v5_eligible<float>(cols, cols_packed, x, ldx, out, ldo, n_src, num_edges, D, reduce_op))
            return spmm_v5_run<float>(indptr, cols, x, ldx, out, ldo, n_dst, num_edges, D, reduce_op, scale_src,
                                      scale_slot, scale_dst, cols_packed, l2_hints, accumulate, ws, ws_bytes, stream);
        return spmm_stream_run(indptr, cols, x, ldx, out, ldo, n_dst, n_src, num_edges, D, reduce_op, scale_src,
                               scale_dst, mode == 0 ? cols_packed : nullptr, l2_hints, accumulate, eid,
                               mode == 1 ? y : nullptr, ldy, y_bcast, (int)head_dim, msg_op, ws, ws_bytes, stream);
    }
    return spmm_generic_run<float>(indptr, cols, eid, x, ldx, y, ldy, y_bcast, out, ldo, n_dst, num_edges, D, head_dim,
                                   msg_op, reduce_op, scale_src, scale_dst, max_degree_hint, accumulate, vec4, ws,
                                   ws_bytes, stream);
}

extern "C" int pglb_propagate_f32(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx, float *out,
                                  int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D,
                                  const float *scale_src, const float *scale_slot, const float *scale_dst, float a,
                                  float b, const float *h, int64_t ldh, const float *acc_in, int64_t ld_acc_in,
                                  float *acc_out, int64_t ld_acc_out, float c, const float *c_dev,
                                  const uint32_t *cols_packed, int64_t max_degree_hint, int flags, void *ws,
                                  size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(!scale_slot || scale_src, PGLB_EINVAL, "pglb_propagate_f32: scale_slot needs scale_src");
    {
        int rc = spmm_check_args("pglb_propagate_f32", indptr, x, ldx, out, ldo, n_dst, n_src, num_edges, D,
                                 PGLB_REDUCE_SUM);
        if (rc) return rc;
        rc = prop_check_args("pglb_propagate_f32", x, ldx, n_src, out, ldo, n_dst, D, h, ldh, acc_in, ld_acc_in,
                             acc_out, ld_acc_out, flags);
        if (rc) return rc;
    }
    if (n_dst == 0 || D == 0) return PGLB_OK;
    const PropEpi e{h, ldh, acc_in, ld_acc_in, acc_out, ld_acc_out, a, b, c, c_dev};
    // the route pglb_spmm_csr_slot_scale_f32 takes for copy sum, so the row sums t are the same
    const bool vec4 = (D % 4 == 0) && (ldx % 4 == 0) && (ldo % 4 == 0) && aligned16(x) && aligned16(out);
    PGLB_CHECK_ARG(!vec4 || prop_rows16(e), PGLB_EUNSUPPORTED,
                   "pglb_propagate_f32: h / acc rows must be 16-byte aligned like x and out");
    if (vec4 && D > 64 && num_edges > 0) {
        PGLB_CHECK_ARG(v5_eligible<float>(cols, cols_packed, x, ldx, out, ldo, n_src, num_edges, D, PGLB_REDUCE_SUM),
                       PGLB_EUNSUPPORTED, "pglb_propagate_f32: this wide-row shape takes spmm_stream, which has no "
                       "epilogue (identity columns, ids or rows past 2^31)");
        PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                       "pglb_propagate_f32: workspace must be 256-byte aligned");
        return propagate_v5_run(indptr, cols, x, ldx, out, ldo, n_dst, num_edges, D, scale_src, scale_slot, scale_dst,
                                cols_packed, (flags & PGLB_SPMM_L2_HINTS) ? 1 : 0, e, ws, ws_bytes, stream);
    }
    return spmm_generic_run<float>(indptr, cols, nullptr, x, ldx, nullptr, 0, 0, out, ldo, n_dst, num_edges, D, 1,
                                   PGLB_MSG_COPY, PGLB_REDUCE_SUM, scale_src, scale_dst, max_degree_hint, 0, vec4, ws,
                                   ws_bytes, stream, &e);
}

extern "C" int pglb_spmm_csr_x16(const int64_t *indptr, const int64_t *cols, const void *x, int64_t ldx, void *out,
                                 int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, int dtype,
                                 int reduce_op, const float *scale_src, const float *scale_slot,
                                 const float *scale_dst, const uint32_t *cols_packed, int64_t max_degree_hint,
                                 int flags, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_spmm_csr_x16: unknown dtype %d", dtype);
    PGLB_CHECK_ARG(!scale_slot || scale_src, PGLB_EINVAL, "pglb_spmm_csr_x16: scale_slot needs scale_src");
    PGLB_CHECK_ARG(!(flags & PGLB_SPMM_ACCUMULATE), PGLB_EUNSUPPORTED,
                   "pglb_spmm_csr_x16: PGLB_SPMM_ACCUMULATE would round the output twice");
    {
        const int rc = spmm_check_args("pglb_spmm_csr_x16", indptr, x, ldx, out, ldo, n_dst, n_src, num_edges, D,
                                       reduce_op);
        if (rc) return rc;
    }
    if (n_dst == 0 || D == 0) return PGLB_OK;
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        if (num_edges > 0 && v5_eligible<T>(cols, cols_packed, x, ldx, out, ldo, n_src, num_edges, D, reduce_op)) {
            PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                           "pglb_spmm_csr_x16: workspace must be 256-byte aligned");
            return spmm_v5_run<T>(indptr, cols, x, ldx, out, ldo, n_dst, num_edges, D, reduce_op, scale_src, scale_slot,
                                  scale_dst, cols_packed, (flags & PGLB_SPMM_L2_HINTS) ? 1 : 0, 0, ws, ws_bytes,
                                  stream);
        }
        // every other shape: the node-parallel kernel, 8 bytes (4 elements) per lane when rows allow it
        auto aligned8 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 7u) == 0; };
        const bool vec4 = (D % 4 == 0) && (ldx % 4 == 0) && (ldo % 4 == 0) && aligned8(x) && aligned8(out);
        return spmm_generic_run<T>(indptr, cols, nullptr, x, ldx, nullptr, 0, 0, out, ldo, n_dst, num_edges, D, 1,
                                   PGLB_MSG_COPY, reduce_op, scale_src, scale_dst, max_degree_hint, 0, vec4, ws,
                                   ws_bytes, stream);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// The argument checks and the launch of the fused GAT entries.  T: element type of f and out.  A 16-bit call also
// needs 16-byte rows (ldf, ldo % 8 == 0) and a shape the TMA kernel takes; both are checked before any CUDA call.
template <typename T>
static int gat_fused_entry(const char *name, const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                           const float *attn_src, const float *attn_dst, float negative_slope, void *out, int64_t ldo,
                           float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim,
                           void *ws, size_t ws_bytes, void *stream_, const AttnDrop *drop = nullptr) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(n_dst >= 0 && n_src >= 0 && num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && num_edges < 0x7fffffffLL && n_src < 0xffffffffLL,
                   PGLB_EUNSUPPORTED, "%s: needs H*head_dim <= 128 and head_dim %% 4 == 0", name);
    if (n_dst == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ldf >= D && ldo >= D && (ldf * B) % 16 == 0 && (ldo * B) % 16 == 0 && aligned16(f) && aligned16(out),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    if constexpr (B == 2) {
        PGLB_CHECK_ARG(num_edges == 0 || (cols && f && attn_src && attn_dst), PGLB_EINVAL, "%s: NULL pointer", name);
        PGLB_CHECK_ARG(num_edges == 0 || (ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0), PGLB_EWORKSPACE,
                       "%s: workspace NULL or not 256-byte aligned", name);
        PGLB_CHECK_ARG(gat5_takes<T>(D, negative_slope, f, ldf, attn_src, H, n_src), PGLB_EUNSUPPORTED,
                       "%s: shape outside the 16-bit kernel (H %% 4, H <= 32, D %% 8, 16-byte attention rows, "
                       "0 <= slope <= 1)", name);
    }
    if (num_edges == 0) {
        PGLB_CUDA(cudaMemset2DAsync(out, B * ldo, 0, B * D, n_dst, stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(cols && f && attn_src && attn_dst, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                   "%s: workspace NULL or not 256-byte aligned", name);
    return gat_fused_run<T>(indptr, cols, f, ldf, out, ldo, n_dst, n_src, num_edges, D, H, attn_src, attn_dst,
                            negative_slope, lse, drop, ws, ws_bytes, stream);
}

extern "C" int pglb_gat_fused_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f,
                                      int64_t ldf, const float *attn_src, const float *attn_dst,
                                      float negative_slope, float *out, int64_t ldo, int64_t n_dst,
                                      int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim,
                                      void *ws, size_t ws_bytes, void *stream_) {
    return gat_fused_entry<float>("pglb_gat_fused_csr_f32", indptr, cols, f, ldf, attn_src, attn_dst, negative_slope,
                                  out, ldo, nullptr, n_dst, n_src, num_edges, H, head_dim, ws, ws_bytes, stream_);
}

// Training forward: the same launch, which additionally leaves lse[d, h] = log sum_j exp(leaky(as[src_j,h] + ad[d,h]))
// for every row with at least one in-edge (rows without are not written) -- all pglb_gat_bwd_edge_f32 needs to rebuild
// the attention weights.  PGLB_EUNSUPPORTED when the shape is outside the TMA kernel (the caller keeps the op-by-op path).
extern "C" int pglb_gat_fused_train_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f,
                                            int64_t ldf, const float *attn_src, const float *attn_dst,
                                            float negative_slope, float *out, int64_t ldo, float *lse,
                                            int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                            int64_t head_dim, void *ws, size_t ws_bytes, void *stream_) {
    PGLB_CHECK_ARG(lse != nullptr || n_dst == 0, PGLB_EINVAL, "pglb_gat_fused_train_csr_f32: NULL lse");
    return gat_fused_entry<float>("pglb_gat_fused_train_csr_f32", indptr, cols, f, ldf, attn_src, attn_dst,
                                  negative_slope, out, ldo, lse, n_dst, n_src, num_edges, H, head_dim, ws, ws_bytes,
                                  stream_);
}

// 16-bit f / out (include/pglb.h): the fp32 entries' arguments plus `dtype`
extern "C" int pglb_gat_fused_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                      const float *attn_src, const float *attn_dst, float negative_slope, void *out,
                                      int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                      int64_t head_dim, int dtype, void *ws, size_t ws_bytes, void *stream_) {
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_gat_fused_csr_x16: unknown dtype %d", dtype);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return gat_fused_entry<T>("pglb_gat_fused_csr_x16", indptr, cols, f, ldf, attn_src, attn_dst, negative_slope,
                                  out, ldo, nullptr, n_dst, n_src, num_edges, H, head_dim, ws, ws_bytes, stream_);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

extern "C" int pglb_gat_fused_train_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                            const float *attn_src, const float *attn_dst, float negative_slope,
                                            void *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src,
                                            int64_t num_edges, int64_t H, int64_t head_dim, int dtype, void *ws,
                                            size_t ws_bytes, void *stream_) {
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_gat_fused_train_csr_x16: unknown dtype %d", dtype);
    PGLB_CHECK_ARG(lse != nullptr || n_dst == 0, PGLB_EINVAL, "pglb_gat_fused_train_csr_x16: NULL lse");
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return gat_fused_entry<T>("pglb_gat_fused_train_csr_x16", indptr, cols, f, ldf, attn_src, attn_dst,
                                  negative_slope, out, ldo, lse, n_dst, n_src, num_edges, H, head_dim, ws, ws_bytes,
                                  stream_);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// Training forward with attention dropout (include/pglb.h): the train entries' arguments plus attn_drop, seed, offset.
// The dropout arguments are checked first, before any CUDA call.
extern "C" int pglb_gat_fused_train_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f,
                                                 int64_t ldf, const float *attn_src, const float *attn_dst,
                                                 float negative_slope, float *out, int64_t ldo, float *lse,
                                                 int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                                 int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                                 void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gat_fused_train_drop_csr_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(lse != nullptr || n_dst == 0, PGLB_EINVAL, "%s: NULL lse", name);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return gat_fused_entry<float>(name, indptr, cols, f, ldf, attn_src, attn_dst, negative_slope, out, ldo, lse, n_dst,
                                  n_src, num_edges, H, head_dim, ws, ws_bytes, stream_, &drop);
}

extern "C" int pglb_gat_fused_train_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f,
                                                 int64_t ldf, const float *attn_src, const float *attn_dst,
                                                 float negative_slope, void *out, int64_t ldo, float *lse,
                                                 int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                                 int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                                 uint64_t offset, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gat_fused_train_drop_csr_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    PGLB_CHECK_ARG(lse != nullptr || n_dst == 0, PGLB_EINVAL, "%s: NULL lse", name);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return gat_fused_entry<T>(name, indptr, cols, f, ldf, attn_src, attn_dst, negative_slope, out, ldo, lse, n_dst,
                                  n_src, num_edges, H, head_dim, ws, ws_bytes, stream_, &drop);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// The argument checks and the launch of the dot-product attention entries (include/pglb.h).  T: element type of q, k,
// v, e and out.  Every check precedes any CUDA call.  drop (nullable): the attention-dropout stream.  ef: an edge-feature
// entry (pglb_dot_attn_e_*), whose eid and e must then be given when there are edges.
template <typename T>
static int dot_attn_entry(const char *name, const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq,
                          const void *k, int64_t ldk, const void *v, int64_t ldv, void *out, int64_t ldo, float *lse,
                          int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, void *ws,
                          size_t ws_bytes, void *stream_, const AttnDrop *drop, bool ef = false,
                          const int64_t *eid = nullptr, const void *e = nullptr, int64_t lde = 0) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(n_dst >= 0 && n_src >= 0 && num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    const int64_t lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0 && (D * B) % 16 == 0 &&
                       num_edges < 0x7fffffffLL && n_src < 0x7fffffffLL,
                   PGLB_EUNSUPPORTED, "%s: needs H*head_dim <= 128 in 16-byte rows, head_dim in {4, 8, ..., 128}", name);
    PGLB_CHECK_ARG(!drop || H % 4 == 0, PGLB_EUNSUPPORTED, "%s: attention dropout needs H %% 4 == 0", name);
    if (n_dst == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ldq >= D && ldk >= D && ldv >= D && ldo >= D && (ldo * B) % 16 == 0 && aligned16(out) &&
                       (!ef || lde >= D) && dot_attn_takes<T>(D, head_dim, q, ldq, k, ldk, v, ldv, e, lde, n_src),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    if (num_edges == 0) {
        PGLB_CUDA(cudaMemset2DAsync(out, B * ldo, 0, B * D, n_dst, stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(cols && q && k && v && (!ef || (eid && e)), PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                   "%s: workspace NULL or not 256-byte aligned", name);
    return dot_attn_run<T>(indptr, cols, q, ldq, k, ldk, v, ldv, eid, e, lde, out, ldo, lse, n_dst, num_edges, H,
                           head_dim, drop, ws, ws_bytes, stream);
}

extern "C" int pglb_dot_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *q, int64_t ldq,
                                     const float *k, int64_t ldk, const float *v, int64_t ldv, float *out, int64_t ldo,
                                     float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                     int64_t head_dim, void *ws, size_t ws_bytes, void *stream_) {
    return dot_attn_entry<float>("pglb_dot_attn_csr_f32", indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst,
                                 n_src, num_edges, H, head_dim, ws, ws_bytes, stream_, nullptr);
}

extern "C" int pglb_dot_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq,
                                     const void *k, int64_t ldk, const void *v, int64_t ldv, void *out, int64_t ldo,
                                     float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                     int64_t head_dim, int dtype, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_csr_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return dot_attn_entry<T>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, nullptr);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

extern "C" int pglb_dot_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *q, int64_t ldq,
                                          const float *k, int64_t ldk, const float *v, int64_t ldv, float *out,
                                          int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                                          int64_t H, int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                          void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_drop_csr_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return dot_attn_entry<float>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, &drop);
}

extern "C" int pglb_dot_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq,
                                          const void *k, int64_t ldk, const void *v, int64_t ldv, void *out,
                                          int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                                          int64_t H, int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                          uint64_t offset, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_drop_csr_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return dot_attn_entry<T>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, &drop);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// Dot-product attention with edge features (include/pglb.h): the pglb_dot_attn_* arguments plus eid (dst-CSR slot ->
// edge id), e [num_edges, H * head_dim] in edge-id order and its row stride lde.
extern "C" int pglb_dot_attn_e_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const float *q,
                                       int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv,
                                       const float *e, int64_t lde, float *out, int64_t ldo, float *lse, int64_t n_dst,
                                       int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, void *ws,
                                       size_t ws_bytes, void *stream_) {
    return dot_attn_entry<float>("pglb_dot_attn_e_csr_f32", indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst,
                                 n_src, num_edges, H, head_dim, ws, ws_bytes, stream_, nullptr, true, eid, e, lde);
}

extern "C" int pglb_dot_attn_e_csr_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *q,
                                       int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                       const void *e, int64_t lde, void *out, int64_t ldo, float *lse, int64_t n_dst,
                                       int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                                       void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_e_csr_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return dot_attn_entry<T>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, nullptr, true, eid, e, lde);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

extern "C" int pglb_dot_attn_e_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                            const float *q, int64_t ldq, const float *k, int64_t ldk, const float *v,
                                            int64_t ldv, const float *e, int64_t lde, float *out, int64_t ldo,
                                            float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                            int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                            void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_e_drop_csr_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return dot_attn_entry<float>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, &drop, true, eid, e, lde);
}

extern "C" int pglb_dot_attn_e_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                            const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v,
                                            int64_t ldv, const void *e, int64_t lde, void *out, int64_t ldo,
                                            float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                            int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                            uint64_t offset, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_dot_attn_e_drop_csr_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return dot_attn_entry<T>(name, indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, num_edges, H,
                                 head_dim, ws, ws_bytes, stream_, &drop, true, eid, e, lde);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// The argument checks and the launch of the GATv2 attention entries (include/pglb.h).  T: element type of f and out.
// Every check precedes any CUDA call.  drop (nullable): the attention-dropout stream.
template <typename T>
static int gatv2_attn_entry(const char *name, const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                            const float *attn, float slope, void *out, int64_t ldo, float *lse, int64_t n,
                            int64_t num_edges, int64_t H, int64_t head_dim, void *ws, size_t ws_bytes, void *stream_,
                            const AttnDrop *drop) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(n >= 0 && num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    const int64_t lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0 && (D * B) % 16 == 0 &&
                       num_edges < 0x7fffffffLL && n < 0x7fffffffLL,
                   PGLB_EUNSUPPORTED, "%s: needs H*head_dim <= 128 in 16-byte rows, head_dim in {4, 8, ..., 128}", name);
    PGLB_CHECK_ARG(slope >= 0.0f && slope <= 1.0f, PGLB_EUNSUPPORTED, "%s: needs 0 <= negative_slope <= 1", name);
    PGLB_CHECK_ARG(!drop || H % 4 == 0, PGLB_EUNSUPPORTED, "%s: attention dropout needs H %% 4 == 0", name);
    if (n == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ldf >= D && ldo >= D && (ldo * B) % 16 == 0 && aligned16(out) &&
                       (num_edges == 0 || gatv2_attn_takes<T>(D, head_dim, slope, f, ldf, attn, n)),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    if (num_edges == 0) {
        PGLB_CUDA(cudaMemset2DAsync(out, B * ldo, 0, B * D, n, stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(cols && f && attn, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                   "%s: workspace NULL or not 256-byte aligned", name);
    return gatv2_attn_run<T>(indptr, cols, f, ldf, attn, slope, out, ldo, lse, n, num_edges, H, head_dim, drop, ws,
                             ws_bytes, stream);
}

extern "C" int pglb_gatv2_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                       const float *attn, float negative_slope, float *out, int64_t ldo, float *lse,
                                       int64_t n, int64_t num_edges, int64_t H, int64_t head_dim, void *ws,
                                       size_t ws_bytes, void *stream_) {
    return gatv2_attn_entry<float>("pglb_gatv2_attn_csr_f32", indptr, cols, f, ldf, attn, negative_slope, out, ldo, lse,
                                   n, num_edges, H, head_dim, ws, ws_bytes, stream_, nullptr);
}

extern "C" int pglb_gatv2_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                       const float *attn, float negative_slope, void *out, int64_t ldo, float *lse,
                                       int64_t n, int64_t num_edges, int64_t H, int64_t head_dim, int dtype, void *ws,
                                       size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gatv2_attn_csr_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return gatv2_attn_entry<T>(name, indptr, cols, f, ldf, attn, negative_slope, out, ldo, lse, n, num_edges, H,
                                   head_dim, ws, ws_bytes, stream_, nullptr);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

extern "C" int pglb_gatv2_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                            const float *attn, float negative_slope, float *out, int64_t ldo,
                                            float *lse, int64_t n, int64_t num_edges, int64_t H, int64_t head_dim,
                                            float attn_drop, uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes,
                                            void *stream_) {
    const char *name = "pglb_gatv2_attn_drop_csr_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return gatv2_attn_entry<float>(name, indptr, cols, f, ldf, attn, negative_slope, out, ldo, lse, n, num_edges, H,
                                   head_dim, ws, ws_bytes, stream_, &drop);
}

extern "C" int pglb_gatv2_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                            const float *attn, float negative_slope, void *out, int64_t ldo,
                                            float *lse, int64_t n, int64_t num_edges, int64_t H, int64_t head_dim,
                                            int dtype, float attn_drop, uint64_t seed, uint64_t offset, void *ws,
                                            size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gatv2_attn_drop_csr_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return gatv2_attn_entry<T>(name, indptr, cols, f, ldf, attn, negative_slope, out, ldo, lse, n, num_edges, H,
                                   head_dim, ws, ws_bytes, stream_, &drop);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// The argument checks and the launch of the FAConv aggregation entries (include/pglb.h).  T: element type of f and
// out.  Every check precedes any CUDA call.  drop (nullable): the attention-dropout stream.
template <typename T>
static int fa_attn_entry(const char *name, const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                         const float *rec, void *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D, void *ws,
                         size_t ws_bytes, void *stream_, const AttnDrop *drop) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(n >= 0 && num_edges >= 0 && D > 0, PGLB_EINVAL, "%s: bad size", name);
    PGLB_CHECK_ARG(D <= 128 && (D * B) % 16 == 0 && num_edges < 0x7fffffffLL && n < 0x7fffffffLL, PGLB_EUNSUPPORTED,
                   "%s: needs D <= 128 in 16-byte rows (D %% 4 == 0 float32, D %% 8 == 0 16-bit)", name);
    if (n == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(num_edges == 0 || (cols && f && rec), PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ldf >= D && ldo >= D && (ldo * B) % 16 == 0 && aligned16(out) &&
                       (num_edges == 0 || fa_attn_takes<T>(D, f, ldf, rec, n)),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    if (num_edges == 0) {
        PGLB_CUDA(cudaMemset2DAsync(out, B * ldo, 0, B * D, n, stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, PGLB_EWORKSPACE,
                   "%s: workspace NULL or not 256-byte aligned", name);
    return fa_attn_run<T>(indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, drop, ws, ws_bytes, stream);
}

extern "C" int pglb_fa_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                    const float *rec, float *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D,
                                    void *ws, size_t ws_bytes, void *stream_) {
    return fa_attn_entry<float>("pglb_fa_attn_csr_f32", indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws,
                                ws_bytes, stream_, nullptr);
}

extern "C" int pglb_fa_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                    const float *rec, void *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D,
                                    int dtype, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_fa_attn_csr_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return fa_attn_entry<__nv_bfloat16>(name, indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws, ws_bytes,
                                            stream_, nullptr);
    return fa_attn_entry<__half>(name, indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws, ws_bytes, stream_,
                                 nullptr);
}

extern "C" int pglb_fa_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                         const float *rec, float *out, int64_t ldo, int64_t n, int64_t num_edges,
                                         int64_t D, float attn_drop, uint64_t seed, uint64_t offset, void *ws,
                                         size_t ws_bytes, void *stream_) {
    const char *name = "pglb_fa_attn_drop_csr_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return fa_attn_entry<float>(name, indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws, ws_bytes, stream_,
                                &drop);
}

extern "C" int pglb_fa_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                         const float *rec, void *out, int64_t ldo, int64_t n, int64_t num_edges,
                                         int64_t D, int dtype, float attn_drop, uint64_t seed, uint64_t offset,
                                         void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_fa_attn_drop_csr_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return fa_attn_entry<__nv_bfloat16>(name, indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws, ws_bytes,
                                            stream_, &drop);
    return fa_attn_entry<__half>(name, indptr, cols, f, ldf, rec, out, ldo, n, num_edges, D, ws, ws_bytes, stream_,
                                 &drop);
}

// Send/recv with an edge operand over 16-bit x / out (include/pglb.h): the node-parallel kernel with MODE 1 -- the
// reverse-CSR aggregation of the fused GAT backward (grad f = sum over out-edges of alpha * grad_out[dst]).
extern "C" int pglb_spmm_csr_ue_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *x,
                                    int64_t ldx, const float *y, int64_t ldy, int y_bcast, void *out, int64_t ldo,
                                    int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, int64_t head_dim,
                                    int dtype, int msg_op, int reduce_op, const float *scale_src,
                                    const float *scale_dst, int64_t max_degree_hint, int flags, void *ws,
                                    size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_spmm_csr_ue_x16: unknown dtype %d", dtype);
    PGLB_CHECK_ARG(msg_op >= PGLB_MSG_COPY && msg_op <= PGLB_MSG_DIV, PGLB_EINVAL,
                   "pglb_spmm_csr_ue_x16: unknown msg_op %d", msg_op);
    PGLB_CHECK_ARG(y_bcast >= PGLB_BCAST_FULL && y_bcast <= PGLB_BCAST_SCALAR, PGLB_EINVAL,
                   "pglb_spmm_csr_ue_x16: unknown y_bcast %d", y_bcast);
    {
        const int rc = spmm_check_args("pglb_spmm_csr_ue_x16", indptr, x, ldx, out, ldo, n_dst, n_src, num_edges, D,
                                       reduce_op);
        if (rc) return rc;
    }
    PGLB_CHECK_ARG(msg_op == PGLB_MSG_MUL || msg_op == PGLB_MSG_ADD, PGLB_EUNSUPPORTED,
                   "pglb_spmm_csr_ue_x16: mul / add messages only");
    PGLB_CHECK_ARG(reduce_op == PGLB_REDUCE_SUM, PGLB_EUNSUPPORTED, "pglb_spmm_csr_ue_x16: sum only");
    PGLB_CHECK_ARG(y_bcast != PGLB_BCAST_FULL, PGLB_EUNSUPPORTED,
                   "pglb_spmm_csr_ue_x16: per-head or scalar edge operands only");
    PGLB_CHECK_ARG(!(flags & PGLB_SPMM_ACCUMULATE), PGLB_EUNSUPPORTED,
                   "pglb_spmm_csr_ue_x16: PGLB_SPMM_ACCUMULATE would round the output twice");
    if (n_dst == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(num_edges == 0 || y, PGLB_EINVAL, "pglb_spmm_csr_ue_x16: y is NULL");
    PGLB_CHECK_ARG(D % 4 == 0, PGLB_EUNSUPPORTED, "pglb_spmm_csr_ue_x16: D %% 4 == 0 needed");
    if (y_bcast == PGLB_BCAST_HEAD)
        PGLB_CHECK_ARG(head_dim > 0 && D % head_dim == 0, PGLB_ESHAPE, "pglb_spmm_csr_ue_x16: head_dim must divide D");
    auto aligned8 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 7u) == 0; };
    PGLB_CHECK_ARG(ldx % 4 == 0 && ldo % 4 == 0 && aligned8(x) && aligned8(out), PGLB_ESHAPE,
                   "pglb_spmm_csr_ue_x16: rows must be 8-byte aligned (ldx, ldo %% 4 == 0)");
    auto run = [&](auto *elem) -> int {
        using T = std::remove_pointer_t<decltype(elem)>;
        return spmm_generic_run<T>(indptr, cols, eid, x, ldx, y, ldy, y_bcast, out, ldo, n_dst, num_edges, D,
                                   head_dim, msg_op, reduce_op, scale_src, scale_dst, max_degree_hint, 0, true, ws,
                                   ws_bytes, stream);
    };
    return dtype == PGLB_DTYPE_BF16 ? run((__nv_bfloat16 *)nullptr) : run((__half *)nullptr);
}

// The checks and the launch of the GATv2 score-gradient entries (include/pglb.h).  T: element type of f.
template <typename T>
static int gatv2_score_grad_entry(const char *name, const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                  const void *f, int64_t ldf, const float *attn, float slope, const float *ds,
                                  float *out, int64_t ldo, int64_t n_rows, int64_t num_edges, int64_t H,
                                  int64_t head_dim, int accumulate, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(n_rows >= 0 && num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (D * B) % 16 == 0, PGLB_EUNSUPPORTED,
                   "%s: needs H*head_dim <= 128 in 16-byte rows and head_dim %% 4 == 0", name);
    PGLB_CHECK_ARG(slope >= 0.0f && slope <= 1.0f, PGLB_EUNSUPPORTED, "%s: needs 0 <= negative_slope <= 1", name);
    if (n_rows == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && out && (num_edges == 0 || (cols && f && attn && ds)), PGLB_EINVAL, "%s: NULL pointer",
                   name);
    PGLB_CHECK_ARG(ldf >= D && ldo >= D && (ldf * B) % 16 == 0 && ldo % 4 == 0 && aligned16(f) && aligned16(out) &&
                       aligned16(attn),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    if (num_edges == 0) {
        if (!accumulate) PGLB_CUDA(cudaMemset2DAsync(out, 4 * ldo, 0, 4 * D, n_rows, stream));
        return PGLB_OK;
    }
    return gatv2_score_grad_run<T>(indptr, cols, eid, f, ldf, attn, slope, ds, out, ldo, n_rows, num_edges, H,
                                   head_dim, accumulate, ws, ws_bytes, stream);
}

extern "C" int pglb_gatv2_score_grad_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const float *f,
                                         int64_t ldf, const float *attn, float negative_slope, const float *ds,
                                         float *out, int64_t ldo, int64_t n_rows, int64_t num_edges, int64_t H,
                                         int64_t head_dim, int accumulate, void *ws, size_t ws_bytes, void *stream_) {
    return gatv2_score_grad_entry<float>("pglb_gatv2_score_grad_f32", indptr, cols, eid, f, ldf, attn, negative_slope,
                                         ds, out, ldo, n_rows, num_edges, H, head_dim, accumulate, ws, ws_bytes,
                                         stream_);
}

extern "C" int pglb_gatv2_score_grad_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *f,
                                         int64_t ldf, const float *attn, float negative_slope, const float *ds,
                                         float *out, int64_t ldo, int64_t n_rows, int64_t num_edges, int64_t H,
                                         int64_t head_dim, int dtype, int accumulate, void *ws, size_t ws_bytes,
                                         void *stream_) {
    const char *name = "pglb_gatv2_score_grad_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return gatv2_score_grad_entry<__nv_bfloat16>(name, indptr, cols, eid, f, ldf, attn, negative_slope, ds, out,
                                                     ldo, n_rows, num_edges, H, head_dim, accumulate, ws, ws_bytes,
                                                     stream_);
    return gatv2_score_grad_entry<__half>(name, indptr, cols, eid, f, ldf, attn, negative_slope, ds, out, ldo, n_rows,
                                          num_edges, H, head_dim, accumulate, ws, ws_bytes, stream_);
}
