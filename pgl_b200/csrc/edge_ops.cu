// edge_ops.cu -- edge-parallel and small per-row kernels of the send/recv path:
// send_uv (K3), gather/scatter rows (K6/K7), fused per-row edge softmax (K5), degree_norm.
#include "common.cuh"

namespace pglb {

constexpr int64_t SM_HUB_T = 256;  // rows longer than this use one CTA (8 warps) instead of one warp:
                                   // a single warp walks a long row as a chain of dependent loads

__device__ __forceinline__ float msg_apply(int op, float a, float b) {
    switch (op) {
        case PGLB_MSG_ADD: return __fadd_rn(a, b);
        case PGLB_MSG_SUB: return __fsub_rn(a, b);
        case PGLB_MSG_MUL: return __fmul_rn(a, b);
        case PGLB_MSG_DIV: return __fdiv_rn(a, b);
        default: return a;
    }
}

// ---- send_uv : out[e,:] = x[src[e],:] op y[dst[e],:] ----------------------------------
// 2^lsh lanes share one edge (lane l handles vectors l, l + 2^lsh, ...): row / lane come from
// shifts, not from a 64-bit division per element.
template <int VEC>
__global__ void __launch_bounds__(256) send_uv_kernel(const float *__restrict__ x,
                                                      const float *__restrict__ y,
                                                      const int64_t *__restrict__ src, int64_t ss,
                                                      const int64_t *__restrict__ dst, int64_t ds,
                                                      int64_t E, int D, int lsh, int op,
                                                      float *__restrict__ out) {
    const int dv = D / VEC;
    const int lanes = 1 << lsh;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = (int)(t0 & (lanes - 1));
    const int64_t estride = ((int64_t)gridDim.x * blockDim.x) >> lsh;
    for (int64_t e = t0 >> lsh; e < E; e += estride) {
        const int64_t s = __ldg((const long long *)src + e * ss);
        const int64_t d = __ldg((const long long *)dst + e * ds);
        const float *xr = x + s * D, *yr = y + d * D;
        float *orow = out + e * D;
        for (int v = lane; v < dv; v += lanes) {
            const int c = v * VEC;
            if (VEC == 4) {
                const float4 a = __ldg(reinterpret_cast<const float4 *>(xr + c));
                const float4 b = __ldg(reinterpret_cast<const float4 *>(yr + c));
                float4 r;
                r.x = msg_apply(op, a.x, b.x);
                r.y = msg_apply(op, a.y, b.y);
                r.z = msg_apply(op, a.z, b.z);
                r.w = msg_apply(op, a.w, b.w);
                __stcs(reinterpret_cast<float4 *>(orow + c), r);
            } else {
                orow[c] = msg_apply(op, __ldg(xr + c), __ldg(yr + c));
            }
        }
    }
}

// ---- gather / scatter rows -------------------------------------------------------------
// Small, fixed footprint (2 blocks of 256 threads per SM) with 8 independent 16-byte loads in
// flight per thread: 8.6 MB outstanding on 132 SMs, more than the ~1.5 MB (2 us x 770 GB/s) an NVLink peer
// needs and enough to keep HBM busy, while leaving most of every SM to a concurrently running
// aggregation kernel (the multi-GPU halo pull overlaps with the local-source aggregation).
constexpr int MV_UNROLL = 8;

template <int VEC, bool SCATTER>
__global__ void __launch_bounds__(256) move_rows_kernel(const float *__restrict__ x, int64_t ldx,
                                                        const int64_t *__restrict__ index,
                                                        int64_t istride, int64_t n, int D, int lsh,
                                                        float *__restrict__ out, int64_t ldo) {
    // 2^lsh lanes share a row (lane l moves vectors l, l + 2^lsh, ...); every thread keeps
    // MV_UNROLL rows in flight.
    const int dv = D / VEC;
    const int lanes = 1 << lsh;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = (int)(t0 & (lanes - 1));
    const int64_t rstride = ((int64_t)gridDim.x * blockDim.x) >> lsh;
    for (int64_t r0 = t0 >> lsh; r0 < n; r0 += rstride * MV_UNROLL) {
        for (int v = lane; v < dv; v += lanes) {
            const int c = v * VEC;
            float4 v4[MV_UNROLL];
            float v1[MV_UNROLL];
            int64_t dsto[MV_UNROLL];
#pragma unroll
            for (int u = 0; u < MV_UNROLL; ++u) {
                const int64_t r = r0 + u * rstride;
                dsto[u] = -1;
                if (r < n) {
                    const int64_t k = __ldg((const long long *)index + r * istride);
                    const int64_t rs = SCATTER ? r : k;
                    const int64_t rd = SCATTER ? k : r;
                    dsto[u] = rd * ldo + c;
                    if (VEC == 4) v4[u] = __ldg(reinterpret_cast<const float4 *>(x + rs * ldx + c));
                    else v1[u] = __ldg(x + rs * ldx + c);
                }
            }
#pragma unroll
            for (int u = 0; u < MV_UNROLL; ++u) {
                if (dsto[u] >= 0) {
                    if (VEC == 4) *reinterpret_cast<float4 *>(out + dsto[u]) = v4[u];
                    else out[dsto[u]] = v1[u];
                }
            }
        }
    }
}

// ---- fused edge softmax over CSR rows --------------------------------------------------
// A cooperative group of NT threads (a warp, or a whole CTA for long rows) owns one row.
// Thread t handles head (t % HP) of slots (t / HP), (t / HP) + NT/HP, ...
template <int NT>
__device__ __forceinline__ float group_reduce(float v, bool is_max, int hp, float *smem) {
    // reduce over threads with equal (t % hp); result valid in every thread
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        if (o >= hp) {
            const float t = __shfl_xor_sync(0xffffffffu, v, o);
            v = is_max ? fmaxf(v, t) : (v + t);
        }
    }
    if (NT > 32) {
        // now lanes 0..hp-1 of each warp hold the warp's value for head = lane
        const int wid = threadIdx.x >> 5;
        __syncthreads();
        if (lane < hp) smem[wid * 32 + lane] = v;
        __syncthreads();
        float r = smem[lane % hp];
        for (int w = 1; w < NT / 32; ++w) {
            const float t = smem[w * 32 + (lane % hp)];
            r = is_max ? fmaxf(r, t) : (r + t);
        }
        v = r;
    }
    return v;
}

// Where a row's logits come from.  pos(j): element index of slot j (also where the result goes);
// val(p, head): the logit.
struct LogitSrc {  // stored logits [E, H], optionally permuted through eid (original edge order)
    const int64_t *eid;
    const float *logits;
    int H;
    __device__ __forceinline__ int64_t pos(int64_t j) const {
        return eid ? __ldg((const long long *)eid + j) : j;
    }
    __device__ __forceinline__ float val(int64_t p, int64_t /*j*/, int head) const {
        return __ldg(logits + p * H + head);
    }
};
struct GatSrc {  // GAT attention logits recomputed on the fly, results in CSR slot order
    const int64_t *cols;
    const float *attn_src;
    float ad;  // attn_dst[row, head] of the calling thread
    float slope;
    int H;
    __device__ __forceinline__ int64_t pos(int64_t j) const { return j; }
    __device__ __forceinline__ float val(int64_t /*p*/, int64_t j, int head) const {
        const float v = __ldg(attn_src + __ldg((const long long *)cols + j) * H + head) + ad;
        return v >= 0.0f ? v : v * slope;
    }
};

template <int NT, typename Src>
__device__ __forceinline__ void softmax_row(const Src src, float *__restrict__ out, int64_t b,
                                            int64_t e, int H, int head, bool hact, int srow,
                                            int sstep, int hp, float *smem) {
    // every pass keeps 8 independent load chains in flight per thread: long rows (one CTA per hub
    // row) are latency bound otherwise
    constexpr int SU = 8;
    float m = -INFINITY;
    for (int64_t j0 = b + srow; j0 < e; j0 += (int64_t)sstep * SU) {
        float v[SU];
#pragma unroll
        for (int u = 0; u < SU; ++u) {
            const int64_t j = j0 + (int64_t)u * sstep;
            v[u] = -INFINITY;
            if (j < e && hact) v[u] = src.val(src.pos(j), j, head);
        }
#pragma unroll
        for (int u = 0; u < SU; ++u) m = fmaxf(m, v[u]);
    }
    m = group_reduce<NT>(m, true, hp, smem);
    float s = 0.0f;
    for (int64_t j0 = b + srow; j0 < e; j0 += (int64_t)sstep * SU) {
        float v[SU];
        bool ok[SU];
#pragma unroll
        for (int u = 0; u < SU; ++u) {
            const int64_t j = j0 + (int64_t)u * sstep;
            ok[u] = (j < e) && hact;
            v[u] = 0.0f;
            if (ok[u]) v[u] = src.val(src.pos(j), j, head);
        }
#pragma unroll
        for (int u = 0; u < SU; ++u)
            if (ok[u]) s += expf(v[u] - m);
    }
    s = group_reduce<NT>(s, false, hp, smem);
    for (int64_t j0 = b + srow; j0 < e; j0 += (int64_t)sstep * SU) {
        float v[SU];
        int64_t ids[SU];
#pragma unroll
        for (int u = 0; u < SU; ++u) {
            const int64_t j = j0 + (int64_t)u * sstep;
            ids[u] = -1;
            if (j < e && hact) {
                ids[u] = src.pos(j);
                v[u] = src.val(ids[u], j, head);
            }
        }
#pragma unroll
        for (int u = 0; u < SU; ++u)
            if (ids[u] >= 0) out[ids[u] * H + head] = __fdiv_rn(expf(v[u] - m), s);
    }
}

// MODE 0: stored logits (edge_softmax / segment_softmax); MODE 1: GAT logits on the fly
template <int MODE>
__global__ void __launch_bounds__(256) edge_softmax_warp_kernel(
    const int64_t *__restrict__ indptr, const int64_t *__restrict__ eid_or_cols,
    const float *__restrict__ logits_or_asrc, const float *__restrict__ attn_dst, float slope,
    float *__restrict__ out, int64_t n_rows, int H, int hp, unsigned long long *hub_count,
    int64_t *hub_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int head = blockIdx.y * hp + (lane % hp);
    const bool hact = head < H;
    for (int64_t r = warp; r < n_rows; r += nwarps) {
        const int64_t b = ld_ro(indptr + r), e = ld_ro(indptr + r + 1);
        if (e == b) continue;
        if (e - b > SM_HUB_T) {
            if (lane == 0 && blockIdx.y == 0) {
                unsigned long long s = atomicAdd(hub_count, 1ull);
                hub_rows[s] = r;
            }
            continue;
        }
        if (MODE == 0) {
            const LogitSrc src{eid_or_cols, logits_or_asrc, H};
            softmax_row<32>(src, out, b, e, H, head, hact, lane / hp, 32 / hp, hp, nullptr);
        } else {
            const GatSrc src{eid_or_cols, logits_or_asrc, hact ? __ldg(attn_dst + r * H + head) : 0.0f,
                             slope, H};
            softmax_row<32>(src, out, b, e, H, head, hact, lane / hp, 32 / hp, hp, nullptr);
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(256) edge_softmax_hub_kernel(
    const int64_t *__restrict__ indptr, const int64_t *__restrict__ eid_or_cols,
    const float *__restrict__ logits_or_asrc, const float *__restrict__ attn_dst, float slope,
    float *__restrict__ out, int H, int hp, const unsigned long long *hub_count,
    const int64_t *hub_rows) {
    __shared__ float smem[8 * 32];
    const int64_t n = (int64_t)*hub_count;
    const int t = threadIdx.x;
    const int head = blockIdx.y * hp + (t % hp);
    const bool hact = head < H;
    for (int64_t i = blockIdx.x; i < n; i += gridDim.x) {
        const int64_t r = hub_rows[i];
        const int64_t b = indptr[r], e = indptr[r + 1];
        if (MODE == 0) {
            const LogitSrc src{eid_or_cols, logits_or_asrc, H};
            softmax_row<256>(src, out, b, e, H, head, hact, t / hp, 256 / hp, hp, smem);
        } else {
            const GatSrc src{eid_or_cols, logits_or_asrc, hact ? __ldg(attn_dst + r * H + head) : 0.0f,
                             slope, H};
            softmax_row<256>(src, out, b, e, H, head, hact, t / hp, 256 / hp, hp, smem);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) degree_norm_kernel(const int64_t *__restrict__ degree,
                                                          int64_t n, float *__restrict__ norm) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        float d = (float)degree[i];
        d = fmaxf(d, 1.0f);
        norm[i] = __fdiv_rn(1.0f, __fsqrt_rn(d));
    }
}


// GATConv's two attention projections in one pass over the transformed features (reference pgl/nn/conv.py:323-326:
// attn_src = sum(feature * weight_src, -1), attn_dst = sum(feature * weight_dst, -1) -- four elementwise / reduce
// launches and two [N, H, Dh] temporaries there):  as[n,h] = <f[n,h,:], ws[h,:]>,  ad[n,h] = <f[n,h,:], wd[h,:]>.
// A warp per row, a float4 per lane, LPH = Dh / 4 lanes per head (shuffle reduce), weights in registers.
// T: element type of f (float, or the 16-bit type of pglb_head_dots_x16: 8 bytes per lane, widened exactly, then the
// float32 kernel's products and adds).  Weights and outputs are fp32.
template <int LPH, typename T>
__global__ void __launch_bounds__(256) head_dots_kernel(const T *__restrict__ f, int64_t ldf, int64_t n, int D,
                                                        int H, const float *__restrict__ ws,
                                                        const float *__restrict__ wd, float *__restrict__ as,
                                                        float *__restrict__ ad) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool act = lane * 4 < D;
    const int head = act ? lane / LPH : 0;
    const bool lead = act && (lane % LPH) == 0;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (act) {
        a = __ldg(reinterpret_cast<const float4 *>(ws + lane * 4));
        b = __ldg(reinterpret_cast<const float4 *>(wd + lane * 4));
    }
    auto head_sum = [&](float v) {
#pragma unroll
        for (int o = LPH / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    constexpr int U = 4;
    for (int64_t r0 = warp * U; r0 < n; r0 += nwarps * U) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (act && r0 + u < n) v[u] = ldg_row4<T>(f + (r0 + u) * ldf + lane * 4);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            // products rounded one by one and added in index order inside the lane, like the elementwise multiply +
            // sum they replace; the LPH partial sums are combined by the shuffle tree
            float s = __fmul_rn(v[u].x, a.x), d = __fmul_rn(v[u].x, b.x);
            s = __fadd_rn(s, __fmul_rn(v[u].y, a.y)); d = __fadd_rn(d, __fmul_rn(v[u].y, b.y));
            s = __fadd_rn(s, __fmul_rn(v[u].z, a.z)); d = __fadd_rn(d, __fmul_rn(v[u].z, b.z));
            s = __fadd_rn(s, __fmul_rn(v[u].w, a.w)); d = __fadd_rn(d, __fmul_rn(v[u].w, b.w));
            s = head_sum(s);
            d = head_sum(d);
            if (lead && r0 + u < n) {
                as[(r0 + u) * H + head] = s;
                ad[(r0 + u) * H + head] = d;
            }
        }
    }
}

static inline bool a16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int lane_shift(int64_t dv) {  // lanes per row = min(32, next pow2 >= dv)
    int l = 0;
    while ((1 << l) < dv && l < 5) ++l;
    return l;
}
static inline int grid_move(int64_t total) {
    int64_t b = (total + 256 * MV_UNROLL - 1) / (256 * MV_UNROLL);
    const int64_t cap = (int64_t)sm_count() * 2;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}
static inline int grid_for(int64_t total) {
    int64_t b = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 32;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_send_uv_f32(const float *x, const float *y, const int64_t *src,
                                int64_t src_stride, const int64_t *dst, int64_t dst_stride,
                                int64_t E, int64_t D, int msg_op, float *out, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(E >= 0 && D >= 0 && D <= INT32_MAX, PGLB_EINVAL, "pglb_send_uv_f32: bad size");
    PGLB_CHECK_ARG(msg_op >= PGLB_MSG_ADD && msg_op <= PGLB_MSG_DIV, PGLB_EINVAL,
                   "pglb_send_uv_f32: unknown msg_op %d", msg_op);
    if (E == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(x && y && src && dst && out, PGLB_EINVAL, "pglb_send_uv_f32: NULL pointer");
    PGLB_CHECK_ARG(src_stride >= 1 && dst_stride >= 1, PGLB_EINVAL, "pglb_send_uv_f32: bad stride");
    if (D % 4 == 0 && a16(x) && a16(y) && a16(out)) {
        const int l = lane_shift(D / 4);
        send_uv_kernel<4><<<grid_for(E << l), 256, 0, stream>>>(
            x, y, src, src_stride, dst, dst_stride, E, (int)D, l, msg_op, out);
    } else {
        const int l = lane_shift(D);
        send_uv_kernel<1><<<grid_for(E << l), 256, 0, stream>>>(x, y, src, src_stride, dst,
                                                                 dst_stride, E, (int)D, l, msg_op, out);
    }
    PGLB_LAUNCH_CHECK("send_uv_kernel");
    return PGLB_OK;
}

extern "C" int pglb_gather_rows_f32(const float *x, int64_t ldx, const int64_t *index,
                                    int64_t index_stride, int64_t n, int64_t D, float *out,
                                    int64_t ldo, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n >= 0 && D >= 0 && D <= INT32_MAX, PGLB_EINVAL, "pglb_gather_rows_f32: bad size");
    if (n == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(x && index && out, PGLB_EINVAL, "pglb_gather_rows_f32: NULL pointer");
    PGLB_CHECK_ARG(ldx >= D && ldo >= D && index_stride >= 1, PGLB_ESHAPE,
                   "pglb_gather_rows_f32: bad leading dimension / stride");
    if (D % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && a16(x) && a16(out))
        move_rows_kernel<4, false><<<grid_move(n << lane_shift(D / 4)), 256, 0, stream>>>(
            x, ldx, index, index_stride, n, (int)D, lane_shift(D / 4), out, ldo);
    else
        move_rows_kernel<1, false><<<grid_move(n << lane_shift(D)), 256, 0, stream>>>(
            x, ldx, index, index_stride, n, (int)D, lane_shift(D), out, ldo);
    PGLB_LAUNCH_CHECK("gather_rows_kernel");
    return PGLB_OK;
}

extern "C" int pglb_scatter_rows_f32(const float *x, int64_t ldx, const int64_t *index, int64_t n,
                                     int64_t D, float *out, int64_t ldo, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n >= 0 && D >= 0 && D <= INT32_MAX, PGLB_EINVAL, "pglb_scatter_rows_f32: bad size");
    if (n == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(x && index && out, PGLB_EINVAL, "pglb_scatter_rows_f32: NULL pointer");
    PGLB_CHECK_ARG(ldx >= D && ldo >= D, PGLB_ESHAPE, "pglb_scatter_rows_f32: bad leading dimension");
    if (D % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && a16(x) && a16(out))
        move_rows_kernel<4, true><<<grid_move(n << lane_shift(D / 4)), 256, 0, stream>>>(
            x, ldx, index, 1, n, (int)D, lane_shift(D / 4), out, ldo);
    else
        move_rows_kernel<1, true><<<grid_move(n << lane_shift(D)), 256, 0, stream>>>(
            x, ldx, index, 1, n, (int)D, lane_shift(D), out, ldo);
    PGLB_LAUNCH_CHECK("scatter_rows_kernel");
    return PGLB_OK;
}

extern "C" int pglb_edge_softmax_csr_ws(int64_t num_edges, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr && num_edges >= 0, PGLB_EINVAL,
                   "pglb_edge_softmax_csr_ws: bad args");
    *ws_bytes = 256 + sizeof(int64_t) * (size_t)(num_edges / (SM_HUB_T + 1) + 1);
    return PGLB_OK;
}

extern "C" int pglb_edge_softmax_csr_f32(const int64_t *indptr, const int64_t *eid,
                                         const float *logits, float *out, int64_t n_rows,
                                         int64_t E, int64_t H, void *ws, size_t ws_bytes,
                                         void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_rows >= 0 && E >= 0 && H >= 0 && H <= INT32_MAX, PGLB_EINVAL,
                   "pglb_edge_softmax_csr_f32: bad size");
    if (n_rows == 0 || E == 0 || H == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && logits && out, PGLB_EINVAL, "pglb_edge_softmax_csr_f32: NULL pointer");
    size_t need = 0;
    pglb_edge_softmax_csr_ws(E, &need);
    PGLB_CHECK_ARG(ws && ws_bytes >= need, PGLB_EWORKSPACE,
                   "pglb_edge_softmax_csr_f32: workspace of %zu bytes needed (got %zu)", need,
                   ws_bytes);
    unsigned long long *hub_count = reinterpret_cast<unsigned long long *>(ws);
    int64_t *hub_rows = reinterpret_cast<int64_t *>(reinterpret_cast<char *>(ws) + 256);
    PGLB_CUDA(cudaMemsetAsync(hub_count, 0, 8, stream));
    int hp = 1;
    while (hp < H && hp < 32) hp <<= 1;
    const int tiles = (int)((H + hp - 1) / hp);
    int64_t blocks = (n_rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 64;
    if (blocks > cap) blocks = cap;
    dim3 grid((unsigned)blocks, (unsigned)tiles);
    edge_softmax_warp_kernel<0><<<grid, 256, 0, stream>>>(indptr, eid, logits, nullptr, 0.0f, out, n_rows,
                                                          (int)H, hp, hub_count, hub_rows);
    PGLB_LAUNCH_CHECK("edge_softmax_warp_kernel");
    if (E > SM_HUB_T) {
        dim3 hgrid((unsigned)(sm_count() * 8), (unsigned)tiles);
        edge_softmax_hub_kernel<0><<<hgrid, 256, 0, stream>>>(indptr, eid, logits, nullptr, 0.0f, out,
                                                              (int)H, hp, hub_count, hub_rows);
        PGLB_LAUNCH_CHECK("edge_softmax_hub_kernel");
    }
    return PGLB_OK;
}

extern "C" int pglb_gat_attention_csr_f32(const int64_t *indptr, const int64_t *cols,
                                          const float *attn_src, const float *attn_dst,
                                          float negative_slope, float *alpha_slots, int64_t n_rows,
                                          int64_t E, int64_t H, void *ws, size_t ws_bytes,
                                          void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_rows >= 0 && E >= 0 && H >= 0 && H <= INT32_MAX, PGLB_EINVAL,
                   "pglb_gat_attention_csr_f32: bad size");
    if (n_rows == 0 || E == 0 || H == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && cols && attn_src && attn_dst && alpha_slots, PGLB_EINVAL,
                   "pglb_gat_attention_csr_f32: NULL pointer");
    size_t need = 0;
    pglb_edge_softmax_csr_ws(E, &need);
    PGLB_CHECK_ARG(ws && ws_bytes >= need, PGLB_EWORKSPACE,
                   "pglb_gat_attention_csr_f32: workspace of %zu bytes needed (got %zu)", need, ws_bytes);
    unsigned long long *hub_count = reinterpret_cast<unsigned long long *>(ws);
    int64_t *hub_rows = reinterpret_cast<int64_t *>(reinterpret_cast<char *>(ws) + 256);
    PGLB_CUDA(cudaMemsetAsync(hub_count, 0, 8, stream));
    int hp = 1;
    while (hp < H && hp < 32) hp <<= 1;
    const int tiles = (int)((H + hp - 1) / hp);
    int64_t blocks = (n_rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 64;
    if (blocks > cap) blocks = cap;
    dim3 grid((unsigned)blocks, (unsigned)tiles);
    edge_softmax_warp_kernel<1><<<grid, 256, 0, stream>>>(indptr, cols, attn_src, attn_dst, negative_slope,
                                                          alpha_slots, n_rows, (int)H, hp, hub_count,
                                                          hub_rows);
    PGLB_LAUNCH_CHECK("gat_attention_warp_kernel");
    if (E > SM_HUB_T) {
        dim3 hgrid((unsigned)(sm_count() * 8), (unsigned)tiles);
        edge_softmax_hub_kernel<1><<<hgrid, 256, 0, stream>>>(indptr, cols, attn_src, attn_dst,
                                                              negative_slope, alpha_slots, (int)H, hp,
                                                              hub_count, hub_rows);
        PGLB_LAUNCH_CHECK("gat_attention_hub_kernel");
    }
    return PGLB_OK;
}

extern "C" int pglb_degree_norm_f32(const int64_t *degree, int64_t n, float *norm, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n >= 0, PGLB_EINVAL, "pglb_degree_norm_f32: bad size");
    if (n == 0) return PGLB_OK;
    PGLB_CHECK_ARG(degree && norm, PGLB_EINVAL, "pglb_degree_norm_f32: NULL pointer");
    degree_norm_kernel<<<grid_for(n), 256, 0, stream>>>(degree, n, norm);
    PGLB_LAUNCH_CHECK("degree_norm_kernel");
    return PGLB_OK;
}

// The checks and the launch of both head-dots entries.  T: element type of f; rows 16-byte aligned for either type.
template <typename T>
static int head_dots_entry(const char *name, const void *f_, int64_t ldf, int64_t n, int64_t H, int64_t head_dim,
                           const float *w_src, const float *w_dst, float *attn_src, float *attn_dst, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const T *f = reinterpret_cast<const T *>(f_);
    PGLB_CHECK_ARG(n >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim, lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0, PGLB_EUNSUPPORTED,
                   "%s: needs H*head_dim <= 128 and head_dim in {4, 8, 16, 32, 64, 128}", name);
    if (n == 0) return PGLB_OK;
    PGLB_CHECK_ARG(f && w_src && w_dst && attn_src && attn_dst, PGLB_EINVAL, "%s: NULL pointer", name);
    PGLB_CHECK_ARG(ldf >= D && (ldf * (int64_t)sizeof(T)) % 16 == 0 && a16(f) && a16(w_src) && a16(w_dst), PGLB_ESHAPE,
                   "%s: rows / weights must be 16-byte aligned", name);
    const int grid = grid_for(n * 8);   // a warp per 4 rows
#define PGLB_HD(L) head_dots_kernel<L, T><<<grid, 256, 0, stream>>>(f, ldf, n, (int)D, (int)H, w_src, w_dst, attn_src, attn_dst)
    switch ((int)lph) {
        case 1: PGLB_HD(1); break;
        case 2: PGLB_HD(2); break;
        case 4: PGLB_HD(4); break;
        case 8: PGLB_HD(8); break;
        case 16: PGLB_HD(16); break;
        default: PGLB_HD(32); break;
    }
#undef PGLB_HD
    PGLB_LAUNCH_CHECK("head_dots_kernel");
    return PGLB_OK;
}

extern "C" int pglb_head_dots_f32(const float *f, int64_t ldf, int64_t n, int64_t H, int64_t head_dim,
                                  const float *w_src, const float *w_dst, float *attn_src, float *attn_dst,
                                  void *stream_) {
    return head_dots_entry<float>("pglb_head_dots_f32", f, ldf, n, H, head_dim, w_src, w_dst, attn_src, attn_dst,
                                  stream_);
}

extern "C" int pglb_head_dots_x16(const void *f, int64_t ldf, int64_t n, int64_t H, int64_t head_dim, int dtype,
                                  const float *w_src, const float *w_dst, float *attn_src, float *attn_dst,
                                  void *stream_) {
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_head_dots_x16: unknown dtype %d", dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return head_dots_entry<__nv_bfloat16>("pglb_head_dots_x16", f, ldf, n, H, head_dim, w_src, w_dst, attn_src,
                                              attn_dst, stream_);
    return head_dots_entry<__half>("pglb_head_dots_x16", f, ldf, n, H, head_dim, w_src, w_dst, attn_src, attn_dst,
                                   stream_);
}

// ---- packed column ids + source hotness (L2 residency hint) --------------------------------
namespace pglb {
__global__ void __launch_bounds__(256) col_count_kernel(const int64_t *__restrict__ cols, int64_t E,
                                                        int *__restrict__ count) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E;
         i += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(count + __ldcs((const long long *)cols + i), 1);
}
__global__ void __launch_bounds__(256) pack_cols_kernel(const int64_t *__restrict__ cols, int64_t E,
                                                        const int *__restrict__ count,
                                                        int64_t min_count,
                                                        uint32_t *__restrict__ packed) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = __ldcs((const long long *)cols + i);
        const uint32_t hot = ((int64_t)__ldg(count + c) >= min_count) ? 0x80000000u : 0u;
        packed[i] = (uint32_t)c | hot;
    }
}
}  // namespace pglb

extern "C" int pglb_pack_cols(const int64_t *cols, int64_t E, int64_t n_src, int32_t *count,
                              int64_t min_count, uint32_t *packed, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(E >= 0 && n_src >= 0, PGLB_EINVAL, "pglb_pack_cols: bad size");
    PGLB_CHECK_ARG(n_src < 0x7fffffffLL, PGLB_ESHAPE, "pglb_pack_cols: needs n_src < 2^31");
    if (n_src == 0 || E == 0) return PGLB_OK;
    PGLB_CHECK_ARG(count && packed && cols, PGLB_EINVAL, "pglb_pack_cols: NULL pointer");
    PGLB_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t) * n_src, stream));
    col_count_kernel<<<grid_for(E), 256, 0, stream>>>(cols, E, count);
    PGLB_LAUNCH_CHECK("col_count_kernel");
    pack_cols_kernel<<<grid_for(E), 256, 0, stream>>>(cols, E, count, min_count, packed);
    PGLB_LAUNCH_CHECK("pack_cols_kernel");
    return PGLB_OK;
}
