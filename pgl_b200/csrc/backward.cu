// backward.cu -- gradient kernels of the send/recv path (SURVEY.md section 8f rank 1).
// The reference gets these from Paddle autograd; here:
//   * sum / mean copy aggregation backward  = the forward kernel on the reverse CSR (no new code)
//   * send_ue_recv(mul) wrt the edge operand = per-head dot of x[src] and grad[dst]  (sddmm_dot)
//   * edge_softmax backward                 = alpha * (g - sum_row(alpha * g))
//   * max / min copy aggregation backward   = grad routed to the entries that equal the output
//   * fused GAT aggregation backward        = one edge kernel (attention weights rebuilt from the saved row
//     log-sum-exp, SDDMM dot, softmax / LeakyReLU backward) + the existing reverse-CSR aggregations
#include "common.cuh"

namespace pglb {

// out[e, h] = sum_k a[ia[e], h, k] * b[ib[e], h, k]
template <int VEC>
__global__ void __launch_bounds__(256) sddmm_dot_kernel(const float *__restrict__ a,
                                                        const float *__restrict__ b,
                                                        const int64_t *__restrict__ ia, int64_t sa,
                                                        const int64_t *__restrict__ ib, int64_t sb,
                                                        int64_t E, int H, int Dh,
                                                        float *__restrict__ out) {
    const int64_t total = E * H;
    const int64_t D = (int64_t)H * Dh;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = i / H;
        const int h = (int)(i - e * H);
        const float *pa = a + __ldg((const long long *)ia + e * sa) * D + (int64_t)h * Dh;
        const float *pb = b + __ldg((const long long *)ib + e * sb) * D + (int64_t)h * Dh;
        float acc = 0.0f;
        if (VEC == 4) {
            for (int k = 0; k < Dh; k += 4) {
                const float4 x = __ldg(reinterpret_cast<const float4 *>(pa + k));
                const float4 y = __ldg(reinterpret_cast<const float4 *>(pb + k));
                acc = fmaf(x.x, y.x, acc);
                acc = fmaf(x.y, y.y, acc);
                acc = fmaf(x.z, y.z, acc);
                acc = fmaf(x.w, y.w, acc);
            }
        } else {
            for (int k = 0; k < Dh; ++k) acc = fmaf(__ldg(pa + k), __ldg(pb + k), acc);
        }
        out[i] = acc;
    }
}

// per CSR row: s_h = sum_j alpha[e_j,h] * g[e_j,h];  gl[e_j,h] = alpha[e_j,h] * (g[e_j,h] - s_h)
__global__ void __launch_bounds__(256) edge_softmax_bwd_kernel(
    const int64_t *__restrict__ indptr, const int64_t *__restrict__ eid,
    const float *__restrict__ alpha, const float *__restrict__ g, float *__restrict__ gl,
    int64_t n_rows, int H, int hp) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int head = blockIdx.y * hp + (lane % hp);
    const int srow = lane / hp, sstep = 32 / hp;
    const bool hact = head < H;
    for (int64_t r = warp; r < n_rows; r += nwarps) {
        const int64_t b = ld_ro(indptr + r), e = ld_ro(indptr + r + 1);
        if (e == b) continue;
        float s = 0.0f;
        for (int64_t j = b + srow; j < e; j += sstep) {
            const int64_t id = eid ? __ldg((const long long *)eid + j) : j;
            if (hact) s = fmaf(__ldg(alpha + id * H + head), __ldg(g + id * H + head), s);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1)
            if (o >= hp) s += __shfl_xor_sync(0xffffffffu, s, o);
        for (int64_t j = b + srow; j < e; j += sstep) {
            const int64_t id = eid ? __ldg((const long long *)eid + j) : j;
            if (hact) gl[id * H + head] = __ldg(alpha + id * H + head) * (__ldg(g + id * H + head) - s);
        }
    }
}

// reverse (src-keyed) CSR: gx[s, k] = sum_{slots j of row s} g[cols[j], k] * (x[s, k] == out[cols[j], k])
__global__ void __launch_bounds__(256) maxmin_bwd_kernel(const int64_t *__restrict__ indptr,
                                                         const int64_t *__restrict__ cols,
                                                         const float *__restrict__ x,
                                                         const float *__restrict__ out,
                                                         const float *__restrict__ g,
                                                         float *__restrict__ gx, int64_t n_src,
                                                         int D) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = warp; s < n_src; s += nwarps) {
        const int64_t b = ld_ro(indptr + s), e = ld_ro(indptr + s + 1);
        for (int c = lane; c < D; c += 32) {
            const float xv = __ldg(x + s * D + c);
            float acc = 0.0f;
            for (int64_t j = b; j < e; ++j) {
                const int64_t d = ld_ro(cols + j);
                if (__ldg(out + d * D + c) == xv) acc += __ldg(g + d * D + c);
            }
            gx[s * D + c] = acc;
        }
    }
}


// Backward of the single-pass GAT aggregation (pglb_gat_fused_train_csr_f32), the per-edge part.  With
//   z = as[src,h] + ad[dst,h],  lz = leaky_relu(z),  alpha = exp(lz - lse[dst,h]),  out[dst,h,:] = sum alpha f[src,h,:]
// and G = d loss / d out:
//   d alpha = <G[dst,h,:], f[src,h,:]>,   d lz = alpha (d alpha - <G[dst,h,:], out[dst,h,:]>),   d z = d lz * leaky'(z)
//   (leaky'(z) = 1 for z > 0, slope otherwise).
// One launch rebuilds alpha and produces dz for every edge, both written in ORIGINAL edge order, which is what the
// reverse-CSR aggregations that finish the job read (grad f = sum over out-edges alpha G[dst]; grad as / grad ad =
// segment sums of dz over the src- / dst-CSR, exactly send_uv(add)'s backward).  Neither logits nor alpha were kept by
// the forward.  Walks the dst-CSR slots (rows[] = destination of every slot, so G / out / ad / lse are re-read only when
// the row changes); a warp owns 32 consecutive slots, the D/4 active lanes hold one float4 of the row each, LPH = Dh/4
// lanes form a head; four gathered feature rows are in flight per lane before the first dot product.
// T: element type of f, g and out (float, or the 16-bit type of pglb_gat_bwd_edge_x16: a lane reads 8 bytes and widens
// them exactly, and the arithmetic after that is the float32 kernel's).  a_s, a_d, lse, alpha_e and dz_e are fp32.
// DROP (attention dropout, pglb_gat_bwd_edge_drop_*): the forward was out = sum beta f[src] with beta = s m alpha
// (m = the keep bit of the slot and head, s = 1 / (1 - p)).  Then d alpha = s m <G, f[src]>, sum_k alpha_k d alpha_k
// = <G, out> is still delta, and the edge kernel writes beta in place of alpha (what grad f is aggregated with).  Each
// lane recomputes its own slot's keep word; the consume loop shuffles it along with the slot's row and edge id.
template <int LPH, typename T, bool DROP>
__global__ void __launch_bounds__(256) gat_bwd_edge_kernel(
    const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, const int64_t *__restrict__ eid,
    const T *__restrict__ f, int64_t ldf, const T *__restrict__ g, int64_t ldg,
    const T *__restrict__ out, int64_t ldo, const float *__restrict__ a_s, const float *__restrict__ a_d,
    const float *__restrict__ lse, float slope, int64_t E, int H, int D, float *__restrict__ alpha_e,
    float *__restrict__ dz_e, const AttnDrop drop) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool act = lane * 4 < D;
    const int head = act ? lane / LPH : 0;
    const bool lead = act && (lane % LPH) == 0;
    auto head_sum = [&](float v) {
#pragma unroll
        for (int o = LPH / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    auto dot4 = [](const float4 &a, const float4 &b) {
        return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
    };
    for (int64_t base = warp * 32; base < E; base += nwarps * 32) {
        const int64_t j = base + lane;
        const bool in = j < E;
        const long long r_l = in ? ld_stream(rows + j) : 0;
        const long long c_l = in ? ld_stream(cols + j) : 0;
        const long long i_l = in ? (eid ? ld_stream(eid + j) : j) : 0;
        unsigned kw_l = 0;
        if constexpr (DROP) kw_l = attn_keep_word(drop, (uint64_t)j, H);
        const int cnt = (E - base) < 32 ? (int)(E - base) : 32;
        long long cur = -1;
        float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float ad = 0.f, ls = 0.f, delta = 0.f;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            float4 fv[4];
            float as[4];
            long long rr[4], ii[4];
            unsigned kk[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int k = (k0 + u) & 31;
                const long long cc = __shfl_sync(0xffffffffu, c_l, k);
                rr[u] = __shfl_sync(0xffffffffu, r_l, k);
                ii[u] = __shfl_sync(0xffffffffu, i_l, k);
                if constexpr (DROP) kk[u] = __shfl_sync(0xffffffffu, kw_l, k);
                fv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                as[u] = 0.f;
                if (k0 + u < cnt && act) {
                    fv[u] = ldg_row4<T>(f + cc * ldf + lane * 4);
                    as[u] = __ldg(a_s + cc * H + head);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (k0 + u >= cnt) break;
                if (rr[u] != cur) {  // warp-uniform
                    cur = rr[u];
                    float d = 0.f;
                    if (act) {
                        g4 = ldg_row4<T>(g + cur * ldg + lane * 4);
                        const float4 o4 = ldg_row4<T>(out + cur * ldo + lane * 4);
                        ad = __ldg(a_d + cur * H + head);
                        ls = __ldg(lse + cur * H + head);
                        d = dot4(g4, o4);
                    }
                    delta = head_sum(d);
                }
                float da = head_sum(dot4(fv[u], g4));
                const float z = as[u] + ad;
                const bool pos = z > 0.0f;   // leaky_relu'(0) = slope, the convention of the framework's LeakyReLU backward
                const float alpha = expf((pos ? z : z * slope) - ls);
                float beta = alpha;
                if constexpr (DROP) {
                    const bool keep = (kk[u] >> head) & 1u;
                    da = keep ? drop.scale * da : 0.f;
                    beta = keep ? alpha * drop.scale : 0.f;
                }
                const float dl = alpha * (da - delta);
                if (lead) {
                    alpha_e[ii[u] * H + head] = beta;
                    dz_e[ii[u] * H + head] = pos ? dl : dl * slope;
                }
            }
        }
    }
}

// Backward of the single-pass dot-product attention (pglb_dot_attn_*), the per-edge part.  With
//   s = <q[dst,h,:], k[src,h,:]>,  a = exp(s - lse[dst,h]),  out[dst,h,:] = sum a v[src,h,:],  G = d loss / d out:
//   da = <G[dst,h,:], v[src,h,:]>,   delta = <G[dst,h,:], out[dst,h,:]>,   ds = a (da - delta)
// written, with beta = a (the weight grad v is aggregated with), as [E, H] fp32 in ORIGINAL edge order.  The walk is
// gat_bwd_edge_kernel's: dst-CSR slots, q / G / out / lse re-read only when the row changes, four slots' k and v rows
// in flight per lane.  s is formed by the forward's dot4_lane + head_sum_lanes, so it is the forward's score bit for bit.
// T: element type of q, k, v, G and out (16-bit rows are widened exactly; everything after is the fp32 kernel's).
// DROP: da = s m da and beta = m ? fl(a s) : 0 (m the slot and head's keep bit, s = 1 / (1 - p)); delta is unchanged.
// EF (pglb_dot_attn_e_*, launched as <LPH, T, DROP, true>): edge features e [E, D] in edge-id order; k + e and v + e
// (add4, as the forward forms them) take the places of k and v, and grad_e (nullable) gets
// grad_e[e,h,:] = ds q[dst,h,:] + beta G[dst,h,:], each edge's row written once by the lanes of its slot, in T.  EF is a
// trailing pack so the instantiations without edge features keep their names, <LPH, T, DROP>, in profiles and traces.
template <int LPH, typename T, bool DROP, bool... EF>
__global__ void __launch_bounds__(256) dot_attn_bwd_edge_kernel(
    const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, const int64_t *__restrict__ eid,
    const T *__restrict__ q, int64_t ldq, const T *__restrict__ k, int64_t ldk, const T *__restrict__ v, int64_t ldv,
    const T *__restrict__ g, int64_t ldg, const T *__restrict__ out, int64_t ldo, const float *__restrict__ lse,
    int64_t E, int H, int D, float *__restrict__ beta_e, float *__restrict__ ds_e, const AttnDrop drop,
    const T *__restrict__ e = nullptr, int64_t lde = 0, T *__restrict__ grad_e = nullptr, int64_t ldge = 0) {
    constexpr bool kEF = (false || ... || EF);
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool act = lane * 4 < D;
    const int head = act ? lane / LPH : 0;
    const bool lead = act && (lane % LPH) == 0;
    for (int64_t base = warp * 32; base < E; base += nwarps * 32) {
        const int64_t j = base + lane;
        const bool in = j < E;
        const long long r_l = in ? ld_stream(rows + j) : 0;
        const long long c_l = in ? ld_stream(cols + j) : 0;
        const long long i_l = in ? (eid ? ld_stream(eid + j) : j) : 0;
        unsigned kw_l = 0;
        if constexpr (DROP) kw_l = attn_keep_word(drop, (uint64_t)j, H);
        const int cnt = (E - base) < 32 ? (int)(E - base) : 32;
        long long cur = -1;
        float4 q4 = make_float4(0.f, 0.f, 0.f, 0.f), g4 = q4;
        float ls = 0.f, delta = 0.f;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            float4 kv[4], vv[4];
            long long rr[4], ii[4];
            unsigned kk[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int s = (k0 + u) & 31;
                const long long cc = __shfl_sync(0xffffffffu, c_l, s);
                rr[u] = __shfl_sync(0xffffffffu, r_l, s);
                ii[u] = __shfl_sync(0xffffffffu, i_l, s);
                if constexpr (DROP) kk[u] = __shfl_sync(0xffffffffu, kw_l, s);
                kv[u] = vv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (k0 + u < cnt && act) {
                    kv[u] = ldg_row4<T>(k + cc * ldk + lane * 4);
                    vv[u] = ldg_row4<T>(v + cc * ldv + lane * 4);
                    if constexpr (kEF) {
                        const float4 e4 = ldg_row4<T>(e + ii[u] * lde + lane * 4);
                        kv[u] = add4(kv[u], e4);
                        vv[u] = add4(vv[u], e4);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (k0 + u >= cnt) break;
                if (rr[u] != cur) {  // warp-uniform
                    cur = rr[u];
                    float d = 0.f;
                    if (act) {
                        q4 = ldg_row4<T>(q + cur * ldq + lane * 4);
                        g4 = ldg_row4<T>(g + cur * ldg + lane * 4);
                        d = dot4_lane(g4, ldg_row4<T>(out + cur * ldo + lane * 4));
                        ls = __ldg(lse + cur * H + head);
                    }
                    delta = head_sum_lanes(d, LPH);
                }
                const float sc = head_sum_lanes(dot4_lane(q4, kv[u]), LPH);
                float da = head_sum_lanes(dot4_lane(g4, vv[u]), LPH);
                const float a = expf(sc - ls);
                float beta = a;
                if constexpr (DROP) {
                    const bool keep = (kk[u] >> head) & 1u;
                    da = keep ? drop.scale * da : 0.f;
                    beta = keep ? a * drop.scale : 0.f;
                }
                if (lead) {
                    beta_e[ii[u] * H + head] = beta;
                    ds_e[ii[u] * H + head] = a * (da - delta);
                }
                if constexpr (kEF) {
                    if (grad_e && act) {
                        const float ds = a * (da - delta);
                        const float4 ge = make_float4(fmaf(beta, g4.x, ds * q4.x), fmaf(beta, g4.y, ds * q4.y),
                                                      fmaf(beta, g4.z, ds * q4.z), fmaf(beta, g4.w, ds * q4.w));
                        if constexpr (sizeof(T) == 4)
                            __stcs(reinterpret_cast<float4 *>(grad_e + ii[u] * ldge + lane * 4), ge);
                        else
                            __stcs(reinterpret_cast<uint2 *>(grad_e + ii[u] * ldge + lane * 4), round4<T>(ge));
                    }
                }
            }
        }
    }
}

// Backward of the single-pass GATv2 attention (pglb_gatv2_attn_*), the per-edge part, on dot_attn_bwd_edge_kernel's
// walk.  With z = f[src,h,:] + f[dst,h,:], s = sum_c a[h,c] lrelu(z_c), a = exp(s - lse[dst,h]), G = d loss / d out:
//   da = <G[dst,h,:], f[src,h,:]>,   delta = <G[dst,h,:], out[dst,h,:]>,   ds = a (da - delta)
// written, with beta = a, as [E, H] fp32 in ORIGINAL edge order.  s is formed by the forward's gatv2_lane +
// head_sum_lanes, so it is the forward's score bit for bit.  ga_part (nullable): grad a = sum_e ds lrelu(z), each block's
// share (its warps' lane sums added in warp order) at ga_part[blockIdx.x * 128 ...]; gatv2_ga_reduce_kernel adds the
// blocks in order.  The grid is fixed, so grad a is bit-identical run to run.  T: element type of f, G and out.
// DROP: da = s m da and beta = m ? fl(a s) : 0 (m the slot and head's keep bit, s = 1 / (1 - p)); delta is unchanged.
template <int LPH, typename T, bool DROP>
__global__ void __launch_bounds__(256) gatv2_bwd_edge_kernel(
    const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, const int64_t *__restrict__ eid,
    const T *__restrict__ f, int64_t ldf, const float *__restrict__ attn, float slope, const T *__restrict__ g,
    int64_t ldg, const T *__restrict__ out, int64_t ldo, const float *__restrict__ lse, int64_t E, int H, int D,
    float *__restrict__ beta_e, float *__restrict__ ds_e, float *__restrict__ ga_part, const AttnDrop drop) {
    __shared__ float4 ga_warp[8][32];
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool act = lane * 4 < D;
    const int head = act ? lane / LPH : 0;
    const bool lead = act && (lane % LPH) == 0;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a4 = act ? __ldg(reinterpret_cast<const float4 *>(attn) + lane) : zero;
    float4 ga = zero;
    for (int64_t base = warp * 32; base < E; base += nwarps * 32) {
        const int64_t j = base + lane;
        const bool in = j < E;
        const long long r_l = in ? ld_stream(rows + j) : 0;
        const long long c_l = in ? ld_stream(cols + j) : 0;
        const long long i_l = in ? (eid ? ld_stream(eid + j) : j) : 0;
        unsigned kw_l = 0;
        if constexpr (DROP) kw_l = attn_keep_word(drop, (uint64_t)j, H);
        const int cnt = (E - base) < 32 ? (int)(E - base) : 32;
        long long cur = -1;
        float4 fd = zero, g4 = zero;
        float ls = 0.f, delta = 0.f;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            float4 fs[4];
            long long rr[4], ii[4];
            unsigned kk[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int s = (k0 + u) & 31;
                const long long cc = __shfl_sync(0xffffffffu, c_l, s);
                rr[u] = __shfl_sync(0xffffffffu, r_l, s);
                ii[u] = __shfl_sync(0xffffffffu, i_l, s);
                if constexpr (DROP) kk[u] = __shfl_sync(0xffffffffu, kw_l, s);
                fs[u] = zero;
                if (k0 + u < cnt && act) fs[u] = ldg_row4<T>(f + cc * ldf + lane * 4);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (k0 + u >= cnt) break;
                if (rr[u] != cur) {  // warp-uniform
                    cur = rr[u];
                    float d = 0.f;
                    if (act) {
                        fd = ldg_row4<T>(f + cur * ldf + lane * 4);
                        g4 = ldg_row4<T>(g + cur * ldg + lane * 4);
                        d = dot4_lane(g4, ldg_row4<T>(out + cur * ldo + lane * 4));
                        ls = __ldg(lse + cur * H + head);
                    }
                    delta = head_sum_lanes(d, LPH);
                }
                const float sc = head_sum_lanes(gatv2_lane(a4, fs[u], fd, slope), LPH);
                float da = head_sum_lanes(dot4_lane(g4, fs[u]), LPH);
                const float a = expf(sc - ls);
                float beta = a;
                if constexpr (DROP) {
                    const bool keep = (kk[u] >> head) & 1u;
                    da = keep ? drop.scale * da : 0.f;
                    beta = keep ? a * drop.scale : 0.f;
                }
                const float ds = a * (da - delta);
                if (lead) {
                    beta_e[ii[u] * H + head] = beta;
                    ds_e[ii[u] * H + head] = ds;
                }
                ga.x = fmaf(ds, lrelu_of(fs[u].x + fd.x, slope), ga.x);
                ga.y = fmaf(ds, lrelu_of(fs[u].y + fd.y, slope), ga.y);
                ga.z = fmaf(ds, lrelu_of(fs[u].z + fd.z, slope), ga.z);
                ga.w = fmaf(ds, lrelu_of(fs[u].w + fd.w, slope), ga.w);
            }
        }
    }
    if (ga_part == nullptr) return;   // uniform over the grid
    ga_warp[threadIdx.x >> 5][lane] = ga;
    __syncthreads();
    if (threadIdx.x < 32) {
        float4 t = ga_warp[0][lane];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
            const float4 v = ga_warp[w][lane];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        reinterpret_cast<float4 *>(ga_part + (int64_t)blockIdx.x * 128)[lane] = t;
    }
}

// Backward of the single-pass FAConv aggregation (pglb_fa_attn_*), the per-edge part, on gat_bwd_edge_kernel's walk of
// the dst-CSR slots (rows[] = destination of every slot).  With (t, w) = fa_weight(g_src[src], g_dst[dst], norm[src],
// norm[dst]) rebuilt -- w the forward's weight bit for bit -- and G = d loss / d out:
//   beta_e = w,   dz_e = keep s ((norm[src] norm[dst]) (1 - t^2)) <G[dst,:], f[src,:]>     (keep s = 1 without dropout)
// both [E] fp32 in ORIGINAL edge order: grad f = sum over out-edges of beta G[dst], grad g_src / grad g_dst = segment
// sums of dz over the src- / dst-CSR.  rec: [n] node records (g_src, norm, g_dst, 0).  A warp owns 32 consecutive
// slots; each lane loads its own slot's column, edge id, source record (and, DROP, keep word) and the consume loop shuffles
// them; the D / 4 active lanes hold one float4 of the rows and the dot is summed over the warp.  T: element type of f
// and G (16-bit rows are widened exactly; everything after that is the float32 kernel's arithmetic).
template <typename T, bool DROP>
__global__ void __launch_bounds__(256) fa_bwd_edge_kernel(
    const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, const int64_t *__restrict__ eid,
    const T *__restrict__ f, int64_t ldf, const float4 *__restrict__ rec, const T *__restrict__ g, int64_t ldg,
    int64_t E, int D, float *__restrict__ beta_e, float *__restrict__ dz_e, const AttnDrop drop) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool act = lane * 4 < D;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t base = warp * 32; base < E; base += nwarps * 32) {
        const int64_t j = base + lane;
        const bool in = j < E;
        const long long r_l = in ? ld_stream(rows + j) : 0;
        const long long c_l = in ? ld_stream(cols + j) : 0;
        const long long i_l = in ? (eid ? ld_stream(eid + j) : j) : 0;
        const float4 rs_l = in ? __ldg(rec + c_l) : zero;   // the slot's source record
        unsigned kw_l = 0;
        if constexpr (DROP) kw_l = attn_keep_word(drop, (uint64_t)j, 4);
        const int cnt = (E - base) < 32 ? (int)(E - base) : 32;
        long long cur = -1;
        float4 g4 = zero;
        float gd = 0.f, nd = 0.f;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            float4 fs[4];
            long long rr[4], ii[4];
            float gs[4], nu[4];
            unsigned kk[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int s = (k0 + u) & 31;
                const long long cc = __shfl_sync(0xffffffffu, c_l, s);
                rr[u] = __shfl_sync(0xffffffffu, r_l, s);
                ii[u] = __shfl_sync(0xffffffffu, i_l, s);
                gs[u] = __shfl_sync(0xffffffffu, rs_l.x, s);
                nu[u] = __shfl_sync(0xffffffffu, rs_l.y, s);
                kk[u] = 1u;
                if constexpr (DROP) kk[u] = __shfl_sync(0xffffffffu, kw_l, s);
                fs[u] = zero;
                if (k0 + u < cnt && act) fs[u] = ldg_row4<T>(f + cc * ldf + lane * 4);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (k0 + u >= cnt) break;
                if (rr[u] != cur) {  // warp-uniform
                    cur = rr[u];
                    if (act) g4 = ldg_row4<T>(g + cur * ldg + lane * 4);
                    const float4 rd = __ldg(rec + cur);
                    gd = rd.z;
                    nd = rd.y;
                }
                const float dot = head_sum_lanes(dot4_lane(g4, fs[u]), 32);
                const bool keep = kk[u] & 1u;
                float t;
                const float w = fa_weight<DROP>(gs[u], gd, nu[u], nd, keep, drop.scale, &t);
                float dz = ((nu[u] * nd) * (1.0f - t * t)) * dot;
                if constexpr (DROP) dz = keep ? drop.scale * dz : 0.0f;
                if (lane == 0) {
                    beta_e[ii[u]] = w;
                    dz_e[ii[u]] = dz;
                }
            }
        }
    }
}

// grad a[c] = sum over the nb blocks' shares ga_part[b * 128 + c], in a fixed order: block c of the grid, thread t adds
// b = t, t + 256, ..., then a fixed tree over the threads.
__global__ void __launch_bounds__(256) gatv2_ga_reduce_kernel(const float *__restrict__ ga_part, int nb,
                                                              float *__restrict__ grad_attn) {
    __shared__ float red[256];
    const int c = blockIdx.x, t = threadIdx.x;
    float v = 0.f;
    for (int b = t; b < nb; b += 256) v += ga_part[(int64_t)b * 128 + c];
    red[t] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o) red[t] += red[t + o];
        __syncthreads();
    }
    if (t == 0) grad_attn[c] = red[0];
}

static inline int grid_of(int64_t total, int cap_mult) {
    int64_t b = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * cap_mult;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_sddmm_dot_f32(const float *a, const float *b, const int64_t *ia, int64_t ia_stride,
                                  const int64_t *ib, int64_t ib_stride, int64_t E, int64_t H,
                                  int64_t Dh, float *out, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(E >= 0 && H >= 0 && Dh >= 0 && H * Dh <= INT32_MAX, PGLB_EINVAL,
                   "pglb_sddmm_dot_f32: bad size");
    if (E == 0 || H == 0) return PGLB_OK;
    PGLB_CHECK_ARG(a && b && ia && ib && out, PGLB_EINVAL, "pglb_sddmm_dot_f32: NULL pointer");
    PGLB_CHECK_ARG(ia_stride >= 1 && ib_stride >= 1, PGLB_EINVAL, "pglb_sddmm_dot_f32: bad stride");
    const bool v4 = (Dh % 4 == 0) && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15u) == 0;
    if (v4)
        sddmm_dot_kernel<4><<<grid_of(E * H, 32), 256, 0, stream>>>(a, b, ia, ia_stride, ib, ib_stride,
                                                                    E, (int)H, (int)Dh, out);
    else
        sddmm_dot_kernel<1><<<grid_of(E * H, 32), 256, 0, stream>>>(a, b, ia, ia_stride, ib, ib_stride,
                                                                    E, (int)H, (int)Dh, out);
    PGLB_LAUNCH_CHECK("sddmm_dot_kernel");
    return PGLB_OK;
}

extern "C" int pglb_edge_softmax_bwd_csr_f32(const int64_t *indptr, const int64_t *eid,
                                             const float *alpha, const float *grad,
                                             float *grad_logits, int64_t n_rows, int64_t E,
                                             int64_t H, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_rows >= 0 && E >= 0 && H >= 0 && H <= INT32_MAX, PGLB_EINVAL,
                   "pglb_edge_softmax_bwd_csr_f32: bad size");
    if (n_rows == 0 || E == 0 || H == 0) return PGLB_OK;
    PGLB_CHECK_ARG(indptr && alpha && grad && grad_logits, PGLB_EINVAL,
                   "pglb_edge_softmax_bwd_csr_f32: NULL pointer");
    int hp = 1;
    while (hp < H && hp < 32) hp <<= 1;
    const int tiles = (int)((H + hp - 1) / hp);
    dim3 grid((unsigned)grid_of(n_rows * 32, 64), (unsigned)tiles);
    edge_softmax_bwd_kernel<<<grid, 256, 0, stream>>>(indptr, eid, alpha, grad, grad_logits, n_rows,
                                                      (int)H, hp);
    PGLB_LAUNCH_CHECK("edge_softmax_bwd_kernel");
    return PGLB_OK;
}

// The checks and the launch of both edge-backward entries.  T: element type of f, grad_out and out; their rows are
// 16-byte aligned (ld * sizeof(T) % 16 == 0) for either type.
// drop (nullable): the attention-dropout stream of the DROP kernel (H % 4 == 0 and H <= 32 then).
template <typename T>
static int gat_bwd_edge_entry(const char *name, const int64_t *rows, const int64_t *cols, const int64_t *eid,
                              const void *f_, int64_t ldf, const void *grad_out_, int64_t ldg, const void *out_,
                              int64_t ldo, const float *attn_src, const float *attn_dst, const float *lse,
                              float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim, float *alpha_e,
                              float *dz_e, void *stream_, const AttnDrop *drop = nullptr) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const T *f = reinterpret_cast<const T *>(f_), *grad_out = reinterpret_cast<const T *>(grad_out_),
            *out = reinterpret_cast<const T *>(out_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    const int64_t lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0, PGLB_EUNSUPPORTED,
                   "%s: needs H*head_dim <= 128 and head_dim in {4, 8, 16, 32, 64, 128}", name);
    PGLB_CHECK_ARG(!drop || H % 4 == 0, PGLB_EUNSUPPORTED, "%s: needs H %% 4 == 0", name);
    if (num_edges == 0) return PGLB_OK;
    PGLB_CHECK_ARG(rows && cols && f && grad_out && out && attn_src && attn_dst && lse && alpha_e && dz_e, PGLB_EINVAL,
                   "%s: NULL pointer", name);
    auto a16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    PGLB_CHECK_ARG(ldf >= D && ldg >= D && ldo >= D && (ldf * B) % 16 == 0 && (ldg * B) % 16 == 0 &&
                       (ldo * B) % 16 == 0 && a16(f) && a16(grad_out) && a16(out),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    const int grid = grid_of(num_edges * 1, 64);  // a warp per 32 slots, grid-stride
#define PGLB_GBE(L)                                                                                                   \
    do {                                                                                                              \
        if (drop)                                                                                                     \
            gat_bwd_edge_kernel<L, T, true><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, grad_out, ldg, out,    \
                                                                      ldo, attn_src, attn_dst, lse, negative_slope,   \
                                                                      num_edges, (int)H, (int)D, alpha_e, dz_e,       \
                                                                      *drop);                                         \
        else                                                                                                          \
            gat_bwd_edge_kernel<L, T, false><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, grad_out, ldg, out,   \
                                                                       ldo, attn_src, attn_dst, lse, negative_slope,  \
                                                                       num_edges, (int)H, (int)D, alpha_e, dz_e,      \
                                                                       AttnDrop{});                                   \
    } while (0)
    switch ((int)lph) {
        case 1: PGLB_GBE(1); break;
        case 2: PGLB_GBE(2); break;
        case 4: PGLB_GBE(4); break;
        case 8: PGLB_GBE(8); break;
        case 16: PGLB_GBE(16); break;
        default: PGLB_GBE(32); break;
    }
#undef PGLB_GBE
    PGLB_LAUNCH_CHECK("gat_bwd_edge_kernel");
    return PGLB_OK;
}

extern "C" int pglb_gat_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                                     int64_t ldf, const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                     const float *attn_src, const float *attn_dst, const float *lse,
                                     float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim,
                                     float *alpha_e, float *dz_e, void *stream_) {
    return gat_bwd_edge_entry<float>("pglb_gat_bwd_edge_f32", rows, cols, eid, f, ldf, grad_out, ldg, out, ldo,
                                     attn_src, attn_dst, lse, negative_slope, num_edges, H, head_dim, alpha_e, dz_e,
                                     stream_);
}

extern "C" int pglb_gat_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                     int64_t ldf, const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                     const float *attn_src, const float *attn_dst, const float *lse,
                                     float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                                     float *alpha_e, float *dz_e, void *stream_) {
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL,
                   "pglb_gat_bwd_edge_x16: unknown dtype %d", dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return gat_bwd_edge_entry<__nv_bfloat16>("pglb_gat_bwd_edge_x16", rows, cols, eid, f, ldf, grad_out, ldg, out,
                                                 ldo, attn_src, attn_dst, lse, negative_slope, num_edges, H, head_dim,
                                                 alpha_e, dz_e, stream_);
    return gat_bwd_edge_entry<__half>("pglb_gat_bwd_edge_x16", rows, cols, eid, f, ldf, grad_out, ldg, out, ldo,
                                      attn_src, attn_dst, lse, negative_slope, num_edges, H, head_dim, alpha_e, dz_e,
                                      stream_);
}

// Edge backward with attention dropout (include/pglb.h): the edge entries' arguments plus attn_drop, seed, offset,
// which are checked first, before any CUDA call.
extern "C" int pglb_gat_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                                          int64_t ldf, const float *grad_out, int64_t ldg, const float *out,
                                          int64_t ldo, const float *attn_src, const float *attn_dst, const float *lse,
                                          float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim,
                                          float attn_drop, uint64_t seed, uint64_t offset, float *alpha_e,
                                          float *dz_e, void *stream_) {
    const char *name = "pglb_gat_bwd_edge_drop_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return gat_bwd_edge_entry<float>(name, rows, cols, eid, f, ldf, grad_out, ldg, out, ldo, attn_src, attn_dst, lse,
                                     negative_slope, num_edges, H, head_dim, alpha_e, dz_e, stream_, &drop);
}

extern "C" int pglb_gat_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                          int64_t ldf, const void *grad_out, int64_t ldg, const void *out,
                                          int64_t ldo, const float *attn_src, const float *attn_dst, const float *lse,
                                          float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim,
                                          int dtype, float attn_drop, uint64_t seed, uint64_t offset, float *alpha_e,
                                          float *dz_e, void *stream_) {
    const char *name = "pglb_gat_bwd_edge_drop_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return gat_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, f, ldf, grad_out, ldg, out, ldo, attn_src,
                                                 attn_dst, lse, negative_slope, num_edges, H, head_dim, alpha_e, dz_e,
                                                 stream_, &drop);
    return gat_bwd_edge_entry<__half>(name, rows, cols, eid, f, ldf, grad_out, ldg, out, ldo, attn_src, attn_dst, lse,
                                      negative_slope, num_edges, H, head_dim, alpha_e, dz_e, stream_, &drop);
}

// The checks and the launch of the dot-product attention's edge-backward entries (include/pglb.h).  T: element type of
// q, k, v, e, grad_out, out and grad_e, rows 16-byte aligned.  drop (nullable): the attention-dropout stream (H % 4 == 0
// then).  ef: an edge-feature entry (pglb_dot_attn_e_bwd_edge_*, the kernel's EF): e must be given, grad_e is
// nullable.
template <typename T>
static int dot_attn_bwd_edge_entry(const char *name, const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                   const void *q_, int64_t ldq, const void *k_, int64_t ldk, const void *v_, int64_t ldv,
                                   const void *g_, int64_t ldg, const void *out_, int64_t ldo, const float *lse,
                                   int64_t num_edges, int64_t H, int64_t head_dim, float *beta_e, float *ds_e,
                                   void *stream_, const AttnDrop *drop, bool ef = false, const void *e_ = nullptr,
                                   int64_t lde = 0, void *grad_e_ = nullptr, int64_t ldge = 0) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const T *q = reinterpret_cast<const T *>(q_), *k = reinterpret_cast<const T *>(k_),
            *v = reinterpret_cast<const T *>(v_), *g = reinterpret_cast<const T *>(g_),
            *out = reinterpret_cast<const T *>(out_), *e = reinterpret_cast<const T *>(e_);
    T *grad_e = reinterpret_cast<T *>(grad_e_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    const int64_t lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0, PGLB_EUNSUPPORTED,
                   "%s: needs H*head_dim <= 128 and head_dim in {4, 8, 16, 32, 64, 128}", name);
    PGLB_CHECK_ARG(!drop || H % 4 == 0, PGLB_EUNSUPPORTED, "%s: needs H %% 4 == 0", name);
    if (num_edges == 0) return PGLB_OK;
    PGLB_CHECK_ARG(rows && cols && q && k && v && g && out && lse && beta_e && ds_e && (!ef || e), PGLB_EINVAL,
                   "%s: NULL pointer", name);
    auto a16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    PGLB_CHECK_ARG(ldq >= D && ldk >= D && ldv >= D && ldg >= D && ldo >= D && (ldq * B) % 16 == 0 &&
                       (ldk * B) % 16 == 0 && (ldv * B) % 16 == 0 && (ldg * B) % 16 == 0 && (ldo * B) % 16 == 0 &&
                       a16(q) && a16(k) && a16(v) && a16(g) && a16(out),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    PGLB_CHECK_ARG(!ef || (lde >= D && (lde * B) % 16 == 0 && a16(e) &&
                           (!grad_e || (ldge >= D && (ldge * B) % 16 == 0 && a16(grad_e)))),
                   PGLB_ESHAPE, "%s: e / grad_e rows must be 16-byte aligned", name);
    const int grid = grid_of(num_edges, 64);  // a warp per 32 slots, grid-stride
    const AttnDrop dr = drop ? *drop : AttnDrop{};
#define PGLB_DBE(L)                                                                                                   \
    do {                                                                                                              \
        if (ef && drop)                                                                                               \
            dot_attn_bwd_edge_kernel<L, T, true, true><<<grid, 256, 0, stream>>>(                                     \
                rows, cols, eid, q, ldq, k, ldk, v, ldv, g, ldg, out, ldo, lse, num_edges, (int)H, (int)D, beta_e,    \
                ds_e, dr, e, lde, grad_e, ldge);                                                                      \
        else if (ef)                                                                                                  \
            dot_attn_bwd_edge_kernel<L, T, false, true><<<grid, 256, 0, stream>>>(                                    \
                rows, cols, eid, q, ldq, k, ldk, v, ldv, g, ldg, out, ldo, lse, num_edges, (int)H, (int)D, beta_e,    \
                ds_e, dr, e, lde, grad_e, ldge);                                                                      \
        else if (drop)                                                                                                \
            dot_attn_bwd_edge_kernel<L, T, true><<<grid, 256, 0, stream>>>(rows, cols, eid, q, ldq, k, ldk, v, ldv,   \
                                                                           g, ldg, out, ldo, lse, num_edges, (int)H,  \
                                                                           (int)D, beta_e, ds_e, dr);                 \
        else                                                                                                          \
            dot_attn_bwd_edge_kernel<L, T, false><<<grid, 256, 0, stream>>>(rows, cols, eid, q, ldq, k, ldk, v, ldv,  \
                                                                            g, ldg, out, ldo, lse, num_edges, (int)H, \
                                                                            (int)D, beta_e, ds_e, dr);                \
    } while (0)
    switch ((int)lph) {
        case 1: PGLB_DBE(1); break;
        case 2: PGLB_DBE(2); break;
        case 4: PGLB_DBE(4); break;
        case 8: PGLB_DBE(8); break;
        case 16: PGLB_DBE(16); break;
        default: PGLB_DBE(32); break;
    }
#undef PGLB_DBE
    PGLB_LAUNCH_CHECK("dot_attn_bwd_edge_kernel");
    return PGLB_OK;
}

extern "C" int pglb_dot_attn_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *q,
                                          int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv,
                                          const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                          const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                          float *beta_e, float *ds_e, void *stream_) {
    return dot_attn_bwd_edge_entry<float>("pglb_dot_attn_bwd_edge_f32", rows, cols, eid, q, ldq, k, ldk, v, ldv,
                                          grad_out, ldg, out, ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_,
                                          nullptr);
}

extern "C" int pglb_dot_attn_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *q,
                                          int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                          const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                          const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                                          float *beta_e, float *ds_e, void *stream_) {
    const char *name = "pglb_dot_attn_bwd_edge_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return dot_attn_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out,
                                                      ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_, nullptr);
    return dot_attn_bwd_edge_entry<__half>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                           num_edges, H, head_dim, beta_e, ds_e, stream_, nullptr);
}

extern "C" int pglb_dot_attn_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                               const float *q, int64_t ldq, const float *k, int64_t ldk, const float *v,
                                               int64_t ldv, const float *grad_out, int64_t ldg, const float *out,
                                               int64_t ldo, const float *lse, int64_t num_edges, int64_t H,
                                               int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                               float *beta_e, float *ds_e, void *stream_) {
    const char *name = "pglb_dot_attn_bwd_edge_drop_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return dot_attn_bwd_edge_entry<float>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                          num_edges, H, head_dim, beta_e, ds_e, stream_, &drop);
}

extern "C" int pglb_dot_attn_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                               const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v,
                                               int64_t ldv, const void *grad_out, int64_t ldg, const void *out,
                                               int64_t ldo, const float *lse, int64_t num_edges, int64_t H,
                                               int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                               uint64_t offset, float *beta_e, float *ds_e, void *stream_) {
    const char *name = "pglb_dot_attn_bwd_edge_drop_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return dot_attn_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out,
                                                      ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_, &drop);
    return dot_attn_bwd_edge_entry<__half>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                           num_edges, H, head_dim, beta_e, ds_e, stream_, &drop);
}

// Edge backward with edge features (include/pglb.h): the pglb_dot_attn_bwd_edge_* arguments plus e [num_edges, H *
// head_dim] in edge-id order (row stride lde) and grad_e (nullable, row stride ldge).
extern "C" int pglb_dot_attn_e_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                            const float *q, int64_t ldq, const float *k, int64_t ldk, const float *v,
                                            int64_t ldv, const float *e, int64_t lde, const float *grad_out,
                                            int64_t ldg, const float *out, int64_t ldo, const float *lse,
                                            int64_t num_edges, int64_t H, int64_t head_dim, float *beta_e, float *ds_e,
                                            float *grad_e, int64_t ldge, void *stream_) {
    return dot_attn_bwd_edge_entry<float>("pglb_dot_attn_e_bwd_edge_f32", rows, cols, eid, q, ldq, k, ldk, v, ldv,
                                          grad_out, ldg, out, ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_,
                                          nullptr, true, e, lde, grad_e, ldge);
}

extern "C" int pglb_dot_attn_e_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                            const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v,
                                            int64_t ldv, const void *e, int64_t lde, const void *grad_out,
                                            int64_t ldg, const void *out, int64_t ldo, const float *lse,
                                            int64_t num_edges, int64_t H, int64_t head_dim, int dtype, float *beta_e,
                                            float *ds_e, void *grad_e, int64_t ldge, void *stream_) {
    const char *name = "pglb_dot_attn_e_bwd_edge_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return dot_attn_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out,
                                                      ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_, nullptr,
                                                      true, e, lde, grad_e, ldge);
    return dot_attn_bwd_edge_entry<__half>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                           num_edges, H, head_dim, beta_e, ds_e, stream_, nullptr, true, e, lde,
                                           grad_e, ldge);
}

extern "C" int pglb_dot_attn_e_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                                 const float *q, int64_t ldq, const float *k, int64_t ldk,
                                                 const float *v, int64_t ldv, const float *e, int64_t lde,
                                                 const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                                 const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                                 float attn_drop, uint64_t seed, uint64_t offset, float *beta_e,
                                                 float *ds_e, float *grad_e, int64_t ldge, void *stream_) {
    const char *name = "pglb_dot_attn_e_bwd_edge_drop_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return dot_attn_bwd_edge_entry<float>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                          num_edges, H, head_dim, beta_e, ds_e, stream_, &drop, true, e, lde, grad_e,
                                          ldge);
}

extern "C" int pglb_dot_attn_e_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                                 const void *q, int64_t ldq, const void *k, int64_t ldk,
                                                 const void *v, int64_t ldv, const void *e, int64_t lde,
                                                 const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                                 const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                                 int dtype, float attn_drop, uint64_t seed, uint64_t offset,
                                                 float *beta_e, float *ds_e, void *grad_e, int64_t ldge,
                                                 void *stream_) {
    const char *name = "pglb_dot_attn_e_bwd_edge_drop_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return dot_attn_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out,
                                                      ldo, lse, num_edges, H, head_dim, beta_e, ds_e, stream_, &drop,
                                                      true, e, lde, grad_e, ldge);
    return dot_attn_bwd_edge_entry<__half>(name, rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse,
                                           num_edges, H, head_dim, beta_e, ds_e, stream_, &drop, true, e, lde, grad_e,
                                           ldge);
}

// The checks and the launch of the GATv2 edge-backward entries (include/pglb.h).  T: element type of f, grad_out and
// out, rows 16-byte aligned.  drop (nullable): the attention-dropout stream (H % 4 == 0 then).
static size_t gatv2_bwd_edge_ws_bytes(int64_t num_edges) { return (size_t)grid_of(num_edges, 64) * 128 * 4; }

template <typename T>
static int gatv2_bwd_edge_entry(const char *name, const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                const void *f_, int64_t ldf, const float *attn, float slope, const void *g_,
                                int64_t ldg, const void *out_, int64_t ldo, const float *lse, int64_t num_edges,
                                int64_t H, int64_t head_dim, float *beta_e, float *ds_e, float *grad_attn, void *ws,
                                size_t ws_bytes, void *stream_, const AttnDrop *drop) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const T *f = reinterpret_cast<const T *>(f_), *g = reinterpret_cast<const T *>(g_),
            *out = reinterpret_cast<const T *>(out_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(num_edges >= 0 && H > 0 && head_dim > 0, PGLB_EINVAL, "%s: bad size", name);
    const int64_t D = H * head_dim;
    const int64_t lph = head_dim / 4;
    PGLB_CHECK_ARG(D <= 128 && head_dim % 4 == 0 && (lph & (lph - 1)) == 0 && (D * B) % 16 == 0, PGLB_EUNSUPPORTED,
                   "%s: needs H*head_dim <= 128 in 16-byte rows and head_dim in {4, 8, 16, 32, 64, 128}", name);
    PGLB_CHECK_ARG(slope >= 0.0f && slope <= 1.0f, PGLB_EUNSUPPORTED, "%s: needs 0 <= negative_slope <= 1", name);
    PGLB_CHECK_ARG(!drop || H % 4 == 0, PGLB_EUNSUPPORTED, "%s: needs H %% 4 == 0", name);
    if (num_edges == 0) {
        if (grad_attn) PGLB_CUDA(cudaMemsetAsync(grad_attn, 0, sizeof(float) * D, stream));
        return PGLB_OK;
    }
    PGLB_CHECK_ARG(rows && cols && f && attn && g && out && lse && beta_e && ds_e, PGLB_EINVAL, "%s: NULL pointer",
                   name);
    auto a16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    PGLB_CHECK_ARG(ldf >= D && ldg >= D && ldo >= D && (ldf * B) % 16 == 0 && (ldg * B) % 16 == 0 &&
                       (ldo * B) % 16 == 0 && a16(f) && a16(g) && a16(out) && a16(attn),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    PGLB_CHECK_ARG(!grad_attn || (ws && ws_bytes >= gatv2_bwd_edge_ws_bytes(num_edges) && a16(ws)), PGLB_EWORKSPACE,
                   "%s: workspace of %zu bytes needed (got %zu)", name, gatv2_bwd_edge_ws_bytes(num_edges), ws_bytes);
    const int grid = grid_of(num_edges, 64);  // a warp per 32 slots, grid-stride
    const AttnDrop dr = drop ? *drop : AttnDrop{};
    float *ga_part = grad_attn ? reinterpret_cast<float *>(ws) : nullptr;
#define PGLB_V2E(L)                                                                                                   \
    do {                                                                                                              \
        if (drop)                                                                                                     \
            gatv2_bwd_edge_kernel<L, T, true><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, attn, slope, g, ldg, \
                                                                        out, ldo, lse, num_edges, (int)H, (int)D,     \
                                                                        beta_e, ds_e, ga_part, dr);                   \
        else                                                                                                          \
            gatv2_bwd_edge_kernel<L, T, false><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, attn, slope, g,     \
                                                                         ldg, out, ldo, lse, num_edges, (int)H,       \
                                                                         (int)D, beta_e, ds_e, ga_part, dr);          \
    } while (0)
    switch ((int)lph) {
        case 1: PGLB_V2E(1); break;
        case 2: PGLB_V2E(2); break;
        case 4: PGLB_V2E(4); break;
        case 8: PGLB_V2E(8); break;
        case 16: PGLB_V2E(16); break;
        default: PGLB_V2E(32); break;
    }
#undef PGLB_V2E
    PGLB_LAUNCH_CHECK("gatv2_bwd_edge_kernel");
    if (grad_attn) {
        gatv2_ga_reduce_kernel<<<(unsigned)D, 256, 0, stream>>>(ga_part, grid, grad_attn);
        PGLB_LAUNCH_CHECK("gatv2_ga_reduce_kernel");
    }
    return PGLB_OK;
}

extern "C" int pglb_gatv2_bwd_edge_ws(int64_t num_edges, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr, PGLB_EINVAL, "pglb_gatv2_bwd_edge_ws: ws_bytes is NULL");
    PGLB_CHECK_ARG(num_edges >= 0, PGLB_EINVAL, "pglb_gatv2_bwd_edge_ws: negative size");
    *ws_bytes = gatv2_bwd_edge_ws_bytes(num_edges);
    return PGLB_OK;
}

extern "C" int pglb_gatv2_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                                       int64_t ldf, const float *attn, float negative_slope, const float *grad_out,
                                       int64_t ldg, const float *out, int64_t ldo, const float *lse, int64_t num_edges,
                                       int64_t H, int64_t head_dim, float *beta_e, float *ds_e, float *grad_attn,
                                       void *ws, size_t ws_bytes, void *stream_) {
    return gatv2_bwd_edge_entry<float>("pglb_gatv2_bwd_edge_f32", rows, cols, eid, f, ldf, attn, negative_slope,
                                       grad_out, ldg, out, ldo, lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn,
                                       ws, ws_bytes, stream_, nullptr);
}

extern "C" int pglb_gatv2_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                       int64_t ldf, const float *attn, float negative_slope, const void *grad_out,
                                       int64_t ldg, const void *out, int64_t ldo, const float *lse, int64_t num_edges,
                                       int64_t H, int64_t head_dim, int dtype, float *beta_e, float *ds_e,
                                       float *grad_attn, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gatv2_bwd_edge_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return gatv2_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, f, ldf, attn, negative_slope, grad_out, ldg,
                                                   out, ldo, lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn, ws,
                                                   ws_bytes, stream_, nullptr);
    return gatv2_bwd_edge_entry<__half>(name, rows, cols, eid, f, ldf, attn, negative_slope, grad_out, ldg, out, ldo,
                                        lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn, ws, ws_bytes, stream_,
                                        nullptr);
}

extern "C" int pglb_gatv2_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                            const float *f, int64_t ldf, const float *attn, float negative_slope,
                                            const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                            const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                            float attn_drop, uint64_t seed, uint64_t offset, float *beta_e,
                                            float *ds_e, float *grad_attn, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gatv2_bwd_edge_drop_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return gatv2_bwd_edge_entry<float>(name, rows, cols, eid, f, ldf, attn, negative_slope, grad_out, ldg, out, ldo,
                                       lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn, ws, ws_bytes, stream_,
                                       &drop);
}

extern "C" int pglb_gatv2_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                            const void *f, int64_t ldf, const float *attn, float negative_slope,
                                            const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                            const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                            int dtype, float attn_drop, uint64_t seed, uint64_t offset, float *beta_e,
                                            float *ds_e, float *grad_attn, void *ws, size_t ws_bytes, void *stream_) {
    const char *name = "pglb_gatv2_bwd_edge_drop_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return gatv2_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, f, ldf, attn, negative_slope, grad_out, ldg,
                                                   out, ldo, lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn, ws,
                                                   ws_bytes, stream_, &drop);
    return gatv2_bwd_edge_entry<__half>(name, rows, cols, eid, f, ldf, attn, negative_slope, grad_out, ldg, out, ldo,
                                        lse, num_edges, H, head_dim, beta_e, ds_e, grad_attn, ws, ws_bytes, stream_,
                                        &drop);
}

// The checks and the launch of the FAConv edge-backward entries (include/pglb.h).  T: element type of f and grad_out,
// rows 16-byte aligned.  drop (nullable): the attention-dropout stream.
template <typename T>
static int fa_bwd_edge_entry(const char *name, const int64_t *rows, const int64_t *cols, const int64_t *eid,
                             const void *f_, int64_t ldf, const float *rec, const void *g_, int64_t ldg,
                             int64_t num_edges, int64_t D, float *beta_e, float *dz_e, void *stream_,
                             const AttnDrop *drop) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const T *f = reinterpret_cast<const T *>(f_), *g = reinterpret_cast<const T *>(g_);
    constexpr int64_t B = sizeof(T);
    PGLB_CHECK_ARG(num_edges >= 0 && D > 0, PGLB_EINVAL, "%s: bad size", name);
    PGLB_CHECK_ARG(D <= 128 && (D * B) % 16 == 0, PGLB_EUNSUPPORTED,
                   "%s: needs D <= 128 in 16-byte rows (D %% 4 == 0 float32, D %% 8 == 0 16-bit)", name);
    if (num_edges == 0) return PGLB_OK;
    PGLB_CHECK_ARG(rows && cols && f && rec && g && beta_e && dz_e, PGLB_EINVAL, "%s: NULL pointer", name);
    auto a16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    PGLB_CHECK_ARG(ldf >= D && ldg >= D && (ldf * B) % 16 == 0 && (ldg * B) % 16 == 0 && a16(f) && a16(g) && a16(rec),
                   PGLB_ESHAPE, "%s: rows must be 16-byte aligned", name);
    const int grid = grid_of(num_edges, 64);  // a warp per 32 slots, grid-stride
    const float4 *rec4 = reinterpret_cast<const float4 *>(rec);
    if (drop)
        fa_bwd_edge_kernel<T, true><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, rec4, g, ldg, num_edges, (int)D,
                                                              beta_e, dz_e, *drop);
    else
        fa_bwd_edge_kernel<T, false><<<grid, 256, 0, stream>>>(rows, cols, eid, f, ldf, rec4, g, ldg, num_edges,
                                                               (int)D, beta_e, dz_e, AttnDrop{});
    PGLB_LAUNCH_CHECK("fa_bwd_edge_kernel");
    return PGLB_OK;
}

extern "C" int pglb_fa_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                                    int64_t ldf, const float *rec, const float *grad_out, int64_t ldg,
                                    int64_t num_edges, int64_t D, float *beta_e, float *dz_e, void *stream_) {
    return fa_bwd_edge_entry<float>("pglb_fa_bwd_edge_f32", rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D,
                                    beta_e, dz_e, stream_, nullptr);
}

extern "C" int pglb_fa_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                    int64_t ldf, const float *rec, const void *grad_out, int64_t ldg,
                                    int64_t num_edges, int64_t D, int dtype, float *beta_e, float *dz_e,
                                    void *stream_) {
    const char *name = "pglb_fa_bwd_edge_x16";
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    if (dtype == PGLB_DTYPE_BF16)
        return fa_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D,
                                                beta_e, dz_e, stream_, nullptr);
    return fa_bwd_edge_entry<__half>(name, rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D, beta_e, dz_e,
                                     stream_, nullptr);
}

extern "C" int pglb_fa_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid,
                                         const float *f, int64_t ldf, const float *rec, const float *grad_out,
                                         int64_t ldg, int64_t num_edges, int64_t D, float attn_drop, uint64_t seed,
                                         uint64_t offset, float *beta_e, float *dz_e, void *stream_) {
    const char *name = "pglb_fa_bwd_edge_drop_f32";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    return fa_bwd_edge_entry<float>(name, rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D, beta_e, dz_e,
                                    stream_, &drop);
}

extern "C" int pglb_fa_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                         int64_t ldf, const float *rec, const void *grad_out, int64_t ldg,
                                         int64_t num_edges, int64_t D, int dtype, float attn_drop, uint64_t seed,
                                         uint64_t offset, float *beta_e, float *dz_e, void *stream_) {
    const char *name = "pglb_fa_bwd_edge_drop_x16";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(dtype == PGLB_DTYPE_BF16 || dtype == PGLB_DTYPE_F16, PGLB_EINVAL, "%s: unknown dtype %d", name,
                   dtype);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    if (dtype == PGLB_DTYPE_BF16)
        return fa_bwd_edge_entry<__nv_bfloat16>(name, rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D,
                                                beta_e, dz_e, stream_, &drop);
    return fa_bwd_edge_entry<__half>(name, rows, cols, eid, f, ldf, rec, grad_out, ldg, num_edges, D, beta_e, dz_e,
                                     stream_, &drop);
}

// The keep words of dst-CSR slots slot0 .. slot0 + n_slots - 1 on the host (include/pglb.h): the same attn_keep_word
// the kernels call, so a test can pin the dropout stream without a GPU.
extern "C" int pglb_attn_dropout_keep_host(uint64_t seed, uint64_t offset, float attn_drop, int64_t slot0,
                                           int64_t n_slots, int64_t H, uint32_t *keep_words) {
    const char *name = "pglb_attn_dropout_keep_host";
    if (const int rc = attn_drop_check(name, attn_drop, offset)) return rc;
    PGLB_CHECK_ARG(slot0 >= 0 && n_slots >= 0, PGLB_EINVAL, "%s: bad slot range", name);
    PGLB_CHECK_ARG(H > 0 && H <= 32 && H % 4 == 0, PGLB_EUNSUPPORTED, "%s: needs H %% 4 == 0 and H <= 32", name);
    if (n_slots == 0) return PGLB_OK;
    PGLB_CHECK_ARG(keep_words != nullptr, PGLB_EINVAL, "%s: NULL pointer", name);
    const AttnDrop drop = attn_drop_of(attn_drop, seed, offset);
    for (int64_t i = 0; i < n_slots; ++i) keep_words[i] = attn_keep_word(drop, (uint64_t)(slot0 + i), (int)H);
    return PGLB_OK;
}

extern "C" int pglb_maxmin_bwd_f32(const int64_t *src_indptr, const int64_t *dst_of_slot,
                                   const float *x, const float *out, const float *grad_out,
                                   float *grad_x, int64_t n_src, int64_t D, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_src >= 0 && D >= 0 && D <= INT32_MAX, PGLB_EINVAL, "pglb_maxmin_bwd_f32: bad size");
    if (n_src == 0 || D == 0) return PGLB_OK;
    PGLB_CHECK_ARG(src_indptr && x && out && grad_out && grad_x, PGLB_EINVAL,
                   "pglb_maxmin_bwd_f32: NULL pointer");
    maxmin_bwd_kernel<<<grid_of(n_src * 32, 64), 256, 0, stream>>>(src_indptr, dst_of_slot, x, out,
                                                                   grad_out, grad_x, n_src, (int)D);
    PGLB_LAUNCH_CHECK("maxmin_bwd_kernel");
    return PGLB_OK;
}
