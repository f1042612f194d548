// spmm_stream.cu -- edge-balanced, shared-memory-staged CSR aggregation for sm_90a.
//
// The wide-row fast path of pglb_spmm_csr_f32 (copy message, 64 < D <= 128, 16-byte aligned
// rows): the kernel the 10M-node / 100M-edge GCN roofline number is measured on.
//
//  * Work unit = a TASK of ~T consecutive CSR slots (not rows): every warp streams about T
//    gathered feature rows whatever the degree distribution, so power-law hubs need no special
//    pass.  A pre-kernel binary-searches the first row of every task and SNAPS the task start
//    past a row of <= T slots that straddles the nominal boundary, so only rows longer than T
//    are ever cut: every row of <= T slots is reduced start to end by one warp, strictly in slot
//    (= ascending edge id) order -- bit-identical to the sequential CPU loop.
//  * Each lane owns a private ring of 32 x 16-byte slots in shared memory.  Gathers are issued
//    with cp.async.cg (LDGSTS, L1-bypassing) LAG groups of 8 rows ahead of the adds, so a warp
//    keeps up to 32 rows (16 KB at D=128) in flight with no registers tied up; 14 warps per
//    SM give ~220 KB of outstanding gathers per SM.  Lane l copies and later reads only its own
//    16 bytes of every row: no cross-lane hand-off, hence no barriers at all.
//  * A row longer than T that is cut by a task boundary leaves per-task partial sums in a side
//    buffer; a fix-up kernel adds them in task order.  Fixed task size => deterministic.
//  * Inner loops are written for instruction count (the first version was issue-bound at ~90
//    warp instructions per edge): 32-bit positions relative to the task start, ring offsets
//    that are compile-time constants, one shuffle + one IMAD.WIDE + one LDGSTS per gathered
//    row, one LDS.128 + 4 FFMA/FADD per consumed row, row pointers prefetched one row ahead.

#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace pglb {

constexpr int RING = 32;  // slots per lane ring == one column batch
constexpr int GRP = 8;    // rows per cp.async commit group
constexpr int LAG = 3;    // groups in flight behind the issue point

struct StreamP {
    const int64_t *indptr;
    const int64_t *cols;  // nullable: identity
    const float *x;  // x / out: float, or the 16-bit element type T of spmm_v5_kernel<T, ...> (ldx / ldo in elements)
    int64_t ldx;
    float *out;
    int64_t ldo;
    int64_t n_rows;
    int64_t E;
    int D;
    int reduce_op;
    const float *scale_src;
    const float *scale_dst;
    const float *scale_slot;  // nullable [E]: scale_src[cols[j]] per slot, streamed by spmm_v5 instead of gathered
    int64_t T;  // nominal slots per task (multiple of 32)
    int64_t ntasks;
    const int64_t *first_row;  // [ntasks]
    const int64_t *start;      // [ntasks + 1] snapped task starts
    float *partial;            // [2*ntasks, dpad]
    int64_t dpad;
    int64_t *tail_row;  // [ntasks]
    const uint32_t *cols32;  // nullable [E]: packed copy of cols, bit 31 = keep-in-L2 hint
    const int64_t *eid;      // nullable: edge id per slot (row of y); identity if NULL
    const float *y;          // nullable: edge operand (send_ue_recv), one scalar per lane per edge
    int64_t ldy;
    int y_bcast;             // PGLB_BCAST_HEAD or PGLB_BCAST_SCALAR
    int head_dim;
    int msg_op;              // PGLB_MSG_MUL or PGLB_MSG_ADD
    const float *attn_dst;   // YM 2 (fused GAT): attn_dst[n_rows, H]; y = attn_src[n_src, H]
    float slope;             // YM 2: LeakyReLU negative slope
    float *partial_ml;       // YM 2: [2*ntasks, 64] running (max, sum) of cut rows, per lane
    int accumulate;          // SUM only: out = (out_prev + sum) * scale_dst
    unsigned *counter;       // task queue head of the persistent kernels, zeroed by task_plan_kernel
    long long *trace;        // debug, nullable: [ntasks, 4] = (start ns, end ns, SM id, warp slot) per task (pglb_debug_task_trace)
    float *lse;              // YM 2, nullable: [n_rows, H] log-sum-exp of every non-empty row's logits (saved for backward)
    int dyn;                 // task order of the queue: 1 ascending, 2 descending
};

__device__ __forceinline__ void cp_async16(unsigned smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16_hint(unsigned smem_dst, const void *gsrc, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;\n" ::"r"(smem_dst),
                 "l"(gsrc), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
__device__ __forceinline__ void cp_async4(unsigned smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ float lds32(unsigned addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];\n" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(unsigned addr, float v) {
    asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}
__device__ __forceinline__ float4 lds128(unsigned addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "r"(addr));
    return v;
}

__device__ __forceinline__ long long global_ns() {
    long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned sm_id() {
    unsigned v;
    asm volatile("mov.u32 %0, %smid;" : "=r"(v));
    return v;
}
// one record per task, written by lane 0 when a debug buffer is armed
__device__ __forceinline__ void trace_task(long long *trace, int64_t task, long long t0) {
    if (trace && (threadIdx.x & 31) == 0) {
        long long *r = trace + task * 4;
        r[0] = t0;
        r[1] = global_ns();
        r[2] = sm_id();
        r[3] = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    }
}

// upper_bound(indptr[0..n_rows], v) - 1 : the non-empty row containing slot v
__device__ __forceinline__ int64_t row_of_slot(const int64_t *__restrict__ indptr, int64_t n_rows,
                                               int64_t v) {
    int64_t lo = 0, hi = n_rows;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg((const long long *)indptr + mid) > v) hi = mid;
        else lo = mid + 1;
    }
    return lo - 1;
}

// out-of-line copy for the (rare) empty-row jump inside the streaming kernels: keeps the binary
// search out of their register allocation and instruction stream
__device__ __noinline__ int64_t row_of_slot_cold(const int64_t *indptr, int64_t n_rows, int64_t v) {
    return row_of_slot(indptr, n_rows, v);
}

// The same answer when the caller knows a row `from` with indptr[from] <= v: gallop (from + 1, + 2, + 4, ...) to a
// row whose start lies beyond v, then bisect the last window.  A run of k empty rows costs ~2 log2(k) loads, the first
// few from the cache line the streaming kernels just read -- instead of the ~log2(n_rows) dependent L2 / DRAM loads
// of the full search.  (RMAT's sparse tail has an empty run after every other one-edge row: at 20 dependent loads
// per jump those tasks ran ~10x longer than the rest and kept a few SMs busy long after the others had finished.)
__device__ __noinline__ int64_t row_of_slot_from(const int64_t *indptr, int64_t n_rows, int64_t from, int64_t v) {
    int64_t lo = from, hi, step = 1;
    for (;;) {
        hi = lo + step;
        if (hi >= n_rows) {
            hi = n_rows;   // indptr[n_rows] = E > v
            break;
        }
        if (__ldg((const long long *)indptr + hi) > v) break;
        lo = hi;
        step <<= 1;
    }
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg((const long long *)indptr + mid) > v) hi = mid;
        else lo = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) task_plan_kernel(const int64_t *__restrict__ indptr,
                                                        int64_t n_rows, int64_t E, int64_t T,
                                                        int64_t snap, int64_t ntasks,
                                                        int64_t *__restrict__ first_row,
                                                        int64_t *__restrict__ start,
                                                        unsigned *__restrict__ counter) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ntasks) return;
    if (t == ntasks) {
        start[t] = E;
        if (counter) *counter = 0u;
        return;
    }
    if (t == 0) {
        first_row[0] = row_of_slot(indptr, n_rows, 0);  // first non-empty row (E > 0)
        start[0] = 0;
        return;
    }
    int64_t a = t * T;
    int64_t r = row_of_slot(indptr, n_rows, a);
    const int64_t s_r = __ldg((const long long *)indptr + r);
    const int64_t e_r = __ldg((const long long *)indptr + r + 1);
    if (s_r < a && e_r - s_r <= snap) {
        // a row of <= snap slots straddles the nominal boundary: the task that holds its first
        // slot finishes it (tasks whose nominal range lies inside such a row become empty)
        a = e_r;
        r = (a < E) ? row_of_slot(indptr, n_rows, a) : n_rows - 1;
    }
    first_row[t] = r;
    start[t] = a;
}

// ---------------------------------------------------------------------------------------------
// D <= 128 (one float4 per lane per row)
// ---------------------------------------------------------------------------------------------
// Ring geometry of the D <= 128 kernel: 16 slots per lane, groups of 4, 14 warps per block (28 per SM).  That is the
// bytes in flight per SM of a 32-slot ring with half the warps, and twice the warps to hide issue and shared-memory
// latency.
template <int YM>
struct Geo {
    static constexpr int kRing = 16;
    static constexpr int kGrp = 4;
    static constexpr int kLag = 3;
    static constexpr int kWarps = YM ? 11 : 14;
    static constexpr int kGpb = 32 / kGrp;       // groups per 32-slot column batch
    static constexpr int kRg = kRing / kGrp;     // groups per turn of the ring
    static constexpr int kSmem = kWarps * kRing * (512 + (YM ? 128 : 0));
};

template <int RK, bool SCALED, int PK, int YM>
__global__ void __launch_bounds__(Geo<YM>::kWarps * 32, 2) spmm_stream128_kernel(const StreamP p) {
    typedef Geo<YM> G_;
    constexpr int RING = G_::kRing, GRP = G_::kGrp, LAG = G_::kLag, GPB = G_::kGpb, RG = G_::kRg;
    // YM 1: message = x[src] (mul|add) y[eid, head(lane)] (send_ue_recv with a per-head or scalar
    // edge operand, the GAT aggregation): the 4-byte operand of every edge rides in a second
    // per-lane ring, fetched with cp.async alongside the feature row.
    constexpr int W = G_::kWarps;
    // PK 0: int64 column ids; 1: pre-packed uint32 ids (half the index bytes); 2: packed ids whose
    // bit 31 carries the source's L2 policy (hub sources that are gathered again and again are
    // kept with evict_last, the long tail streams through with evict_first so it cannot flush
    // them).
    constexpr bool HOT = (PK == 2);
    const uint64_t pol_last = !HOT ? 0 : policy_evict_last();
    const uint64_t pol_first = !HOT ? 0 : policy_evict_first();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const unsigned smem0 = (unsigned)__cvta_generic_to_shared(smem_raw);
    const unsigned ring = smem0 + wib * (RING * 512) + lane * 16;
    const unsigned ring2 = smem0 + W * (RING * 512) + wib * (RING * 128) + lane * 4;
    const float *ylane = nullptr;
    if (YM) ylane = p.y + ((p.y_bcast == PGLB_BCAST_HEAD && lane * 4 < p.D) ? (lane * 4) / p.head_dim : 0);
    // YM 2: the whole GAT aggregation in one pass.  y = attn_src (indexed by the SOURCE id, not
    // the edge id), logit = leaky_relu(attn_src[src,h] + attn_dst[row,h]), and the row is reduced
    // with an online softmax: running max m, running sum l, accumulator rescaled by exp(m - m').
    const int yhead = (lane * 4 < p.D) ? (lane * 4) / p.head_dim : 0;
    float m_run = -INFINITY, l_run = 0.0f, ad = 0.0f;

    const bool is_max = (p.reduce_op == PGLB_REDUCE_MAX);
    const float ident = (RK == 0) ? 0.0f : (is_max ? -INFINITY : INFINITY);
    const bool act = lane * 4 < p.D;
    // inactive lanes (D < 128) alias lane 0's bytes: same sectors, no extra traffic, no predicates
    const char *xlane = reinterpret_cast<const char *>(p.x) + (act ? lane * 16 : 0);
    const unsigned row_bytes = (unsigned)(p.ldx * 4);

    // persistent warps draw task ids from the device-side queue (see spmm_v5_kernel); the per-lane cp.async rings are
    // drained at the end of every task, so a task starts from a clean ring
#pragma unroll 1
    for (;;) {
    unsigned t = 0;
    if (lane == 0) t = atomicAdd(p.counter, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if ((int64_t)t >= p.ntasks) break;
    const int64_t task = p.dyn == 2 ? p.ntasks - 1 - (int64_t)t : (int64_t)t;
    m_run = -INFINITY;
    l_run = 0.0f;
    ad = 0.0f;
    const int64_t a = ld_ro(p.start + task);
    const int64_t b = ld_ro(p.start + task + 1);
    const int cnt = (int)(b - a);
    int64_t row = ld_ro(p.first_row + task);
    int64_t tail = -1;
    if (cnt > 0) {
        auto rel = [&](int64_t v) -> int {
            const int64_t d = v - a;
            return d < -(1 << 30) ? -(1 << 30) : (d > (1 << 30) ? (1 << 30) : (int)d);
        };
        int beg_rel = rel(ld_ro(p.indptr + row));
        int end_rel = rel(ld_ro(p.indptr + row + 1));
        int nxt_rel = (row + 2 <= p.n_rows) ? rel(ld_ro(p.indptr + row + 2)) : (1 << 30);
        bool head = beg_rel < 0;  // first row started in an earlier task (only rows longer than T)
        float4 acc = make_float4(ident, ident, ident, ident);

        auto finish_row = [&]() {
            // row `row` is complete: slots [beg_rel, end_rel) relative to a
            if (head) {
                if (act) *reinterpret_cast<float4 *>(p.partial + (2 * task) * p.dpad + lane * 4) = acc;
                if (YM == 2) {
                    p.partial_ml[(2 * task) * 64 + lane * 2] = m_run;
                    p.partial_ml[(2 * task) * 64 + lane * 2 + 1] = l_run;
                }
                head = false;  // the owner task's fix-up finishes this row
            } else if (act) {
                float4 v = acc;
                const int deg = end_rel - beg_rel;
                if (deg == 0) v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (YM == 2 && deg != 0) {
                    v.x = __fdiv_rn(v.x, l_run); v.y = __fdiv_rn(v.y, l_run);
                    v.z = __fdiv_rn(v.z, l_run); v.w = __fdiv_rn(v.w, l_run);
                }
                if (p.accumulate) {
                    const float4 o = *reinterpret_cast<const float4 *>(p.out + row * p.ldo + lane * 4);
                    v.x = __fadd_rn(o.x, v.x); v.y = __fadd_rn(o.y, v.y);
                    v.z = __fadd_rn(o.z, v.z); v.w = __fadd_rn(o.w, v.w);
                }
                if (p.reduce_op == PGLB_REDUCE_MEAN && deg != 0) {
                    const float c = (float)deg;
                    v.x = __fdiv_rn(v.x, c); v.y = __fdiv_rn(v.y, c);
                    v.z = __fdiv_rn(v.z, c); v.w = __fdiv_rn(v.w, c);
                }
                if (p.scale_dst) {
                    const float sd = __ldg(p.scale_dst + row);
                    v.x = __fmul_rn(v.x, sd); v.y = __fmul_rn(v.y, sd);
                    v.z = __fmul_rn(v.z, sd); v.w = __fmul_rn(v.w, sd);
                }
                __stcs(reinterpret_cast<float4 *>(p.out + row * p.ldo + lane * 4), v);
            }
            ++row;
            beg_rel = end_rel;
            end_rel = nxt_rel;
            nxt_rel = (row + 2 <= p.n_rows) ? rel(ld_ro(p.indptr + row + 2)) : (1 << 30);
            if (end_rel == beg_rel && row < p.n_rows) {
                // the next row is empty: jump over the whole run of empty rows (they are zero-filled
                // by empty_rows_kernel) to the row that owns the next slot -- a single warp must not
                // walk 10^5 empty rows one by one (RMAT graphs have such runs)
                const int64_t pos_abs = a + beg_rel;
                if (pos_abs >= p.E) {
                    row = p.n_rows;
                    end_rel = 1 << 30;
                } else {
                    row = row_of_slot_from(p.indptr, p.n_rows, row, pos_abs);
                    end_rel = rel(ld_ro(p.indptr + row + 1));
                    nxt_rel = (row + 2 <= p.n_rows) ? rel(ld_ro(p.indptr + row + 2)) : (1 << 30);
                }
            }
            acc = make_float4(ident, ident, ident, ident);
            if (YM == 2) {
                m_run = -INFINITY;
                l_run = 0.0f;
                ad = (act && row < p.n_rows) ? __ldg(p.attn_dst + row * p.ldy + yhead) : 0.0f;
            }
        };
        if (YM == 2) ad = act ? __ldg(p.attn_dst + row * p.ldy + yhead) : 0.0f;

        auto load_col = [&](int batch) -> unsigned {
            const int j = batch * 32 + lane;
            if (j >= cnt) return 0u;
            if (PK != 0) return __ldcs(p.cols32 + a + j);
            return (unsigned)(p.cols ? ld_stream(p.cols + a + j) : (a + j));
        };
        auto load_eid = [&](int batch) -> unsigned {
            const int j = batch * 32 + lane;
            if (YM != 1 || j >= cnt) return 0u;
            return (unsigned)(p.eid ? ld_stream(p.eid + a + j) : (a + j));
        };
        // 32-bit column ids: the dispatcher routes n_src >= 2^32 to the generic kernel
        unsigned col_cur = load_col(0);
        unsigned col_nxt = load_col(1);
        unsigned eid_cur = load_eid(0);
        unsigned eid_nxt = load_eid(1);
        float sc_cur = 1.0f, sc_prev = 1.0f;
        if (SCALED) sc_cur = (lane < cnt) ? __ldg(p.scale_src + (col_cur & 0x7fffffffu)) : 1.0f;

        // One rolled loop over groups of 8 slots: issue group g, then consume group g - LAG.
        // Deliberately NOT unrolled over the ring: the unrolled form inlined the row epilogue
        // dozens of times (4096 SASS instructions, beyond the instruction cache); per-warp
        // latency is hidden by the 14 resident warps instead.
        const int ngroups = (cnt + GRP - 1) / GRP;
#pragma unroll 1
        for (int g = 0; g < ngroups + LAG; ++g) {
            const int sub = g % GPB;  // position of the group inside its 32-slot column batch
            if (g < ngroups) {
                if (sub == 0 && g > 0) {
                    const int base = g * GRP;
                    sc_prev = sc_cur;
                    col_cur = col_nxt;
                    col_nxt = load_col(g / GPB + 1);
                    if (YM == 1) {
                        eid_cur = eid_nxt;
                        eid_nxt = load_eid(g / GPB + 1);
                    }
                    if (SCALED)
                        sc_cur = (base + lane < cnt) ? __ldg(p.scale_src + (col_cur & 0x7fffffffu)) : 1.0f;
                }
                const int valid = cnt - g * GRP;
                const int rs = g % RG;  // ring group slot
                const unsigned gaddr = ring + rs * (GRP * 512);
#pragma unroll
                for (int k = 0; k < GRP; ++k) {
                    const unsigned c = __shfl_sync(0xffffffffu, col_cur, sub * GRP + k);
                    if (YM == 1) {
                        const unsigned eidk = __shfl_sync(0xffffffffu, eid_cur, sub * GRP + k);
                        if (k < valid)
                            cp_async4(ring2 + (rs * GRP + k) * 128, ylane + (size_t)eidk * p.ldy);
                    }
                    if (YM == 2 && k < valid)  // attn_src of the SOURCE node
                        cp_async4(ring2 + (rs * GRP + k) * 128, ylane + (size_t)c * p.ldy);
                    if (k < valid) {
                        if (HOT) {
                            const uint64_t pol = (c >> 31) ? pol_last : pol_first;
                            cp_async16_hint(gaddr + k * 512, xlane + (size_t)(c & 0x7fffffffu) * row_bytes, pol);
                        } else {
                            cp_async16(gaddr + k * 512, xlane + (size_t)c * row_bytes);
                        }
                    }
                }
            }
            cp_async_commit();
            if (g >= LAG) {
                cp_async_wait<LAG>();
                const int gc = g - LAG;
                const int csub = gc % GPB;
                const int crs = gc % RG;
                const int base = gc * GRP;
                // which register holds the scales of the consumed group's batch
                const int bcur = (g < ngroups ? g : ngroups - 1) / GPB;
                const float sc_reg = ((gc / GPB) == bcur) ? sc_cur : sc_prev;
                int k_end = end_rel - base;  // where the current row ends inside this group
                int valid = cnt - base;
                valid = valid > GRP ? GRP : valid;
                const unsigned gaddr = ring + crs * (GRP * 512);
#pragma unroll 1
                for (int k = 0; k < valid; ++k) {
                    while (k == k_end) {
                        finish_row();
                        k_end = end_rel - base;
                    }
                    float4 v = lds128(gaddr + k * 512);
                    if (YM == 2) {
                        float lg = lds32(ring2 + (crs * GRP + k) * 128) + ad;
                        lg = lg >= 0.0f ? lg : lg * p.slope;
                        if (lg <= m_run) {  // common case: the running max stands, one exp
                            const float pe = expf(lg - m_run);
                            l_run += pe;
                            acc.x = fmaf(pe, v.x, acc.x); acc.y = fmaf(pe, v.y, acc.y);
                            acc.z = fmaf(pe, v.z, acc.z); acc.w = fmaf(pe, v.w, acc.w);
                        } else {  // new max: rescale what has been accumulated (exp(-inf) = 0 at a row start)
                            const float sc = expf(m_run - lg);
                            l_run = fmaf(l_run, sc, 1.0f);
                            acc.x = fmaf(acc.x, sc, v.x); acc.y = fmaf(acc.y, sc, v.y);
                            acc.z = fmaf(acc.z, sc, v.z); acc.w = fmaf(acc.w, sc, v.w);
                            m_run = lg;
                        }
                        continue;
                    }
                    if (YM == 1) {
                        const float yv = lds32(ring2 + (crs * GRP + k) * 128);
                        if (p.msg_op == PGLB_MSG_MUL) {
                            v.x = __fmul_rn(v.x, yv); v.y = __fmul_rn(v.y, yv);
                            v.z = __fmul_rn(v.z, yv); v.w = __fmul_rn(v.w, yv);
                        } else {
                            v.x = __fadd_rn(v.x, yv); v.y = __fadd_rn(v.y, yv);
                            v.z = __fadd_rn(v.z, yv); v.w = __fadd_rn(v.w, yv);
                        }
                    }
                    float s = 1.0f;
                    if (SCALED) s = __shfl_sync(0xffffffffu, sc_reg, csub * GRP + k);
                    if (RK == 0) {
                        if (SCALED) {
                            // x * norm[src] added in one FMA (more accurate than the reference's
                            // separate multiply; within the 1e-4 bar)
                            acc.x = fmaf(v.x, s, acc.x); acc.y = fmaf(v.y, s, acc.y);
                            acc.z = fmaf(v.z, s, acc.z); acc.w = fmaf(v.w, s, acc.w);
                        } else {
                            acc.x = __fadd_rn(acc.x, v.x); acc.y = __fadd_rn(acc.y, v.y);
                            acc.z = __fadd_rn(acc.z, v.z); acc.w = __fadd_rn(acc.w, v.w);
                        }
                    } else if (is_max) {
                        acc.x = fmaxf(acc.x, v.x * s); acc.y = fmaxf(acc.y, v.y * s);
                        acc.z = fmaxf(acc.z, v.z * s); acc.w = fmaxf(acc.w, v.w * s);
                    } else {
                        acc.x = fminf(acc.x, v.x * s); acc.y = fminf(acc.y, v.y * s);
                        acc.z = fminf(acc.z, v.z * s); acc.w = fminf(acc.w, v.w * s);
                    }
                }
            }
        }
        // rows that end exactly at b (and, for the last non-empty task, every trailing empty row)
        while (row < p.n_rows && end_rel == cnt) finish_row();
        if (row < p.n_rows && beg_rel < cnt) {
            // the open row (longer than T) continues in the next task(s)
            if (act)
                *reinterpret_cast<float4 *>(p.partial + (head ? (2 * task) : (2 * task + 1)) * p.dpad +
                                            lane * 4) = acc;
            if (YM == 2) {
                const int64_t sl = head ? (2 * task) : (2 * task + 1);
                p.partial_ml[sl * 64 + lane * 2] = m_run;
                p.partial_ml[sl * 64 + lane * 2 + 1] = l_run;
            }
            if (!head) tail = row;
        }
    }
    if (lane == 0) p.tail_row[task] = tail;
    cp_async_wait<0>();   // nothing real is pending; keeps the group count of the next task's pipeline exact
    }
}

// ---------------------------------------------------------------------------------------------
// generic ITERS (128 < D <= 512 per column tile): same scheme, straightforward code
// ---------------------------------------------------------------------------------------------
template <int ITERS>
struct StreamCfg {
    static constexpr int kWarps = (ITERS == 2) ? 2 : 1;
    static constexpr int kThreads = kWarps * 32;
    static constexpr int kSmem = kWarps * RING * 32 * ITERS * 16;
};

template <int ITERS, int RK>
__global__ void __launch_bounds__(StreamCfg<ITERS>::kThreads) spmm_stream_kernel(const StreamP p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int64_t task = (int64_t)blockIdx.x * StreamCfg<ITERS>::kWarps + wib;
    if (task >= p.ntasks) return;
    float4 *ring = reinterpret_cast<float4 *>(smem_raw) + (size_t)wib * RING * ITERS * 32 + lane;

    const bool is_max = (p.reduce_op == PGLB_REDUCE_MAX);
    const float ident = (RK == 0) ? 0.0f : (is_max ? -INFINITY : INFINITY);
    const int col_tile = blockIdx.y * (32 * 4 * ITERS);
    int col[ITERS];
    bool act[ITERS];
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        col[it] = col_tile + (it * 32 + lane) * 4;
        act[it] = col[it] < p.D;
    }

    const int64_t a = ld_ro(p.start + task);
    const int64_t b = ld_ro(p.start + task + 1);
    const int cnt = (int)(b - a);
    const int ngroups = (cnt + GRP - 1) / GRP;
    int64_t tail = -1;
    if (cnt > 0) {
        int64_t row = ld_ro(p.first_row + task);
        int64_t cur_beg = ld_ro(p.indptr + row);
        int64_t cur_end = ld_ro(p.indptr + row + 1);
        bool head = cur_beg < a;
        int64_t pos = a;

        float4 acc[ITERS];
#pragma unroll
        for (int it = 0; it < ITERS; ++it) acc[it] = make_float4(ident, ident, ident, ident);

        auto finish_row = [&]() {
            const int64_t deg = cur_end - cur_beg;
            if (head) {
                float *dst = p.partial + (2 * task) * p.dpad;
#pragma unroll
                for (int it = 0; it < ITERS; ++it)
                    if (act[it]) *reinterpret_cast<float4 *>(dst + col[it]) = acc[it];
                head = false;
            } else {
                const float sd = p.scale_dst ? __ldg(p.scale_dst + row) : 1.0f;
                const float cntf = (float)deg;
#pragma unroll
                for (int it = 0; it < ITERS; ++it) {
                    if (!act[it]) continue;
                    float4 v = acc[it];
                    if (deg == 0) v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (p.accumulate) {
                        const float4 o = *reinterpret_cast<const float4 *>(p.out + row * p.ldo + col[it]);
                        v.x = __fadd_rn(o.x, v.x); v.y = __fadd_rn(o.y, v.y);
                        v.z = __fadd_rn(o.z, v.z); v.w = __fadd_rn(o.w, v.w);
                    }
                    if (p.reduce_op == PGLB_REDUCE_MEAN && deg != 0) {
                        v.x = __fdiv_rn(v.x, cntf); v.y = __fdiv_rn(v.y, cntf);
                        v.z = __fdiv_rn(v.z, cntf); v.w = __fdiv_rn(v.w, cntf);
                    }
                    if (p.scale_dst) {
                        v.x = __fmul_rn(v.x, sd); v.y = __fmul_rn(v.y, sd);
                        v.z = __fmul_rn(v.z, sd); v.w = __fmul_rn(v.w, sd);
                    }
                    __stcs(reinterpret_cast<float4 *>(p.out + row * p.ldo + col[it]), v);
                }
            }
            ++row;
            cur_beg = cur_end;
            if (row < p.n_rows) cur_end = ld_ro(p.indptr + row + 1);
            if (row < p.n_rows && cur_end == cur_beg) {  // jump over a run of empty rows
                if (cur_beg >= p.E) {
                    row = p.n_rows;
                } else {
                    row = row_of_slot_from(p.indptr, p.n_rows, row, cur_beg);
                    cur_end = ld_ro(p.indptr + row + 1);
                }
            }
#pragma unroll
            for (int it = 0; it < ITERS; ++it) acc[it] = make_float4(ident, ident, ident, ident);
        };

        auto load_col = [&](int batch) -> int64_t {
            const int j = batch * 32 + lane;
            if (j >= cnt) return 0;
            return p.cols ? ld_stream(p.cols + a + j) : (a + j);
        };
        int64_t col_cur = load_col(0);
        int64_t col_nxt = load_col(1);
        float sc_cur = (p.scale_src && lane < cnt) ? __ldg(p.scale_src + col_cur) : 1.0f;
        float sc_prev = 1.0f;

        for (int g = 0; g < ngroups + LAG; ++g) {
            if (g < ngroups) {
                const int sub = g & 3;
                if (sub == 0 && g > 0) {
                    const int batch = g >> 2;
                    sc_prev = sc_cur;
                    col_cur = col_nxt;
                    col_nxt = load_col(batch + 1);
                    if (p.scale_src)
                        sc_cur = (batch * 32 + lane < cnt) ? __ldg(p.scale_src + col_cur) : 1.0f;
                }
#pragma unroll
                for (int k = 0; k < GRP; ++k) {
                    const int64_t c = __shfl_sync(0xffffffffu, col_cur, sub * GRP + k);
                    const int j = g * GRP + k;
                    if (j < cnt) {
                        const float *xr = p.x + c * p.ldx;
                        float4 *slot = ring + (size_t)((j & (RING - 1)) * ITERS) * 32;
#pragma unroll
                        for (int it = 0; it < ITERS; ++it)
                            if (act[it])
                                cp_async16((unsigned)__cvta_generic_to_shared(slot + it * 32), xr + col[it]);
                    }
                }
            }
            cp_async_commit();
            if (g >= LAG) {
                cp_async_wait<LAG>();
                const int gc = g - LAG;
                const int bcur = (g < ngroups ? g : ngroups - 1) >> 2;
                const bool in_cur = (gc >> 2) == bcur;
#pragma unroll
                for (int k = 0; k < GRP; ++k) {
                    const int j = gc * GRP + k;
                    const float s_c = __shfl_sync(0xffffffffu, sc_cur, (gc & 3) * GRP + k);
                    const float s_p = __shfl_sync(0xffffffffu, sc_prev, (gc & 3) * GRP + k);
                    if (j < cnt) {
                        while (pos == cur_end) finish_row();
                        const float s = in_cur ? s_c : s_p;
                        const float4 *slot = ring + (size_t)((j & (RING - 1)) * ITERS) * 32;
#pragma unroll
                        for (int it = 0; it < ITERS; ++it) {
                            if (!act[it]) continue;
                            float4 v = slot[it * 32];
                            if (p.scale_src) {
                                v.x = __fmul_rn(v.x, s); v.y = __fmul_rn(v.y, s);
                                v.z = __fmul_rn(v.z, s); v.w = __fmul_rn(v.w, s);
                            }
                            if (RK == 0) {
                                acc[it].x = __fadd_rn(acc[it].x, v.x); acc[it].y = __fadd_rn(acc[it].y, v.y);
                                acc[it].z = __fadd_rn(acc[it].z, v.z); acc[it].w = __fadd_rn(acc[it].w, v.w);
                            } else if (is_max) {
                                acc[it].x = fmaxf(acc[it].x, v.x); acc[it].y = fmaxf(acc[it].y, v.y);
                                acc[it].z = fmaxf(acc[it].z, v.z); acc[it].w = fmaxf(acc[it].w, v.w);
                            } else {
                                acc[it].x = fminf(acc[it].x, v.x); acc[it].y = fminf(acc[it].y, v.y);
                                acc[it].z = fminf(acc[it].z, v.z); acc[it].w = fminf(acc[it].w, v.w);
                            }
                        }
                        ++pos;
                    }
                }
            }
        }
        while (row < p.n_rows && cur_end == pos) finish_row();
        if (row < p.n_rows && cur_beg < pos) {
            float *dst = p.partial + (head ? (2 * task) : (2 * task + 1)) * p.dpad;
#pragma unroll
            for (int it = 0; it < ITERS; ++it)
                if (act[it]) *reinterpret_cast<float4 *>(dst + col[it]) = acc[it];
            if (!head) tail = row;
        }
    }
    if (lane == 0 && blockIdx.y == 0) p.tail_row[task] = tail;
}

// One warp per task that owns a cut row: out[r] = epilogue(tail(t) (+) head(t+1) (+) ...).  The partials are fp32;
// TO is the element type of out (a 16-bit out is rounded once, on the store).  PROP (float, copy sum): the row closes
// with epi's epilogue.
template <typename TO, int ITERS, int RK, bool PROP>
__device__ __forceinline__ void spmm_stream_fixup_body(const StreamP &p, const PropEpi &epi) {
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= p.ntasks) return;
    const int64_t r = p.tail_row[t];
    if (r < 0) return;
    const bool is_max = (p.reduce_op == PGLB_REDUCE_MAX);
    const int col_tile = blockIdx.y * (32 * 4 * ITERS);
    const int64_t s_r = ld_ro(p.indptr + r), e_r = ld_ro(p.indptr + r + 1);
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int c = col_tile + (it * 32 + lane) * 4;
        if (c >= p.D) continue;
        float4 acc = *reinterpret_cast<const float4 *>(p.partial + (2 * t + 1) * p.dpad + c);
        // tasks inside a row longer than T are never snapped: task u starts at u*T.  Loads are
        // issued 8 at a time (independent), the adds stay in task order.
        auto comb = [&](const float4 v) {
            if (RK == 0) {
                acc.x = __fadd_rn(acc.x, v.x); acc.y = __fadd_rn(acc.y, v.y);
                acc.z = __fadd_rn(acc.z, v.z); acc.w = __fadd_rn(acc.w, v.w);
            } else if (is_max) {
                acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y);
                acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w);
            } else {
                acc.x = fminf(acc.x, v.x); acc.y = fminf(acc.y, v.y);
                acc.z = fminf(acc.z, v.z); acc.w = fminf(acc.w, v.w);
            }
        };
        const int64_t u_end = (e_r + p.T - 1) / p.T;  // first task that starts at or after e_r
        int64_t u = t + 1;
        for (; u + 8 <= u_end; u += 8) {
            float4 v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q)
                v[q] = *reinterpret_cast<const float4 *>(p.partial + (2 * (u + q)) * p.dpad + c);
#pragma unroll
            for (int q = 0; q < 8; ++q) comb(v[q]);
        }
        for (; u < u_end; ++u)
            comb(*reinterpret_cast<const float4 *>(p.partial + (2 * u) * p.dpad + c));
        if (sizeof(TO) == 4 && p.accumulate) {
            const float4 o = *reinterpret_cast<const float4 *>(p.out + r * p.ldo + c);
            acc.x = __fadd_rn(o.x, acc.x); acc.y = __fadd_rn(o.y, acc.y);
            acc.z = __fadd_rn(o.z, acc.z); acc.w = __fadd_rn(o.w, acc.w);
        }
        if (p.reduce_op == PGLB_REDUCE_MEAN) {
            const float cntf = (float)(e_r - s_r);
            acc.x = __fdiv_rn(acc.x, cntf); acc.y = __fdiv_rn(acc.y, cntf);
            acc.z = __fdiv_rn(acc.z, cntf); acc.w = __fdiv_rn(acc.w, cntf);
        }
        if (p.scale_dst) {
            const float sd = __ldg(p.scale_dst + r);
            acc.x = __fmul_rn(acc.x, sd); acc.y = __fmul_rn(acc.y, sd);
            acc.z = __fmul_rn(acc.z, sd); acc.w = __fmul_rn(acc.w, sd);
        }
        if constexpr (PROP)
            prop_store4(epi, prop_c(epi), p.out, p.ldo, r, c, acc);
        else if constexpr (sizeof(TO) == 4)
            *reinterpret_cast<float4 *>(p.out + r * p.ldo + c) = acc;
        else
            *reinterpret_cast<uint2 *>(reinterpret_cast<TO *>(p.out) + r * p.ldo + c) = round4<TO>(acc);
    }
}
template <typename TO, int ITERS, int RK>
__global__ void __launch_bounds__(256) spmm_stream_fixup_kernel(const StreamP p) {
    spmm_stream_fixup_body<TO, ITERS, RK, false>(p, PropEpi{});
}
// the fix-up of pglb_propagate_*'s cut rows (float32, one float4 per lane)
__global__ void __launch_bounds__(256) spmm_stream_fixup_prop_kernel(const StreamP p, const PropEpi epi) {
    spmm_stream_fixup_body<float, 1, 0, true>(p, epi);
}

// Fused-GAT fix-up: merge the (acc, m, l) partials of a cut row: M = max m_i,
// out = sum_i acc_i e^{m_i - M} / sum_i l_i e^{m_i - M}.  The partials are fp32; TO is the element type of out (a
// 16-bit out is rounded once, on the store).  DROP (attention dropout): the acc partials hold only the kept slots and
// the quotient is multiplied by drop_scale = 1 / (1 - p).
template <typename TO, bool DROP>
__global__ void __launch_bounds__(256) spmm_stream_fixup_gat_kernel(const StreamP p, float drop_scale) {
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= p.ntasks) return;
    const int64_t r = p.tail_row[t];
    if (r < 0) return;
    const int c = lane * 4;
    if (c >= p.D) return;
    const int64_t e_r = ld_ro(p.indptr + r + 1);
    const int64_t u_end = (e_r + p.T - 1) / p.T;
    float M = p.partial_ml[(2 * t + 1) * 64 + lane * 2];
    for (int64_t u = t + 1; u < u_end; ++u) M = fmaxf(M, p.partial_ml[(2 * u) * 64 + lane * 2]);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float L = 0.0f;
    auto add = [&](int64_t slot) {
        const float w = expf(p.partial_ml[slot * 64 + lane * 2] - M);
        const float4 v = *reinterpret_cast<const float4 *>(p.partial + slot * p.dpad + c);
        L = fmaf(p.partial_ml[slot * 64 + lane * 2 + 1], w, L);
        acc.x = fmaf(v.x, w, acc.x); acc.y = fmaf(v.y, w, acc.y);
        acc.z = fmaf(v.z, w, acc.z); acc.w = fmaf(v.w, w, acc.w);
    };
    add(2 * t + 1);
    for (int64_t u = t + 1; u < u_end; ++u) add(2 * u);
    acc.x = __fdiv_rn(acc.x, L); acc.y = __fdiv_rn(acc.y, L);
    acc.z = __fdiv_rn(acc.z, L); acc.w = __fdiv_rn(acc.w, L);
    if constexpr (DROP) {
        acc.x *= drop_scale; acc.y *= drop_scale; acc.z *= drop_scale; acc.w *= drop_scale;
    }
    if constexpr (sizeof(TO) == 4)
        *reinterpret_cast<float4 *>(p.out + r * p.ldo + c) = acc;
    else
        *reinterpret_cast<uint2 *>(reinterpret_cast<TO *>(p.out) + r * p.ldo + c) = round4<TO>(acc);
    if (p.lse && c % p.head_dim == 0) p.lse[r * p.ldy + c / p.head_dim] = M + logf(L);
}

// Rows without a slot: zero (or, when accumulating, out_prev * scale_dst).  One warp looks at 32
// rows at a time; the streaming tasks above never touch empty rows.  TO: element type of out (16-bit: D % 4 == 0,
// rows 8-byte aligned, never accumulating).
template <typename TO>
__global__ void __launch_bounds__(256) empty_rows_kernel(const int64_t *__restrict__ indptr, int64_t n_rows, int D,
                                                         float *__restrict__ out, int64_t ldo,
                                                         const float *__restrict__ scale_dst, int accumulate) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r0 = warp * 32; r0 < n_rows; r0 += nwarps * 32) {
        const int64_t r = r0 + lane;
        bool empty = false;
        if (r < n_rows) empty = ld_ro(indptr + r + 1) == ld_ro(indptr + r);
        unsigned mask = __ballot_sync(0xffffffffu, empty);
        while (mask) {
            const int i = __ffs(mask) - 1;
            mask &= mask - 1;
            float *row = out + (r0 + i) * ldo;
            for (int c = lane * 4; c < D; c += 128) {
                if constexpr (sizeof(TO) == 2) {
                    *reinterpret_cast<uint2 *>(reinterpret_cast<TO *>(out) + (r0 + i) * ldo + c) = make_uint2(0u, 0u);
                    continue;
                }
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (accumulate) {
                    v = *reinterpret_cast<const float4 *>(row + c);
                    if (scale_dst) {
                        const float sd = __ldg(scale_dst + r0 + i);
                        v.x *= sd; v.y *= sd; v.z *= sd; v.w *= sd;
                    }
                }
                *reinterpret_cast<float4 *>(row + c) = v;
            }
        }
    }
}

// Rows without a slot under pglb_propagate_*'s epilogue: t = 0, the value empty_rows_kernel writes (float32 rows,
// D % 4 == 0, 16-byte aligned)
__global__ void __launch_bounds__(256) empty_rows_prop_kernel(const int64_t *__restrict__ indptr, int64_t n_rows, int D,
                                                              float *__restrict__ out, int64_t ldo, const PropEpi epi) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float cc = prop_c(epi);
    for (int64_t r0 = warp * 32; r0 < n_rows; r0 += nwarps * 32) {
        const int64_t r = r0 + lane;
        bool empty = false;
        if (r < n_rows) empty = ld_ro(indptr + r + 1) == ld_ro(indptr + r);
        unsigned mask = __ballot_sync(0xffffffffu, empty);
        while (mask) {
            const int i = __ffs(mask) - 1;
            mask &= mask - 1;
            for (int c = lane * 4; c < D; c += 128) prop_store4(epi, cc, out, ldo, r0 + i, c, make_float4(0.f, 0.f, 0.f, 0.f));
        }
    }
}

template <typename TO>
static int launch_empty_rows(const StreamP &p, cudaStream_t stream) {
    if (p.accumulate && !p.scale_dst) return PGLB_OK;  // out_prev + 0 unchanged
    int64_t blocks = (p.n_rows + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    empty_rows_kernel<TO><<<(unsigned)blocks, 256, 0, stream>>>(p.indptr, p.n_rows, p.D, p.out, p.ldo,
                                                               p.scale_dst, p.accumulate);
    PGLB_LAUNCH_CHECK("empty_rows_kernel");
    return PGLB_OK;
}

static int launch_empty_rows_prop(const StreamP &p, const PropEpi &epi, cudaStream_t stream) {
    int64_t blocks = (p.n_rows + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    empty_rows_prop_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p.indptr, p.n_rows, p.D, p.out, p.ldo, epi);
    PGLB_LAUNCH_CHECK("empty_rows_prop_kernel");
    return PGLB_OK;
}

#include "spmm_v5.inl"
#include "spmm_gat5.inl"
#include "spmm_narrow2.inl"

struct StreamWs {
    int64_t *first_row;
    int64_t *start;
    int64_t *tail_row;
    float *partial;
    float *partial_ml;
    unsigned *counter;
    int64_t ntasks, dpad;
    size_t bytes;
};

static StreamWs stream_layout(void *ws, int64_t E, int64_t D, int64_t T) {
    StreamWs w;
    w.ntasks = (E + T - 1) / T;
    w.dpad = (D + 3) / 4 * 4;
    char *base = reinterpret_cast<char *>(ws);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char *r = base ? base + off : nullptr;
        off += align_up(bytes ? bytes : 1, 256);
        return r;
    };
    w.first_row = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * w.ntasks));
    w.start = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * (w.ntasks + 1)));
    w.tail_row = reinterpret_cast<int64_t *>(take(sizeof(int64_t) * w.ntasks));
    w.partial = reinterpret_cast<float *>(take(sizeof(float) * 2 * w.ntasks * w.dpad));
    w.partial_ml = reinterpret_cast<float *>(take(sizeof(float) * 2 * w.ntasks * 64));
    w.counter = reinterpret_cast<unsigned *>(take(sizeof(unsigned)));
    w.bytes = off;
    return w;
}

static int64_t env_task_size() {
    static int64_t t = -1;
    if (t < 0) {
        t = 0;
        const char *e = getenv("PGLB_STREAM_TASK");
        if (e) {
            long v = atol(e);
            if (v >= 32 && v % 32 == 0) t = v;
        }
    }
    return t;
}

// Slots per task: 2048 for big graphs, smaller when that would leave fewer than ~4 tasks per
// resident warp (a 10M-edge graph gets T = 608, a Cora-sized one T = 32).  PGLB_STREAM_TASK pins it
// (stress tests).
int64_t stream_task_size(int64_t E) {
    const int64_t fixed = env_task_size();
    if (fixed) return fixed;
    const int64_t target = (int64_t)sm_count() * 28 * 4;
    int64_t t = (E / target + 31) / 32 * 32;
    if (t < 32) t = 32;
    if (t > 2048) t = 2048;
    return t;
}

// Rows of up to this many slots are never cut by a task boundary (=> reduced by one warp in slot
// order, bit-identical to the sequential loop).
static int64_t stream_snap(int64_t T) { return env_task_size() ? T : (T > 1024 ? T : 1024); }

// The fused GAT kernel runs on the device-side queue in descending task order and likes tasks half as long: a GAT
// slot costs more than a copy-sum slot, and shorter tasks balance the tail of the launch.
static int64_t gat_task_size(int64_t E) {
    const int64_t fixed = env_task_size();
    if (fixed) return fixed;
    int64_t t = (stream_task_size(E) / 2 + 31) / 32 * 32;
    return t < 32 ? 32 : t;
}

// one workspace size for every kernel of the family: the layout of the smallest task size any of them uses
size_t stream_ws_bytes(int64_t E, int64_t D) { return stream_layout(nullptr, E, D, gat_task_size(E)).bytes; }

// Task order of the persistent kernels' device-side queue (StreamP::dyn): 1 = ascending, 2 = descending.  slot 0: the
// copy-sum kernel (spmm_v5), which takes ascending order when there are many tasks per resident warp and descending
// order when there are few.  Every other kernel (slot >= 1) takes descending order: RMAT puts the expensive tasks
// (one-edge rows) last, the descending queue starts them first and every warp stays busy to the end of the launch.
static int dyn_mode(int slot, int64_t ntasks) {
    if (slot >= 1) return 2;
    const int64_t resident_warps = (int64_t)sm_count() * 2 * 13;
    return ntasks >= 8 * resident_warps ? 1 : 2;
}

// debug: per-task timeline of the next launches of spmm_v5_kernel / spmm_gat5_kernel (scripts/task_trace.py)
static std::atomic<long long *> g_trace{nullptr};
static std::atomic<int64_t> g_trace_cap{0};
static long long *trace_for(int64_t ntasks) {
    long long *t = g_trace.load(std::memory_order_acquire);
    return (t && ntasks <= g_trace_cap.load(std::memory_order_acquire)) ? t : nullptr;
}

template <int RK, bool SCALED, int PK, int YM>
static int launch_stream128(const StreamP &p, cudaStream_t stream) {
    typedef Geo<YM> G_;
    constexpr int W = G_::kWarps;
    const int smem = G_::kSmem;
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(spmm_stream128_kernel<RK, SCALED, PK, YM>, smem, attr_done));
    int64_t blocks = (p.ntasks + W - 1) / W;
    PGLB_CHECK_ARG(blocks <= 0x7fffffffLL, PGLB_ESHAPE, "spmm_stream: grid too large");
    if (blocks > (int64_t)sm_count() * 2) blocks = (int64_t)sm_count() * 2;   // persistent: 2 CTAs per SM
    spmm_stream128_kernel<RK, SCALED, PK, YM><<<(unsigned)blocks, W * 32, smem, stream>>>(p);
    PGLB_LAUNCH_CHECK("spmm_stream128_kernel");
    const int64_t fblocks = (p.ntasks * 32 + 255) / 256;
    if (YM == 2) {
        spmm_stream_fixup_gat_kernel<float, false><<<(unsigned)fblocks, 256, 0, stream>>>(p, 1.0f);
    } else {
        spmm_stream_fixup_kernel<float, 1, RK><<<(unsigned)fblocks, 256, 0, stream>>>(p);
    }
    PGLB_LAUNCH_CHECK("spmm_stream_fixup_kernel");
    return PGLB_OK;
}

template <int ITERS, int RK>
static int launch_stream(const StreamP &p, int tiles, cudaStream_t stream) {
    typedef StreamCfg<ITERS> Cfg;
    static std::atomic<unsigned long long> attr_done{0};
    PGLB_CUDA(ensure_dyn_smem(spmm_stream_kernel<ITERS, RK>, Cfg::kSmem, attr_done));
    const int64_t blocks = (p.ntasks + Cfg::kWarps - 1) / Cfg::kWarps;
    PGLB_CHECK_ARG(blocks <= 0x7fffffffLL, PGLB_ESHAPE, "spmm_stream: grid too large");
    dim3 grid((unsigned)blocks, (unsigned)tiles);
    spmm_stream_kernel<ITERS, RK><<<grid, Cfg::kThreads, Cfg::kSmem, stream>>>(p);
    PGLB_LAUNCH_CHECK("spmm_stream_kernel");
    const int64_t fblocks = (p.ntasks * 32 + 255) / 256;
    dim3 fgrid((unsigned)fblocks, (unsigned)tiles);
    spmm_stream_fixup_kernel<float, ITERS, RK><<<fgrid, 256, 0, stream>>>(p);
    PGLB_LAUNCH_CHECK("spmm_stream_fixup_kernel");
    return PGLB_OK;
}

// Task plan and launch parameters shared by the wide-row runs below: fills everything of p but the edge operand,
// accumulate and the queue order p.dyn (left to the caller), and launches task_plan_kernel for tasks of T slots.
// `ws` holds >= stream_ws_bytes().
static int stream_prepare(StreamP &p, int64_t T, const int64_t *indptr, const int64_t *cols, const void *x, int64_t ldx,
                          void *out, int64_t ldo, int64_t n_dst, int64_t E, int64_t D, int reduce_op,
                          const float *scale_src, const float *scale_slot, const float *scale_dst,
                          const uint32_t *cols32, void *ws, size_t ws_bytes, cudaStream_t stream) {
    PGLB_CHECK_ARG(E > 0, PGLB_EINVAL, "spmm_stream_run: needs at least one slot");
    StreamWs w = stream_layout(ws, E, D, T);
    PGLB_CHECK_ARG(ws != nullptr && ws_bytes >= w.bytes, PGLB_EWORKSPACE,
                   "pglb_spmm_csr: workspace of %zu bytes needed (got %zu)", w.bytes, ws_bytes);
    p.indptr = indptr;
    p.cols = cols;
    p.x = reinterpret_cast<const float *>(x);
    p.ldx = ldx;
    p.out = reinterpret_cast<float *>(out);
    p.ldo = ldo;
    p.n_rows = n_dst;
    p.E = E;
    p.D = (int)D;
    p.reduce_op = reduce_op;
    p.scale_src = scale_src;
    p.scale_dst = scale_dst;
    p.scale_slot = scale_slot;  // spmm_v5 only; the other kernels gather scale_src
    p.T = T;
    p.ntasks = w.ntasks;
    p.first_row = w.first_row;
    p.start = w.start;
    p.partial = w.partial;
    p.partial_ml = w.partial_ml;
    p.dpad = w.dpad;
    p.tail_row = w.tail_row;
    p.cols32 = cols32;
    p.counter = w.counter;
    p.trace = trace_for(w.ntasks);
    {
        const int64_t blocks = (w.ntasks + 1 + 255) / 256;
        task_plan_kernel<<<(unsigned)blocks, 256, 0, stream>>>(indptr, n_dst, E, T, stream_snap(T),
                                                               w.ntasks, w.first_row, w.start, w.counter);
        PGLB_LAUNCH_CHECK("task_plan_kernel");
    }
    return PGLB_OK;
}

// Called by both spmm entries for the calls v5_eligible<T>() accepts; T is the element type of x and out.  `ws` holds
// >= stream_ws_bytes().
template <typename T>
int spmm_v5_run(const int64_t *indptr, const int64_t *cols, const void *x, int64_t ldx, void *out, int64_t ldo,
                int64_t n_dst, int64_t E, int64_t D, int reduce_op, const float *scale_src, const float *scale_slot,
                const float *scale_dst, const uint32_t *cols32, int l2_hints, int accumulate, void *ws,
                size_t ws_bytes, cudaStream_t stream) {
    StreamP p{};
    p.head_dim = 1;
    p.accumulate = accumulate;
    {
        const int rc = stream_prepare(p, stream_task_size(E), indptr, cols, x, ldx, out, ldo, n_dst, E, D, reduce_op,
                                      scale_src, scale_slot, scale_dst, cols32, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(0, p.ntasks);
    {
        const int rc = launch_empty_rows<T>(p, stream);
        if (rc) return rc;
    }
    return launch_v5<T>(p, cols32 != nullptr && cols != nullptr && l2_hints != 0, stream);
}

// pglb_propagate_f32 on the calls spmm_v5_run<float> takes with reduce_op SUM: the same task plan and kernel geometry,
// every row closed with epi's epilogue (empty rows by empty_rows_prop_kernel, cut rows by the fix-up)
int propagate_v5_run(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx, float *out, int64_t ldo,
                     int64_t n_dst, int64_t E, int64_t D, const float *scale_src, const float *scale_slot,
                     const float *scale_dst, const uint32_t *cols32, int l2_hints, const PropEpi &epi, void *ws,
                     size_t ws_bytes, cudaStream_t stream) {
    StreamP p{};
    p.head_dim = 1;
    {
        const int rc = stream_prepare(p, stream_task_size(E), indptr, cols, x, ldx, out, ldo, n_dst, E, D,
                                      PGLB_REDUCE_SUM, scale_src, scale_slot, scale_dst, cols32, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(0, p.ntasks);
    {
        const int rc = launch_empty_rows_prop(p, epi, stream);
        if (rc) return rc;
    }
    return launch_v5<float, true>(p, cols32 != nullptr && cols != nullptr && l2_hints != 0, stream, &epi);
}

template <typename T>
bool gatv2_attn_takes(int64_t D, int64_t head_dim, float slope, const void *f, int64_t ldf, const float *attn,
                      int64_t n_src) {
    return gatv2_attn_eligible<T>(D, head_dim, slope, f, ldf, attn, n_src);
}

// Single-pass GATv2 attention (GATv2Conv): out[d,h,:] = sum_j softmax_j(sum_c a[h,c] lrelu(f[src_j,h,c] + f[d,h,c]))
// f[src_j,h,:] on spmm_gat5_kernel<kScoreV2>.  T: element type of f and out; the call is one gatv2_attn_takes accepts.
// attn: a [H * head_dim] float32.  lse (nullable): the rows' log-sum-exp.  drop (nullable): the attention-dropout stream.
template <typename T>
int gatv2_attn_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *attn,
                   float slope, void *out, int64_t ldo, float *lse, int64_t n, int64_t E, int64_t H, int64_t head_dim,
                   const AttnDrop *drop, void *ws, size_t ws_bytes, cudaStream_t stream) {
    StreamP p{};
    p.ldy = H;
    p.head_dim = (int)head_dim;
    p.slope = slope;
    p.lse = lse;
    {
        const int rc = stream_prepare(p, gat_task_size(E), indptr, cols, f, ldf, out, ldo, n, E, H * head_dim,
                                      PGLB_REDUCE_SUM, nullptr, nullptr, nullptr, nullptr, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(1, p.ntasks);
    {
        const int rc = launch_empty_rows<T>(p, stream);
        if (rc) return rc;
    }
    if (drop) return launch_gatv2_attn<T, true>(p, attn, *drop, stream);
    return launch_gatv2_attn<T, false>(p, attn, AttnDrop{}, stream);
}

template <typename T>
bool fa_attn_takes(int64_t D, const void *f, int64_t ldf, const float *rec, int64_t n) {
    return fa_attn_eligible<T>(D, f, ldf, rec, n);
}

// Single-pass FAConv aggregation: out[d,:] = sum over the dst-CSR slots j of row d of w_j f[src_j,:], w_j =
// fa_weight(rec[src_j].x, rec[d].z, rec[src_j].y, rec[d].y) (common.cuh), on spmm_gat5_kernel<kScoreFA>.  rec: [n, 4]
// float32 node records (g_src, norm, g_dst, 0).  T: element type of f and out; the call is one fa_attn_takes accepts.
// drop (nullable): the attention-dropout stream, keep bit = head 0 of the 4-head keep word of the slot.
template <typename T>
int fa_attn_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *rec, void *out,
                int64_t ldo, int64_t n, int64_t E, int64_t D, const AttnDrop *drop, void *ws, size_t ws_bytes,
                cudaStream_t stream) {
    StreamP p{};
    p.ldy = 1;
    p.head_dim = (int)D;
    {
        const int rc = stream_prepare(p, gat_task_size(E), indptr, cols, f, ldf, out, ldo, n, E, D, PGLB_REDUCE_SUM,
                                      nullptr, nullptr, nullptr, nullptr, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(1, p.ntasks);
    {
        const int rc = launch_empty_rows<T>(p, stream);
        if (rc) return rc;
    }
    if (drop) return launch_fa_attn<T, true>(p, rec, *drop, stream);
    return launch_fa_attn<T, false>(p, rec, AttnDrop{}, stream);
}

// the instantiations the entries in spmm.cu call
template decltype(fa_attn_takes<float>) fa_attn_takes<float>;
template decltype(fa_attn_takes<__nv_bfloat16>) fa_attn_takes<__nv_bfloat16>;
template decltype(fa_attn_takes<__half>) fa_attn_takes<__half>;
template decltype(fa_attn_run<float>) fa_attn_run<float>;
template decltype(fa_attn_run<__nv_bfloat16>) fa_attn_run<__nv_bfloat16>;
template decltype(fa_attn_run<__half>) fa_attn_run<__half>;
template decltype(gatv2_attn_takes<float>) gatv2_attn_takes<float>;
template decltype(gatv2_attn_takes<__nv_bfloat16>) gatv2_attn_takes<__nv_bfloat16>;
template decltype(gatv2_attn_takes<__half>) gatv2_attn_takes<__half>;
template decltype(gatv2_attn_run<float>) gatv2_attn_run<float>;
template decltype(gatv2_attn_run<__nv_bfloat16>) gatv2_attn_run<__nv_bfloat16>;
template decltype(gatv2_attn_run<__half>) gatv2_attn_run<__half>;
template decltype(v5_eligible<float>) v5_eligible<float>;
template decltype(v5_eligible<__nv_bfloat16>) v5_eligible<__nv_bfloat16>;
template decltype(v5_eligible<__half>) v5_eligible<__half>;
template decltype(spmm_v5_run<float>) spmm_v5_run<float>;
template decltype(spmm_v5_run<__nv_bfloat16>) spmm_v5_run<__nv_bfloat16>;
template decltype(spmm_v5_run<__half>) spmm_v5_run<__half>;

// Called by pglb_spmm_csr_f32 for the wide-row shapes spmm_v5_kernel does not take (max / min, edge operands, identity
// columns).  `ws` holds >= stream_ws_bytes().
int spmm_stream_run(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx,
                    float *out, int64_t ldo, int64_t n_dst, int64_t n_src, int64_t E, int64_t D,
                    int reduce_op, const float *scale_src, const float *scale_dst,
                    const uint32_t *cols32, int l2_hints, int accumulate, const int64_t *eid,
                    const float *y, int64_t ldy, int y_bcast, int head_dim, int msg_op, void *ws,
                    size_t ws_bytes, cudaStream_t stream) {
    StreamP p{};
    p.eid = eid;
    p.y = y;
    p.ldy = ldy;
    p.y_bcast = y_bcast;
    p.head_dim = head_dim > 0 ? head_dim : 1;
    p.msg_op = msg_op;
    p.accumulate = accumulate;
    {
        const int rc = stream_prepare(p, stream_task_size(E), indptr, cols, x, ldx, out, ldo, n_dst, E, D, reduce_op,
                                      scale_src, nullptr, scale_dst, cols32, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(2, p.ntasks);   // round 1's kernel (max / min, edge operands): descending queue
    {
        const int rc = launch_empty_rows<float>(p, stream);
        if (rc) return rc;
    }
    const int64_t cv = D / 4;
    const int rk = (reduce_op >= PGLB_REDUCE_MAX) ? 1 : 0;
    const bool small_ids = (cols ? n_src : E) < 0x7fffffffLL && ldx * 4 < 0xffffffffLL;
    if (cv <= 32 && small_ids) {
        if (y) {  // edge operand: plain int64 ids, no source scale
            return rk ? launch_stream128<1, false, 0, 1>(p, stream) : launch_stream128<0, false, 0, 1>(p, stream);
        }
        const int pk = (cols32 && cols) ? (l2_hints ? 2 : 1) : 0;
#define PGLB_S128(RKV, SC)                                                         \
    (pk == 2 ? launch_stream128<RKV, SC, 2, 0>(p, stream)                          \
             : pk == 1 ? launch_stream128<RKV, SC, 1, 0>(p, stream) : launch_stream128<RKV, SC, 0, 0>(p, stream))
        if (scale_src) return rk ? PGLB_S128(1, true) : PGLB_S128(0, true);
        return rk ? PGLB_S128(1, false) : PGLB_S128(0, false);
#undef PGLB_S128
    }
    const int iters = cv <= 64 ? 2 : 4;
    const int tiles = (int)((cv + 32 * iters - 1) / (32 * iters));
    if (iters == 2) return rk ? launch_stream<2, 1>(p, tiles, stream) : launch_stream<2, 0>(p, tiles, stream);
    return rk ? launch_stream<4, 1>(p, tiles, stream) : launch_stream<4, 0>(p, tiles, stream);
}

// ---- narrow2 host side --------------------------------------------------------------------------------------
// Slots per task of the narrow kernel: the wide kernel's choice rounded up to whole chunks of (32 / LPR) * 32 slots
static int narrow2_lpr(int64_t D) { return D <= 16 ? 4 : (D <= 32 ? 8 : 16); }
static int64_t narrow2_task_size(int64_t E, int64_t D) {
    const int64_t chunk = (32 / narrow2_lpr(D)) * 32;
    const int64_t t = stream_task_size(E);
    return (t + chunk - 1) / chunk * chunk;
}
size_t narrow2_ws_bytes(int64_t E, int64_t D) { return stream_layout(nullptr, E, D, narrow2_task_size(E, D)).bytes; }

template <int L>
static void launch_narrow2(const NarrowP &p, int sc, bool hot, bool prop, unsigned blocks, cudaStream_t stream) {
#define PGLB_N2K(SC, MN, HT) spmm_narrow2_kernel<L, SC, MN, HT><<<blocks, kNarrowWarps * 32, 0, stream>>>(p)
#define PGLB_N2P(SC, HT) spmm_narrow2_kernel<L, SC, false, HT, true><<<blocks, kNarrowWarps * 32, 0, stream>>>(p)
    if (prop) {  // pglb_propagate_narrow_f32: sum
        if (sc == 1) hot ? PGLB_N2P(1, true) : PGLB_N2P(1, false);
        else if (sc == 2) hot ? PGLB_N2P(2, true) : PGLB_N2P(2, false);
        else hot ? PGLB_N2P(0, true) : PGLB_N2P(0, false);
        return;
    }
    if (p.mean) {  // mean (GraphSAGE): no L2 hints
        if (sc == 1) PGLB_N2K(1, true, false);
        else if (sc == 2) PGLB_N2K(2, true, false);
        else PGLB_N2K(0, true, false);
        return;
    }
    if (hot) {
        if (sc == 1) PGLB_N2K(1, false, true);
        else if (sc == 2) PGLB_N2K(2, false, true);
        else PGLB_N2K(0, false, true);
    } else {
        if (sc == 1) PGLB_N2K(1, false, false);
        else if (sc == 2) PGLB_N2K(2, false, false);
        else PGLB_N2K(0, false, false);
    }
#undef PGLB_N2K
#undef PGLB_N2P
}

// epi (nullable, sum only): pglb_propagate_narrow_f32's row epilogue
int narrow2_run(const uint32_t *plan, const int32_t *nz_row, const int32_t *blk_k, const int64_t *indptr, const float *x,
                int64_t ldx, float *out, int64_t ldo, int64_t n_dst, int64_t E, int64_t D, int reduce_op,
                const float *scale_src, const float *sval, const float *scale_dst, int hot, void *ws, size_t ws_bytes,
                cudaStream_t stream, const PropEpi *epi = nullptr) {
    const int64_t T = narrow2_task_size(E, D);
    StreamWs w = stream_layout(ws, E, D, T);
    PGLB_CHECK_ARG(ws != nullptr && ws_bytes >= w.bytes, PGLB_EWORKSPACE,
                   "pglb_spmm_narrow_f32: workspace of %zu bytes needed (got %zu)", w.bytes, ws_bytes);
    NarrowP p{};
    p.plan = plan;
    p.nz_row = nz_row;
    p.blk_k = blk_k;
    p.indptr = indptr;
    p.x = x;
    p.ldx = ldx;
    p.out = out;
    p.ldo = ldo;
    p.E = E;
    p.D = (int)D;
    p.mean = reduce_op == PGLB_REDUCE_MEAN;
    p.scale_src = scale_src;
    p.sval = sval;
    p.scale_dst = scale_dst;
    p.T = T;
    p.ntasks = w.ntasks;
    p.partial = w.partial;
    p.dpad = w.dpad;
    p.tail_row = w.tail_row;
    // the shared pieces: zero-fill of empty rows before, fix-up of task-cut rows after
    StreamP sp{};
    sp.indptr = indptr;
    sp.out = out;
    sp.ldo = ldo;
    sp.n_rows = n_dst;
    sp.E = E;
    sp.D = (int)D;
    sp.reduce_op = reduce_op;
    sp.scale_dst = scale_dst;
    sp.T = T;
    sp.ntasks = w.ntasks;
    sp.partial = w.partial;
    sp.dpad = w.dpad;
    sp.tail_row = w.tail_row;
    if (epi) p.epi = *epi;
    {
        const int rc = epi ? launch_empty_rows_prop(sp, *epi, stream) : launch_empty_rows<float>(sp, stream);
        if (rc) return rc;
    }
    const int64_t blocks = (p.ntasks + kNarrowWarps - 1) / kNarrowWarps;
    PGLB_CHECK_ARG(blocks <= 0x7fffffffLL, PGLB_ESHAPE, "spmm_narrow2: grid too large");
    const int lpr = narrow2_lpr(D);
    const int sc = sval ? 2 : (scale_src ? 1 : 0);
    if (lpr == 4) launch_narrow2<4>(p, sc, hot != 0, epi != nullptr, (unsigned)blocks, stream);
    else if (lpr == 8) launch_narrow2<8>(p, sc, hot != 0, epi != nullptr, (unsigned)blocks, stream);
    else launch_narrow2<16>(p, sc, hot != 0, epi != nullptr, (unsigned)blocks, stream);
    PGLB_LAUNCH_CHECK("spmm_narrow2_kernel");
    const int64_t fblocks = (p.ntasks * 32 + 255) / 256;
    if (epi)
        spmm_stream_fixup_prop_kernel<<<(unsigned)fblocks, 256, 0, stream>>>(sp, *epi);
    else
        spmm_stream_fixup_kernel<float, 1, 0><<<(unsigned)fblocks, 256, 0, stream>>>(sp);
    PGLB_LAUNCH_CHECK("spmm_stream_fixup_kernel");
    return PGLB_OK;
}

// Whether spmm_gat5_kernel<T> takes a call (the entries' argument checks, before any CUDA call)
template <typename T>
bool gat5_takes(int64_t D, float slope, const void *f, int64_t ldf, const float *attn_src, int64_t H, int64_t n_src) {
    return gat5_eligible<T>(D, slope, f, ldf, attn_src, H, n_src);
}

// Single-pass GAT aggregation (inference): out[d,h,:] = sum_j softmax_j(leaky(as[src_j,h] + ad[d,h])) f[src_j,h,:].
// T: element type of f and out.  float32 calls outside gat5 take spmm_stream128_kernel<YM = 2>; a 16-bit call must be
// one gat5 takes.  drop (nullable, training only: lse non-NULL): the attention-dropout stream of the DROP kernels.
template <typename T>
int gat_fused_run(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, void *out,
                  int64_t ldo, int64_t n_dst, int64_t n_src, int64_t E, int64_t D, int64_t H,
                  const float *attn_src, const float *attn_dst, float slope, float *lse, const AttnDrop *drop, void *ws,
                  size_t ws_bytes, cudaStream_t stream) {
    // the row statistics are written by spmm_gat5_kernel and the merge kernel only
    const bool tma = gat5_eligible<T>(D, slope, f, ldf, attn_src, H, n_src);
    PGLB_CHECK_ARG(!lse || tma, PGLB_EUNSUPPORTED,
                   "pglb_gat_fused_train_csr_f32: shape outside the TMA kernel (H %% 4, 16-byte rows, 0 <= slope <= 1)");
    PGLB_CHECK_ARG(sizeof(T) == 4 || tma, PGLB_EUNSUPPORTED,
                   "pglb_gat_fused_csr_x16: shape outside the 16-bit kernel (H %% 4, H <= 32, D %% 8, 16-byte rows, "
                   "0 <= slope <= 1)");
    StreamP p{};
    p.y = attn_src;
    p.ldy = H;
    p.y_bcast = PGLB_BCAST_HEAD;
    p.head_dim = (int)(D / H);
    p.attn_dst = attn_dst;
    p.slope = slope;
    p.lse = lse;
    {
        const int rc = stream_prepare(p, gat_task_size(E), indptr, cols, f, ldf, out, ldo, n_dst, E, D, PGLB_REDUCE_SUM,
                                      nullptr, nullptr, nullptr, nullptr, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(1, p.ntasks);
    {
        const int rc = launch_empty_rows<T>(p, stream);
        if (rc) return rc;
    }
    if (tma && drop) return launch_gat5<T, true>(p, attn_src, H, *drop, stream);
    if (tma) return launch_gat5<T, false>(p, attn_src, H, AttnDrop{}, stream);
    if constexpr (sizeof(T) == 4) return launch_stream128<0, false, 0, 2>(p, stream);
    return PGLB_EUNSUPPORTED;   // not reached: refused above
}

template <typename T>
bool dot_attn_takes(int64_t D, int64_t head_dim, const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v,
                    int64_t ldv, const void *e, int64_t lde, int64_t n_src) {
    if (e) return dot_attn_e_eligible<T>(D, head_dim, q, ldq, k, ldk, v, ldv, e, lde, n_src);
    return dot_attn_eligible<T>(D, head_dim, q, ldq, k, ldk, v, ldv, n_src);
}

// Single-pass dot-product attention (TransformerConv): out[d,h,:] = sum_j softmax_j(<q[d,h,:], k[src_j,h,:]>) v[src_j,h,:]
// on spmm_gat5_kernel<DOT>.  With edge features e (nullable; [E, D] in edge-id order, eid the dst-CSR's slot -> edge
// id): k + e and v + e in place of k and v, on spmm_gat5_kernel<DOTE>.  T: element type of q, k, v, e and out; the
// call is one dot_attn_takes accepts.  lse (nullable): the rows' log-sum-exp.  drop (nullable): the attention-dropout
// stream.
template <typename T>
int dot_attn_run(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq, const void *k, int64_t ldk,
                 const void *v, int64_t ldv, const int64_t *eid, const void *e, int64_t lde, void *out, int64_t ldo,
                 float *lse, int64_t n_dst, int64_t E, int64_t H, int64_t head_dim, const AttnDrop *drop, void *ws,
                 size_t ws_bytes, cudaStream_t stream) {
    StreamP p{};
    p.ldy = H;
    p.head_dim = (int)head_dim;
    p.lse = lse;
    {
        const int rc = stream_prepare(p, gat_task_size(E), indptr, cols, v, ldv, out, ldo, n_dst, E, H * head_dim,
                                      PGLB_REDUCE_SUM, nullptr, nullptr, nullptr, nullptr, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    p.dyn = dyn_mode(1, p.ntasks);
    {
        const int rc = launch_empty_rows<T>(p, stream);
        if (rc) return rc;
    }
    if (e && drop) return launch_dot_attn_e<T, true>(p, q, ldq, k, ldk, eid, e, lde, *drop, stream);
    if (e) return launch_dot_attn_e<T, false>(p, q, ldq, k, ldk, eid, e, lde, AttnDrop{}, stream);
    if (drop) return launch_dot_attn<T, true>(p, q, ldq, k, ldk, *drop, stream);
    return launch_dot_attn<T, false>(p, q, ldq, k, ldk, AttnDrop{}, stream);
}

// the instantiations the entries in spmm.cu call
template decltype(dot_attn_takes<float>) dot_attn_takes<float>;
template decltype(dot_attn_takes<__nv_bfloat16>) dot_attn_takes<__nv_bfloat16>;
template decltype(dot_attn_takes<__half>) dot_attn_takes<__half>;
template decltype(dot_attn_run<float>) dot_attn_run<float>;
template decltype(dot_attn_run<__nv_bfloat16>) dot_attn_run<__nv_bfloat16>;
template decltype(dot_attn_run<__half>) dot_attn_run<__half>;
template decltype(gat5_takes<__nv_bfloat16>) gat5_takes<__nv_bfloat16>;
template decltype(gat5_takes<__half>) gat5_takes<__half>;
template decltype(gat_fused_run<float>) gat_fused_run<float>;
template decltype(gat_fused_run<__nv_bfloat16>) gat_fused_run<__nv_bfloat16>;
template decltype(gat_fused_run<__half>) gat_fused_run<__half>;

}  // namespace pglb

using namespace pglb;

extern "C" int pglb_debug_task_trace(void *buffer, int64_t capacity_tasks) {
    g_trace_cap.store(buffer ? capacity_tasks : 0, std::memory_order_release);
    g_trace.store(reinterpret_cast<long long *>(buffer), std::memory_order_release);
    return PGLB_OK;
}

namespace pglb {
// spmm.cu: pglb_propagate_*'s checks of the epilogue operands
int prop_check_args(const char *entry, const void *x, int64_t ldx, int64_t n_src, const void *out, int64_t ldo,
                    int64_t n_dst, int64_t D, const float *h, int64_t ldh, const float *acc_in, int64_t ld_acc_in,
                    const float *acc_out, int64_t ld_acc_out, int flags);
bool prop_rows16(const PropEpi &e);
}  // namespace pglb

extern "C" int pglb_spmm_narrow_ws(int64_t num_edges, int64_t D, size_t *ws_bytes) {
    PGLB_CHECK_ARG(ws_bytes != nullptr && num_edges >= 0 && D > 0, PGLB_EINVAL, "pglb_spmm_narrow_ws: bad argument");
    *ws_bytes = narrow2_ws_bytes(num_edges, D);
    return PGLB_OK;
}

extern "C" int pglb_spmm_narrow_f32(const uint32_t *plan, const int32_t *nz_row, const int32_t *blk_k,
                                    const int64_t *indptr, const float *x, int64_t ldx, float *out, int64_t ldo,
                                    int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, int reduce_op,
                                    const float *scale_src, const float *scale_slot, const float *scale_dst, int flags,
                                    void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_dst > 0 && n_src > 0 && num_edges > 0, PGLB_EINVAL, "pglb_spmm_narrow_f32: empty problem");
    PGLB_CHECK_ARG(D >= 4 && D <= 64 && D % 4 == 0, PGLB_ESHAPE, "pglb_spmm_narrow_f32: D must be 4..64, a multiple of 4");
    PGLB_CHECK_ARG(reduce_op == PGLB_REDUCE_SUM || reduce_op == PGLB_REDUCE_MEAN, PGLB_EINVAL,
                   "pglb_spmm_narrow_f32: sum or mean only");
    PGLB_CHECK_ARG(plan && nz_row && blk_k && indptr && x && out, PGLB_EINVAL, "pglb_spmm_narrow_f32: NULL pointer");
    PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (ldx % 4) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                       (ldo % 4) == 0,
                   PGLB_ESHAPE, "pglb_spmm_narrow_f32: x / out rows must be 16-byte aligned");
    PGLB_CHECK_ARG(n_src < 0x40000000LL && ldx * 4 < 0xffffffffLL, PGLB_ESHAPE, "pglb_spmm_narrow_f32: n_src < 2^30 needed");
    return narrow2_run(plan, nz_row, blk_k, indptr, x, ldx, out, ldo, n_dst, num_edges, D, reduce_op, scale_src, scale_slot,
                       scale_dst, flags & PGLB_SPMM_L2_HINTS, ws, ws_bytes, stream);
}

extern "C" int pglb_propagate_narrow_f32(const uint32_t *plan, const int32_t *nz_row, const int32_t *blk_k,
                                         const int64_t *indptr, const float *x, int64_t ldx, float *out, int64_t ldo,
                                         int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D,
                                         const float *scale_src, const float *scale_slot, const float *scale_dst,
                                         float a, float b, const float *h, int64_t ldh, const float *acc_in,
                                         int64_t ld_acc_in, float *acc_out, int64_t ld_acc_out, float c,
                                         const float *c_dev, int flags, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PGLB_CHECK_ARG(n_dst > 0 && n_src > 0 && num_edges > 0, PGLB_EINVAL, "pglb_propagate_narrow_f32: empty problem");
    PGLB_CHECK_ARG(D >= 4 && D <= 64 && D % 4 == 0, PGLB_ESHAPE,
                   "pglb_propagate_narrow_f32: D must be 4..64, a multiple of 4");
    PGLB_CHECK_ARG(plan && nz_row && blk_k && indptr && x && out, PGLB_EINVAL, "pglb_propagate_narrow_f32: NULL pointer");
    PGLB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (ldx % 4) == 0 &&
                       (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (ldo % 4) == 0,
                   PGLB_ESHAPE, "pglb_propagate_narrow_f32: x / out rows must be 16-byte aligned");
    PGLB_CHECK_ARG(n_src < 0x40000000LL && ldx * 4 < 0xffffffffLL, PGLB_ESHAPE,
                   "pglb_propagate_narrow_f32: n_src < 2^30 needed");
    {
        const int rc = prop_check_args("pglb_propagate_narrow_f32", x, ldx, n_src, out, ldo, n_dst, D, h, ldh, acc_in,
                                       ld_acc_in, acc_out, ld_acc_out, flags);
        if (rc) return rc;
    }
    const PropEpi e{h, ldh, acc_in, ld_acc_in, acc_out, ld_acc_out, a, b, c, c_dev};
    PGLB_CHECK_ARG(prop_rows16(e), PGLB_EUNSUPPORTED,
                   "pglb_propagate_narrow_f32: h / acc rows must be 16-byte aligned like x and out");
    return narrow2_run(plan, nz_row, blk_k, indptr, x, ldx, out, ldo, n_dst, num_edges, D, PGLB_REDUCE_SUM, scale_src,
                       scale_slot, scale_dst, flags & PGLB_SPMM_L2_HINTS, ws, ws_bytes, stream, &e);
}
