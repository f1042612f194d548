// host.cpp -- host-side entry points of libpglb: error reporting, the numpy-mode CSR build
// (twin of pgl/graph_kernel.pyx:59-88) and the METIS K-way wrapper
// (pgl/graph_kernel.pyx:434-472), which dlopen()s a libmetis built with IDXTYPEWIDTH=64, and the alias table build
// (pgl/graph_kernel.pyx:368-393).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "pglb.h"

namespace pglb {
thread_local char g_err[512] = {0};
std::atomic<long long> g_launches{0};

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int cuda_fail(cudaError_t e, const char *what) {
    snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    cudaGetLastError();  // clear sticky-less errors
    return PGLB_CUDA_ERR_BASE + (int)e;
}
}  // namespace pglb

using namespace pglb;

extern "C" int pglb_version(void) { return PGLB_VERSION; }
extern "C" const char *pglb_last_error(void) { return g_err; }
extern "C" int64_t pglb_launch_count(void) { return (int64_t)g_launches.load(); }

extern "C" int pglb_build_index_host(const int64_t *u, int64_t us, const int64_t *v, int64_t vs,
                                     int64_t E, int64_t N, int64_t *degree, int64_t *indptr,
                                     int64_t *sorted_u, int64_t *sorted_v, int64_t *sorted_eid) {
    if (E < 0 || N < 0) return fail(PGLB_EINVAL, "pglb_build_index_host: negative size");
    if (!indptr || (N > 0 && !degree)) return fail(PGLB_EINVAL, "pglb_build_index_host: NULL output");
    if (E > 0 && (!u || !v || !sorted_u || !sorted_v || !sorted_eid))
        return fail(PGLB_EINVAL, "pglb_build_index_host: NULL edge pointer");
    if (us < 1 || vs < 1) return fail(PGLB_EINVAL, "pglb_build_index_host: bad stride");
    for (int64_t i = 0; i < N; ++i) degree[i] = 0;
    for (int64_t i = 0; i < E; ++i) {
        const int64_t k = u[i * us];
        if (k < 0 || k >= N)
            return fail(PGLB_ESHAPE, "pglb_build_index_host: node id %lld out of range [0,%lld)",
                        (long long)k, (long long)N);
        degree[k] += 1;
    }
    indptr[0] = 0;
    for (int64_t i = 0; i < N; ++i) indptr[i + 1] = indptr[i] + degree[i];
    std::vector<int64_t> cursor(indptr, indptr + N);
    for (int64_t i = 0; i < E; ++i) {
        const int64_t k = u[i * us];
        const int64_t p = cursor[k]++;
        sorted_u[p] = k;
        sorted_v[p] = v[i * vs];
        sorted_eid[p] = i;
    }
    return PGLB_OK;
}

extern "C" int pglb_memcpy2d_async(void *dst, size_t dst_pitch, const void *src, size_t src_pitch,
                                   size_t width_bytes, size_t height, int kind, void *stream) {
    if (width_bytes == 0 || height == 0) return PGLB_OK;
    if (!dst || !src || (kind != 1 && kind != 2) || dst_pitch < width_bytes || src_pitch < width_bytes)
        return fail(PGLB_EINVAL, "pglb_memcpy2d_async: bad args");
    cudaError_t e = cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width_bytes, height,
                                      kind == 1 ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost,
                                      reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpy2DAsync");
    return PGLB_OK;
}

// ---- alias table (graph_kernel.pyx:368-393) ------------------------------------------------------
// Vose's construction as the reference runs it: alias = probs * n in float64, the indices above and below 1 on two
// stacks, and each step pairs the top of both.  Built without FMA contraction (pgl_b200/build.py), so every value is
// the reference's bit for bit, its rounding leftovers (entries whose events stay 0) included.
extern "C" int pglb_alias_build_host(const double *probs, int64_t n, double *alias, int64_t *events) {
    if (n < 0) return fail(PGLB_EINVAL, "pglb_alias_build_host: negative n");
    if (n == 0) return PGLB_OK;
    if (!probs || !alias || !events) return fail(PGLB_EINVAL, "pglb_alias_build_host: NULL pointer");
    const double dn = (double)n;
    std::vector<int64_t> larger, smaller;
    for (int64_t i = 0; i < n; ++i) {
        alias[i] = probs[i] * dn;
        events[i] = 0;
    }
    for (int64_t i = 0; i < n; ++i) {
        if (alias[i] > 1) larger.push_back(i);
        else if (alias[i] < 1) smaller.push_back(i);
    }
    while (!smaller.empty() && !larger.empty()) {
        const int64_t s = smaller.back(), l = larger.back();
        smaller.pop_back();
        events[s] = l;
        alias[l] -= (1 - alias[s]);
        if (alias[l] <= 1) larger.pop_back();
        if (alias[l] < 1) smaller.push_back(l);
    }
    return PGLB_OK;
}

// ---- peer-mappable buffers (CUDA IPC) ---------------------------------------------------------
extern "C" int pglb_ipc_alloc(size_t bytes, void **dev_ptr, void *handle64) {
    if (!dev_ptr || !handle64 || bytes == 0) return fail(PGLB_EINVAL, "pglb_ipc_alloc: bad args");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc");
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return cuda_fail(e, "cudaIpcGetMemHandle");
    }
    memcpy(handle64, &h, 64);
    *dev_ptr = p;
    return PGLB_OK;
}

extern "C" int pglb_ipc_free(void *dev_ptr) {
    if (!dev_ptr) return PGLB_OK;
    cudaError_t e = cudaFree(dev_ptr);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFree");
    return PGLB_OK;
}

extern "C" int pglb_ipc_open(const void *handle64, void **peer_ptr) {
    if (!handle64 || !peer_ptr) return fail(PGLB_EINVAL, "pglb_ipc_open: bad args");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void *p = nullptr;
    // opened under the CALLER's current device: the mapping (and lazily enabled peer access)
    // belongs to the GPU whose kernels will read it
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return cuda_fail(e, "cudaIpcOpenMemHandle");
    *peer_ptr = p;
    return PGLB_OK;
}

extern "C" int pglb_ipc_close(void *peer_ptr) {
    if (!peer_ptr) return PGLB_OK;
    cudaError_t e = cudaIpcCloseMemHandle(peer_ptr);
    if (e != cudaSuccess) return cuda_fail(e, "cudaIpcCloseMemHandle");
    return PGLB_OK;
}

// ---- METIS through dlopen ---------------------------------------------------------------
typedef int (*metis_part_fn)(int64_t *nvtxs, int64_t *ncon, int64_t *xadj, int64_t *adjncy,
                             int64_t *vwgt, int64_t *vsize, int64_t *adjwgt, int64_t *nparts,
                             float *tpwgts, float *ubvec, int64_t *options, int64_t *edgecut,
                             int64_t *part);

static std::mutex g_metis_mu;
static void *g_metis_handle = nullptr;
static char g_metis_path[1024] = {0};

extern "C" int pglb_metis_partition(const char *libmetis_path, int64_t num_nodes,
                                    const int64_t *indptr, const int64_t *adjncy, int64_t nparts,
                                    const int64_t *node_weights, const int64_t *edge_weights,
                                    int recursive, int64_t *part) {
    if (num_nodes < 0 || nparts < 1) return fail(PGLB_EINVAL, "pglb_metis_partition: bad size");
    if (num_nodes == 0) return PGLB_OK;
    if (!indptr || !part) return fail(PGLB_EINVAL, "pglb_metis_partition: NULL pointer");
    if (nparts == 1) {  // pgl/partition.py:63-64 short-circuit
        for (int64_t i = 0; i < num_nodes; ++i) part[i] = 0;
        return PGLB_OK;
    }
    metis_part_fn fn = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_metis_mu);
        const char *path = libmetis_path && libmetis_path[0] ? libmetis_path : "libmetis.so";
        if (!g_metis_handle || strncmp(g_metis_path, path, sizeof(g_metis_path)) != 0) {
            void *h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
            if (!h) return fail(PGLB_ENOLIB, "pglb_metis_partition: cannot load %s: %s", path, dlerror());
            g_metis_handle = h;
            strncpy(g_metis_path, path, sizeof(g_metis_path) - 1);
        }
        fn = (metis_part_fn)dlsym(g_metis_handle,
                                  recursive ? "METIS_PartGraphRecursive" : "METIS_PartGraphKway");
        if (!fn) return fail(PGLB_ENOLIB, "pglb_metis_partition: symbol missing in %s", g_metis_path);
    }
    int64_t nv = num_nodes, ncon = 1, np = nparts, edgecut = -1;
    // METIS does not modify xadj/adjncy/vwgt/adjwgt; its prototype is just not const-correct.
    int rc = fn(&nv, &ncon, const_cast<int64_t *>(indptr), const_cast<int64_t *>(adjncy),
                const_cast<int64_t *>(node_weights), nullptr, const_cast<int64_t *>(edge_weights),
                &np, nullptr, nullptr, nullptr, &edgecut, part);
    if (rc != 1) return fail(PGLB_EINVAL, "pglb_metis_partition: METIS returned %d", rc);
    return PGLB_OK;
}
