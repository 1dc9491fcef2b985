// Temporal-graph constructor, device half (SURVEY.md 8f rank 1): edge list -> CSR-by-destination with temporal
// weights, the exact input layout of the GraphSAGE-T kernels.  Spec = nerrf_b200/graph.py csr_from_edges
// (reference prose: docs/content/docs/architecture.mdx:32-42 "sliding window ... edge weight"):
//
//   order  = stable sort of the edges by (dst, t)            (ties keep input order, like np.lexsort)
//   col[i] = src[order[i]]
//   ew[i]  = conf[e] * exp(-(t_ref - t[e]) / tau),  e = order[i]   (every fp32 op individually rounded)
//   rowptr[v] = number of edges with dst < v
//
// One 64-bit key per edge = dst << 32 | orderable(t); ONE stable LSD radix sort over the low 32 + ceil(log2 N)
// bits (library code: cub::DeviceRadixSort, part of the CUDA toolkit -- HBM-bound byte shuffling, nothing to fuse),
// then one fused pass of ours that gathers src/t/conf through the permutation, evaluates the weight and writes
// rowptr from the dst boundaries of the sorted keys (no atomics anywhere: the result is deterministic).
// String work (path/inode dedup, feature counts) stays on the host: nerrf_b200/graph.py graph_from_events.
#include "common.cuh"
#include "radix_sort.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <stdlib.h>

namespace nerrf {

__global__ void __launch_bounds__(256) csr_keys_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                                        const float* __restrict__ t, int64_t E, int64_t N,
                                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                        int* __restrict__ bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride) {
        int32_t d = dst[i];
        const int32_t s = src[i];
        if ((uint32_t)d >= (uint64_t)N || (uint32_t)s >= (uint64_t)N) { *bad = 1; d = 0; }   // keep the later passes in range
        const uint32_t b = __float_as_uint(t[i] + 0.0f);                 // -0.0 -> +0.0: they compare equal on the host
        const uint32_t ord = b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u);   // monotone float -> uint
        if (i > 0) {                                                     // time order of the input (see the sort below)
            const uint32_t bp = __float_as_uint(t[i - 1] + 0.0f);
            if ((bp ^ ((bp >> 31) ? 0xffffffffu : 0x80000000u)) > ord) bad[1] = 1;
        }
        keys[i] = ((uint64_t)(uint32_t)d << 32) | ord;
        vals[i] = (uint32_t)i;
    }
}

// rowptr[lo..hi] = val; short runs inline by the owning lane, long runs (empty-row gaps, the tail after the last
// edge) by the whole warp so a sparse destination range cannot serialise one thread.
template <typename RP>
__device__ __forceinline__ void fill_rows(RP* __restrict__ rowptr, int64_t lo, int64_t hi, int64_t val, bool active, int lane) {
    const bool is_long = active && (hi - lo) >= 16;
    if (active && !is_long) for (int64_t v = lo; v <= hi; ++v) rowptr[v] = (RP)val;
    unsigned m = __ballot_sync(0xffffffffu, is_long);
    while (m) {
        const int l = __ffs(m) - 1;
        m &= m - 1;
        const long long lo_ = __shfl_sync(0xffffffffu, (long long)lo, l), hi_ = __shfl_sync(0xffffffffu, (long long)hi, l);
        const long long val_ = __shfl_sync(0xffffffffu, (long long)val, l);
        for (long long v = lo_ + lane; v <= hi_; v += 32) rowptr[v] = (RP)val_;
    }
}

template <typename RP>
__global__ void __launch_bounds__(256) csr_finish_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ perm,
                                                          const int32_t* __restrict__ src, const float* __restrict__ t,
                                                          const float* __restrict__ conf, int64_t E, int64_t N, float t_ref,
                                                          float tau, RP* __restrict__ rowptr, int32_t* __restrict__ col,
                                                          float* __restrict__ ew, uint32_t* __restrict__ perm_out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    for (int64_t wb = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); wb < E; wb += stride) {   // warp-uniform trip count
        const int64_t i = wb + lane;
        const bool ok = i < E;
        int64_t d = 0, dprev = 0;
        if (ok) {
            d = (int64_t)(keys[i] >> 32);
            dprev = i > 0 ? (int64_t)(keys[i - 1] >> 32) : -1;
        }
        fill_rows(rowptr, dprev + 1, d, i, ok && d > dprev, lane);          // first edge of row d and the empty rows before it
        fill_rows(rowptr, d + 1, N, E, ok && i == E - 1, lane);             // rows after the last edge, and rowptr[N]
        if (ok) {
            const uint32_t e = perm[i];
            if (perm_out) perm_out[i] = e;                               // CSR position -> index in the input edge list
            col[i] = __ldg(src + e);
            const float age = __fsub_rn(t_ref, __ldg(t + e));
            const float z = __fdiv_rn(-age, tau);
            ew[i] = __fmul_rn(__ldg(conf + e), expf(z));
        }
    }
}

template <typename RP>
__global__ void csr_empty_kernel(RP* rowptr, int64_t N) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v <= N; v += stride) rowptr[v] = 0;
}


// ---------------------------------------------------------------------------------------------------------------
// Per-node features (SURVEY.md 8f rank 1, "feature counts"): spec = nerrf_b200/ingest.py graph_from_columns /
// graph.py graph_from_events (node schema: docs/content/docs/architecture.mdx:144-160, threat-model.mdx:154-184).
// Pass 1 over events: integer atomics only (event-kind counts, byte sums, first/last touch time as ordered int64,
// path flag bits, degree) -> deterministic.  Pass 2 over nodes: the 20 used feature columns in double, rounded once.
//
// An event's byte count is the count argument of write(2) as traced at syscall entry: the traced process picks it, up to
// 2^64 - 1.  Every feature reads it as uint64 clamped to Linux's per-call transfer cap MAX_RW_COUNT (graph.py
// MAX_RW_COUNT), so a node's sum of fewer than 2^29 events stays below 2^60: exact in uint64, converted to double once.
constexpr unsigned long long kMaxRwCount = 0x7ffff000ull;

__device__ __forceinline__ unsigned long long clamp_rw(uint64_t b) { return b < kMaxRwCount ? b : kMaxRwCount; }
struct NodeAcc {            // 64 bytes per node
    int32_t cnt[8];
    unsigned long long bytes;
    long long first, last;  // bit patterns of non-negative doubles (monotone as signed integers)
    int32_t flags;          // NERRF_PATH_* bits | 0x100 = label
    int32_t deg;            // in-degree == out-degree: every event adds each edge in both directions
};

__global__ void __launch_bounds__(256) node_acc_init_kernel(NodeAcc* __restrict__ acc, int64_t N) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < N; v += stride) {
        NodeAcc a;
#pragma unroll
        for (int k = 0; k < 8; ++k) a.cnt[k] = 0;
        a.bytes = 0ull; a.first = 0x7fffffffffffffffll; a.last = -0x7fffffffffffffffll - 1; a.flags = 0; a.deg = 0;
        acc[v] = a;
    }
}

__device__ __forceinline__ void touch(NodeAcc* __restrict__ acc, int32_t v, int slot, unsigned long long size, long long tb, int deg) {
    NodeAcc* a = acc + v;
    atomicAdd(&a->cnt[slot], 1);
    if (size) atomicAdd(&a->bytes, size);
    atomicMin(&a->first, tb);
    atomicMax(&a->last, tb);
    atomicAdd(&a->deg, deg);
}

__global__ void __launch_bounds__(256) node_acc_events_kernel(const int32_t* __restrict__ node_p, const int32_t* __restrict__ node_f,
                                                               const int32_t* __restrict__ node_g, const double* __restrict__ t,
                                                               const uint8_t* __restrict__ slot, const uint64_t* __restrict__ bytes,
                                                               const uint8_t* __restrict__ pflags, int64_t n, int64_t N,
                                                               NodeAcc* __restrict__ acc, int* __restrict__ bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int32_t p = node_p[i], f = node_f[i], g = node_g ? node_g[i] : -1;
        const double ti = t[i];
        if ((uint32_t)p >= (uint64_t)N || (uint32_t)f >= (uint64_t)N || g < -1 || (int64_t)g >= N || !(ti >= 0.0) || slot[i] > 7) {
            *bad = 1;
            continue;
        }
        const long long tb = __double_as_longlong(ti + 0.0);
        const int s = slot[i];
        const unsigned long long sz = clamp_rw(bytes[i]);
        touch(acc, p, s, sz, tb, 1);
        touch(acc, f, s, sz, tb, g >= 0 ? 2 : 1);
        if (g >= 0) touch(acc, g, s, sz, tb, 1);
        const int fl = (int)pflags[i] | ((s == 1 || s == 2) ? 0x100 : 0);
        if (fl) atomicOr(&acc[f].flags, fl);
    }
}

__global__ void __launch_bounds__(256) node_features_kernel(const NodeAcc* __restrict__ acc, const int8_t* __restrict__ kind,
                                                             int64_t N, double window, float* __restrict__ x,
                                                             int32_t* __restrict__ label, float* __restrict__ size_mb) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < N; v += stride) {
        const NodeAcc a = acc[v];
        float row[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) row[k] = 0.f;
        const bool is_file = kind[v] == 0;
        row[0] = is_file ? 1.f : 0.f;
        row[1] = kind[v] == 1 ? 1.f : 0.f;
        const float d = (float)log1p((double)a.deg);
        row[3] = d; row[4] = d;
#pragma unroll
        for (int k = 0; k < 8; ++k) row[5 + k] = (float)log1p((double)a.cnt[k]);
        const double nb = (double)a.bytes;
        row[13] = (float)(log1p(nb) / 20.0);
        const double first = __longlong_as_double(a.first), last = __longlong_as_double(a.last);
        row[14] = (float)((last - first) / window);
        row[15] = (float)(first / window);
        row[16] = (a.flags & NERRF_PATH_LOCKBIT) ? 1.f : 0.f;
        row[17] = (a.flags & NERRF_PATH_NOTE) ? 1.f : 0.f;
        row[18] = (a.flags & NERRF_PATH_TMP) ? 1.f : 0.f;
        const double wr = (double)a.cnt[1] + (double)a.cnt[5];
        row[19] = wr > 0.0 ? (float)((double)a.cnt[2] / wr) : 0.f;
        float4* out = reinterpret_cast<float4*>(x + v * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) out[q] = make_float4(row[4 * q], row[4 * q + 1], row[4 * q + 2], row[4 * q + 3]);
        if (label) label[v] = (a.flags & 0x100) ? 1 : 0;
        if (size_mb) {
            const double k3 = fmax((double)a.cnt[0] + (double)a.cnt[1] + (double)a.cnt[2], 1.0);
            size_mb[v] = is_file ? (float)(nb / k3 / 1e6) : 0.f;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Per-file event sequences for the LSTM, on the device (spec = nerrf_b200/ingest.py sequences_core; feature layout
// pipeline.file_sequences): for candidate file node f the in-edges of row f ARE its events in time order (merge mode: every
// event adds exactly one edge process -> file), perm maps a CSR position back to the input edge (= 2 * event rank), `order`
// the rank to the stored event.  One warp per candidate; the last t_max events, oldest first.
template <typename RP>
__global__ void __launch_bounds__(256) trace_sequences_kernel(const int64_t* __restrict__ cand, int n_cand, const RP* __restrict__ rowptr,
                                                               const uint32_t* __restrict__ perm, const int64_t* __restrict__ order,
                                                               const double* __restrict__ ts, const uint8_t* __restrict__ slot,
                                                               const int64_t* __restrict__ bytes, const uint8_t* __restrict__ pflags,
                                                               double t0, double span, int t_max, float* __restrict__ seq,
                                                               int32_t* __restrict__ len_out, int64_t* __restrict__ event_out) {
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (c >= n_cand) return;
    const int64_t f = cand[c];
    const int64_t e0 = (int64_t)rowptr[f], e1 = (int64_t)rowptr[f + 1];
    const int64_t deg = e1 - e0;
    const int64_t start = deg > t_max ? deg - t_max : 0;
    const int len = (int)(deg - start);
    if (lane == 0) len_out[c] = len;
    float* out = seq + (size_t)c * t_max * 16;
    if (event_out)                                                   // the stored row of each step, -1 at padded steps
        for (int k = len + lane; k < t_max; k += 32) event_out[(size_t)c * t_max + k] = -1;
    for (int k = lane; k < len; k += 32) {
        const int64_t e = e0 + start + k;
        const int64_t si = order[perm[e] >> 1];
        if (event_out) event_out[(size_t)c * t_max + k] = si;
        const double t = ts[si];
        double dt = 0.0;
        if (k > 0) { const double tp = ts[order[perm[e - 1] >> 1]]; dt = fmin(t - tp, 10.0); }
        float row[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) row[j] = 0.f;
        const int sl = slot[si];
#pragma unroll
        for (int j = 0; j < 8; ++j) row[j] = (j == sl) ? 1.f : 0.f;
        row[8] = (float)(log1p((double)clamp_rw((uint64_t)bytes[si])) / 20.0);   // the wire's uint64, stored as int64
        row[9] = (float)dt;
        row[10] = (float)((t - t0) / span);
        const int pf = pflags[si];
        row[11] = (pf & 1) ? 1.f : 0.f;
        row[12] = (pf & 4) ? 1.f : 0.f;
        float4* o = reinterpret_cast<float4*>(out + (size_t)k * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) o[q] = make_float4(row[4 * q], row[4 * q + 1], row[4 * q + 2], row[4 * q + 3]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Per-pair edge labels (spec = nerrf_b200/graph.py graph_from_events meta['edge_label']): an edge of the CSR is 1 iff one
// end is a process p, the other a file f, and p emitted an attack event (raw annotation slot 1..3: encrypt start / complete,
// ransom note) on f.  Keys p * N + f of the attack events are radix-sorted (radix_sort.cuh); every other event gets the
// sentinel N * N, which sorts last and equals no pair.  Then one thread per CSR edge finds its row by a binary search of
// rowptr and looks both orientations of (src, dst) up in the sorted keys: the attack pair is stored process-first, so at
// most one orientation can hit, and a file <-> file rename link never does.  Duplicate keys are harmless to the search, so
// no unique pass is needed.  No atomics, no host round trip.
__global__ void __launch_bounds__(256) attack_keys_kernel(const int32_t* __restrict__ node_p, const int32_t* __restrict__ node_f,
                                                          const uint8_t* __restrict__ raw_slot, int64_t n, int64_t N,
                                                          uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const uint64_t none = (uint64_t)N * (uint64_t)N;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int32_t p = node_p[i], f = node_f[i];
        const int s = raw_slot[i];
        const bool attack = s >= 1 && s <= 3 && (uint32_t)p < (uint64_t)N && (uint32_t)f < (uint64_t)N;   // ids outside [0, N) match nothing
        keys[i] = attack ? (uint64_t)p * (uint64_t)N + (uint64_t)f : none;
        vals[i] = (uint32_t)i;
    }
}

__device__ __forceinline__ bool sorted_contains(const uint64_t* __restrict__ keys, int64_t n, uint64_t k) {
    int64_t lo = 0, hi = n;                                          // lower bound
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
    }
    return lo < n && __ldg(keys + lo) == k;
}

template <typename RP>
__global__ void __launch_bounds__(256) edge_label_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col, int64_t E,
                                                         int64_t N, const uint64_t* __restrict__ keys, int64_t n,
                                                         uint8_t* __restrict__ label) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride) {
        int64_t lo = 0, hi = N;                                      // row d = the last row with rowptr[d] <= i
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)__ldg(rowptr + mid) <= i) lo = mid; else hi = mid;
        }
        const uint64_t d = (uint64_t)lo, s = (uint32_t)col[i];
        bool hit = false;
        if (s < (uint64_t)N) hit = sorted_contains(keys, n, s * N + d) || sorted_contains(keys, n, d * N + s);
        label[i] = hit ? 1 : 0;
    }
}

static int pair_key_bits(int64_t N) {                                // bits of N * N, the largest key (the sentinel)
    const uint64_t top = (uint64_t)N * (uint64_t)N;
    int b = 1;
    while (b < 64 && (top >> b)) ++b;
    return b;
}

struct CsrWs {
    size_t keys_a, keys_b, vals_a, vals_b, bad, temp, total, temp_bytes;
};

static inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

static int key_bits(int64_t N) {
    int b = 0;
    while (((int64_t)1 << b) < N) ++b;
    return 32 + (b < 1 ? 1 : b);
}

static int csr_layout(int64_t E, int64_t N, CsrWs* L) {
    size_t temp = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int64_t)(E > 0 ? E : 1), 0, key_bits(N));
    if (e != cudaSuccess) {
        set_error("cub::DeviceRadixSort size query failed: %s", cudaGetErrorString(e));
        cudaGetLastError();
        return NERRF_ERR_CUDA;
    }
    size_t o = 0;
    L->keys_a = o; o += up256((size_t)E * 8);
    L->keys_b = o; o += up256((size_t)E * 8);
    L->vals_a = o; o += up256((size_t)E * 4);
    L->vals_b = o; o += up256((size_t)E * 4);
    L->bad = o;    o += 256;
    const size_t own = rs_scratch_bytes(E > 0 ? E : 1);
    L->temp = o;   o += up256(temp > own ? temp : own);
    L->temp_bytes = temp;
    L->total = o;
    return NERRF_OK;
}

}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_graph_csr_workspace_bytes(int64_t n_edges, int64_t n_nodes, int64_t* bytes) {
    NERRF_REQUIRE(bytes != nullptr, "null bytes pointer");
    NERRF_REQUIRE(n_edges >= 0 && n_edges < ((int64_t)1 << 32), "n_edges=%lld out of range [0, 2^32)", (long long)n_edges);
    NERRF_REQUIRE(n_nodes >= 1 && n_nodes < ((int64_t)1 << 31), "n_nodes=%lld out of range [1, 2^31)", (long long)n_nodes);
    CsrWs L;
    const int rc = csr_layout(n_edges, n_nodes, &L);
    if (rc != NERRF_OK) return rc;
    *bytes = (int64_t)L.total;
    return NERRF_OK;
}

extern "C" int nerrf_graph_build_csr(const int32_t* src, const int32_t* dst, const float* t, const float* conf,
                                     int64_t n_edges, int64_t n_nodes, float t_ref, float tau, void* rowptr_out,
                                     int rowptr_is64, int32_t* col_out, float* ew_out, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
    return nerrf_graph_build_csr_ex(src, dst, t, conf, n_edges, n_nodes, t_ref, tau, rowptr_out, rowptr_is64, col_out, ew_out,
                                    nullptr, workspace, workspace_bytes, stream);
}

extern "C" int nerrf_graph_build_csr_ex(const int32_t* src, const int32_t* dst, const float* t, const float* conf,
                                        int64_t n_edges, int64_t n_nodes, float t_ref, float tau, void* rowptr_out,
                                        int rowptr_is64, int32_t* col_out, float* ew_out, uint32_t* perm_out, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
    NERRF_REQUIRE(n_edges >= 0 && n_edges < ((int64_t)1 << 32), "n_edges=%lld out of range [0, 2^32)", (long long)n_edges);
    NERRF_REQUIRE(n_nodes >= 1 && n_nodes < ((int64_t)1 << 31), "n_nodes=%lld out of range [1, 2^31)", (long long)n_nodes);
    NERRF_REQUIRE(rowptr_out != nullptr, "null rowptr_out");
    NERRF_REQUIRE(rowptr_is64 || n_edges < ((int64_t)1 << 31), "n_edges >= 2^31 needs a 64-bit rowptr");
    NERRF_REQUIRE(tau > 0.f, "tau must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = sm_count() * 8;
    if (n_edges == 0) {
        if (rowptr_is64) csr_empty_kernel<int64_t><<<grid, 256, 0, st>>>((int64_t*)rowptr_out, n_nodes);
        else csr_empty_kernel<int32_t><<<grid, 256, 0, st>>>((int32_t*)rowptr_out, n_nodes);
        return launch_status("csr_empty_kernel");
    }
    NERRF_REQUIRE(src && dst && t && conf && col_out && ew_out, "null edge array");
    CsrWs L;
    int rc = csr_layout(n_edges, n_nodes, &L);
    if (rc != NERRF_OK) return rc;
    NERRF_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)L.total,
                  "workspace too small: %lld < %lld bytes (nerrf_graph_csr_workspace_bytes)", (long long)workspace_bytes,
                  (long long)L.total);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    char* ws = (char*)workspace;
    uint64_t* ka = (uint64_t*)(ws + L.keys_a); uint64_t* kb = (uint64_t*)(ws + L.keys_b);
    uint32_t* va = (uint32_t*)(ws + L.vals_a); uint32_t* vb = (uint32_t*)(ws + L.vals_b);
    int* bad = (int*)(ws + L.bad);
    NERRF_CHECK_CUDA(cudaMemsetAsync(bad, 0, 8, st));
    csr_keys_kernel<<<grid, 256, 0, st>>>(src, dst, t, n_edges, n_nodes, ka, va, bad);
    rc = launch_status("csr_keys_kernel");
    if (rc != NERRF_OK) return rc;
    // the sort: our own stable LSD radix sort (radix_sort.cuh); cub::DeviceRadixSort is kept selectable for comparison
    // (NERRF_GRAPH_SORT=cub) and for edge lists of 2^31 pairs and more (our scatter offsets are 32-bit)
    static const bool want_cub = [] { const char* e = getenv("NERRF_GRAPH_SORT"); return e && e[0] == 'c'; }();
    const uint64_t* ks; const uint32_t* vs;
    if (want_cub || n_edges >= ((int64_t)1 << 31)) {
        cub::DoubleBuffer<uint64_t> k(ka, kb);
        cub::DoubleBuffer<uint32_t> v(va, vb);
        size_t temp = L.temp_bytes;
        NERRF_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.temp, temp, k, v, n_edges, 0, key_bits(n_nodes), st));
        ks = k.Current(); vs = v.Current();
    } else {
        // an edge list that already is in time order (an event stream is) only needs the stable sort by destination: the
        // low 32 key bits (the time) are skipped -- 3 passes instead of 7 at 2^20 nodes.  `bad[1]` was set by csr_keys_kernel
        // if any edge is older than its predecessor.
        int h_unsorted = 1;
        NERRF_CHECK_CUDA(cudaMemcpyAsync(&h_unsorted, bad + 1, 4, cudaMemcpyDeviceToHost, st));
        NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
        const int which = radix_sort_pairs(ka, kb, va, vb, n_edges, h_unsorted ? 0 : 32, key_bits(n_nodes), ws + L.temp, st);
        ks = which ? kb : ka; vs = which ? vb : va;
        rc = launch_status("radix sort");
        if (rc != NERRF_OK) return rc;
    }
    if (rowptr_is64)
        csr_finish_kernel<int64_t><<<grid, 256, 0, st>>>(ks, vs, src, t, conf, n_edges, n_nodes, t_ref, tau,
                                                         (int64_t*)rowptr_out, col_out, ew_out, perm_out);
    else
        csr_finish_kernel<int32_t><<<grid, 256, 0, st>>>(ks, vs, src, t, conf, n_edges, n_nodes, t_ref, tau,
                                                         (int32_t*)rowptr_out, col_out, ew_out, perm_out);
    rc = launch_status("csr_finish_kernel");
    if (rc != NERRF_OK) return rc;
    // the vertex-id check is the one reason this call waits for the stream: out-of-range ids were clamped to row 0
    // on the device (so nothing was written out of bounds) and are reported here as NERRF_ERR_INVALID
    int h_bad = 0;
    NERRF_CHECK_CUDA(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    NERRF_REQUIRE(h_bad == 0, "edge list holds a vertex id outside [0, n_nodes)");
    return NERRF_OK;
}

extern "C" int nerrf_graph_node_features_workspace_bytes(int64_t n_nodes, int64_t* bytes) {
    NERRF_REQUIRE(bytes != nullptr && n_nodes >= 1, "bad arguments");
    *bytes = (int64_t)up256((size_t)n_nodes * sizeof(NodeAcc)) + 256;
    return NERRF_OK;
}

extern "C" int nerrf_graph_node_features(const int32_t* node_p, const int32_t* node_f, const int32_t* node_g, const double* t,
                                         const uint8_t* event_slot, const uint64_t* bytes, const uint8_t* path_flags,
                                         int64_t n_events, const int8_t* node_kind, int64_t n_nodes, double window, float* x_out,
                                         int32_t* label_out, float* size_mb_out, void* workspace, int64_t workspace_bytes,
                                         void* stream) {
    NERRF_REQUIRE(n_events >= 0 && n_nodes >= 1 && n_nodes < ((int64_t)1 << 31), "bad sizes");
    NERRF_REQUIRE((n_events == 0 || (node_p && node_f && t && event_slot && bytes && path_flags)) && node_kind && x_out,
                  "null pointer");
    NERRF_REQUIRE(window > 0.0, "window must be positive");
    int64_t need = 0;
    nerrf_graph_node_features_workspace_bytes(n_nodes, &need);
    NERRF_REQUIRE(workspace != nullptr && workspace_bytes >= need, "workspace too small: %lld < %lld bytes",
                  (long long)workspace_bytes, (long long)need);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0 && ((uintptr_t)x_out & 15) == 0, "workspace / x_out misaligned");
    static_assert(sizeof(NodeAcc) == 64, "NodeAcc layout");
    cudaStream_t st = (cudaStream_t)stream;
    NodeAcc* acc = (NodeAcc*)workspace;
    int* bad = (int*)((char*)workspace + up256((size_t)n_nodes * sizeof(NodeAcc)));
    const int grid = sm_count() * 8;
    NERRF_CHECK_CUDA(cudaMemsetAsync(bad, 0, 4, st));
    node_acc_init_kernel<<<grid, 256, 0, st>>>(acc, n_nodes);
    if (n_events) node_acc_events_kernel<<<grid, 256, 0, st>>>(node_p, node_f, node_g, t, event_slot, bytes, path_flags, n_events,
                                                                n_nodes, acc, bad);
    node_features_kernel<<<grid, 256, 0, st>>>(acc, node_kind, n_nodes, window, x_out, label_out, size_mb_out);
    const int rc = launch_status("node feature kernels");
    if (rc != NERRF_OK) return rc;
    int h_bad = 0;
    NERRF_CHECK_CUDA(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    NERRF_REQUIRE(h_bad == 0, "event columns hold a node id outside [0, n_nodes), a negative time or an event slot > 7");
    return NERRF_OK;
}

static size_t edge_label_layout(int64_t n, size_t* keys_b, size_t* vals_a, size_t* vals_b, size_t* scratch) {
    size_t o = up256((size_t)n * 8);
    *keys_b = o;  o += up256((size_t)n * 8);
    *vals_a = o;  o += up256((size_t)n * 4);
    *vals_b = o;  o += up256((size_t)n * 4);
    *scratch = o; o += up256(rs_scratch_bytes(n > 0 ? n : 1));
    return o;
}

extern "C" int nerrf_trace_edge_labels_workspace_bytes(int64_t n_events, int64_t* bytes) {
    NERRF_REQUIRE(bytes != nullptr, "null bytes pointer");
    NERRF_REQUIRE(n_events >= 0 && n_events < ((int64_t)1 << 31), "n_events=%lld out of range [0, 2^31)", (long long)n_events);
    size_t kb, va, vb, sc;
    *bytes = (int64_t)edge_label_layout(n_events, &kb, &va, &vb, &sc);
    return NERRF_OK;
}

extern "C" int nerrf_trace_edge_labels(const int32_t* node_p, const int32_t* node_f, const uint8_t* raw_slot, int64_t n_events,
                                       const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_edges, int64_t n_nodes,
                                       uint8_t* label_out, void* workspace, int64_t workspace_bytes, void* stream) {
    NERRF_REQUIRE(n_events >= 0 && n_events < ((int64_t)1 << 31), "n_events=%lld out of range [0, 2^31)", (long long)n_events);
    NERRF_REQUIRE(n_edges >= 0 && n_nodes >= 1 && n_nodes < ((int64_t)1 << 31), "bad sizes");
    if (n_edges == 0) return NERRF_OK;
    NERRF_REQUIRE(rowptr && col && label_out, "null CSR / label pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_events == 0) {                                             // no event, no attack pair
        NERRF_CHECK_CUDA(cudaMemsetAsync(label_out, 0, (size_t)n_edges, st));
        return NERRF_OK;
    }
    NERRF_REQUIRE(node_p && node_f && raw_slot, "null event column");
    size_t kb, va, vb, sc;
    const size_t need = edge_label_layout(n_events, &kb, &va, &vb, &sc);
    NERRF_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)need,
                  "workspace too small: %lld < %lld bytes (nerrf_trace_edge_labels_workspace_bytes)", (long long)workspace_bytes,
                  (long long)need);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    char* ws = (char*)workspace;
    uint64_t* ka = (uint64_t*)ws; uint64_t* kbp = (uint64_t*)(ws + kb);
    uint32_t* vap = (uint32_t*)(ws + va); uint32_t* vbp = (uint32_t*)(ws + vb);
    const int grid = sm_count() * 8;
    attack_keys_kernel<<<grid, 256, 0, st>>>(node_p, node_f, raw_slot, n_events, n_nodes, ka, vap);
    int rc = launch_status("attack_keys_kernel");
    if (rc != NERRF_OK) return rc;
    const int which = radix_sort_pairs(ka, kbp, vap, vbp, n_events, 0, pair_key_bits(n_nodes), ws + sc, st);
    rc = launch_status("radix sort");
    if (rc != NERRF_OK) return rc;
    const uint64_t* keys = which ? kbp : ka;
    if (rowptr_is64)
        edge_label_kernel<int64_t><<<grid, 256, 0, st>>>((const int64_t*)rowptr, col, n_edges, n_nodes, keys, n_events, label_out);
    else
        edge_label_kernel<int32_t><<<grid, 256, 0, st>>>((const int32_t*)rowptr, col, n_edges, n_nodes, keys, n_events, label_out);
    return launch_status("edge_label_kernel");
}

extern "C" int nerrf_trace_sequences(const int64_t* cand_nodes, int n_cand, const void* rowptr, int rowptr_is64, const uint32_t* perm,
                                     const int64_t* order, const double* ts, const uint8_t* event_slot, const int64_t* bytes,
                                     const uint8_t* path_flags, double t0, double span, int t_max, float* seq_out,
                                     int32_t* len_out, void* stream) {
    return nerrf_trace_sequences_ex(cand_nodes, n_cand, rowptr, rowptr_is64, perm, order, ts, event_slot, bytes, path_flags, t0, span,
                                    t_max, seq_out, len_out, nullptr, stream);
}

extern "C" int nerrf_trace_sequences_ex(const int64_t* cand_nodes, int n_cand, const void* rowptr, int rowptr_is64,
                                        const uint32_t* perm, const int64_t* order, const double* ts, const uint8_t* event_slot,
                                        const int64_t* bytes, const uint8_t* path_flags, double t0, double span, int t_max,
                                        float* seq_out, int32_t* len_out, int64_t* event_out, void* stream) {
    NERRF_REQUIRE(n_cand >= 0 && t_max >= 1, "bad sizes");
    if (n_cand == 0) return NERRF_OK;
    NERRF_REQUIRE(cand_nodes && rowptr && perm && order && ts && event_slot && bytes && path_flags && seq_out && len_out, "null pointer");
    NERRF_REQUIRE(span > 0.0 && ((uintptr_t)seq_out & 15) == 0, "span must be positive, seq_out 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    NERRF_CHECK_CUDA(cudaMemsetAsync(seq_out, 0, (size_t)n_cand * t_max * 16 * sizeof(float), st));
    const unsigned grid = (unsigned)((n_cand + 7) / 8);
    if (rowptr_is64)
        trace_sequences_kernel<int64_t><<<grid, 256, 0, st>>>(cand_nodes, n_cand, (const int64_t*)rowptr, perm, order, ts, event_slot, bytes,
                                                              path_flags, t0, span, t_max, seq_out, len_out, event_out);
    else
        trace_sequences_kernel<int32_t><<<grid, 256, 0, st>>>(cand_nodes, n_cand, (const int32_t*)rowptr, perm, order, ts, event_slot, bytes,
                                                              path_flags, t0, span, t_max, seq_out, len_out, event_out);
    return launch_status("trace_sequences_kernel");
}
