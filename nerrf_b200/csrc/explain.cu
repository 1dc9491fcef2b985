// Per-node explanations of GraphSAGE-T scores (DESIGN.md 1.1.1): receptive-field extraction and segmented top-k.
//
//   nerrf_explain_subgraph_count / _fill   the L-hop in-neighbourhood of each target as one block-diagonal batched CSR
//   nerrf_explain_topk                     the k edges of largest |ew * d_ew| per target, with their events
//
// Extraction, one CTA per target (grid-strided over the targets, one workspace slot per CTA):
//   level-synchronous BFS over in-edges.  The frontier of distance d (d = 0 .. L-1) contributes every in-edge of its
//   nodes (so each kept row is complete and S_u, m_u are the full graph's) and discovers distance d+1; distance-L nodes
//   contribute their features only.  The visited set is an open-addressing hash table keyed by node id (the pattern of
//   intern_device.cu); the first thread to claim a node appends it.  Append order depends on atomics, the SET does not:
//   the node list is then bitonic-sorted by global id, so local ids, rows and edges are a function of the graph alone.
//   Rows keep their original edge order, so the batched graph's row sums and gathers see the same operands in the same
//   order as the full graph's.  A target whose kept rows hold more than max_edges edges is reported as over budget
//   (counts -1) and is not filled.
//   _count returns per target (nodes, edges); the caller scans them into offsets and calls _fill, which repeats the
//   (deterministic) BFS and writes its block.
//
// Top-k, one CTA per target segment: k rounds of a block arg-max of (|a|, -position) below the previous pick, so ties go
// to the lower CSR position and the result has no order that depends on scheduling.
//
// Sequence steps (DESIGN.md 1.2.1), nerrf_lstm_explain_steps, one warp per sequence: a_t = sum_d x[t,d] * dseq[t,d] over
// the valid steps, as __fmul_rn products summed left to right with __fadd_rn (so a float32 restatement over the same
// dseq reproduces it bit for bit), then k rounds of a warp arg-max of (|a_t|, -t) below the previous pick -- the same
// rule (explain_rank.cuh) as the edge top-k.
#include "common.cuh"
#include "explain_rank.cuh"

namespace nerrf {
namespace {

constexpr int XT = 256;               // threads per CTA

struct Slot {                         // one CTA's scratch
    int32_t* keys;                    // [cap] node id or -1
    int32_t* dist;                    // [cap] BFS distance of the node in the same slot
    int32_t* loc;                     // [cap] local id (position in the sorted node list)
    int32_t* nodes;                   // [lcap] discovered nodes, then sorted
    int32_t* pre;                     // [lcap] exclusive prefix of the kept row lengths
};

__host__ __device__ inline int64_t pow2_at_least(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

__host__ __device__ inline void slot_sizes(int64_t max_edges, int64_t* cap, int64_t* lcap) {
    *lcap = pow2_at_least(max_edges + 1);                 // nodes <= 1 + kept edges
    *cap = 2 * *lcap;                                     // load factor <= 1/2
}

__host__ __device__ inline size_t slot_bytes(int64_t max_edges) {
    int64_t cap, lcap;
    slot_sizes(max_edges, &cap, &lcap);
    return (size_t)(3 * cap + 2 * lcap) * 4;
}

__device__ inline Slot slot_at(unsigned char* ws, int64_t max_edges, int i) {
    int64_t cap, lcap;
    slot_sizes(max_edges, &cap, &lcap);
    int32_t* b = reinterpret_cast<int32_t*>(ws + slot_bytes(max_edges) * (size_t)i);
    return Slot{b, b + cap, b + 2 * cap, b + 3 * cap, b + 3 * cap + lcap};
}

__device__ inline uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

// -> slot of `node` (inserted with distance d when absent); *fresh = 1 iff this call inserted it
__device__ inline int64_t hash_claim(const Slot& s, int64_t cap, int32_t node, int32_t d, bool* fresh) {
    int64_t h = mix((uint32_t)node) & (cap - 1);
    while (true) {
        const int32_t k = atomicCAS(s.keys + h, -1, node);
        if (k == -1) { s.dist[h] = d; *fresh = true; return h; }
        if (k == node) { *fresh = false; return h; }
        h = (h + 1) & (cap - 1);
    }
}

__device__ inline int64_t hash_find(const Slot& s, int64_t cap, int32_t node) {
    int64_t h = mix((uint32_t)node) & (cap - 1);
    while (s.keys[h] != node) h = (h + 1) & (cap - 1);
    return h;
}

__device__ inline int64_t block_sum64(int64_t v, int64_t* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    int64_t t = 0;
    for (int i = 0; i < XT / 32; ++i) t += red[i];
    return t;
}

// The BFS of one target.  -> node count (the node list unsorted in s.nodes), *edges = kept edges; -1 when over budget.
template <typename RP>
__device__ int bfs(const RP* rowptr, const int32_t* col, int32_t target, int hops, int64_t max_edges, const Slot& s,
                   int64_t cap, int64_t* edges_out, int* s_count, int64_t* red) {
    for (int64_t i = threadIdx.x; i < cap; i += XT) s.keys[i] = -1;
    __syncthreads();
    if (threadIdx.x == 0) {
        bool f;
        hash_claim(s, cap, target, 0, &f);
        s.nodes[0] = target;
        *s_count = 1;
    }
    __syncthreads();
    int f0 = 0, f1 = 1;
    int64_t edges = 0;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int d = 0; d < hops; ++d) {
        int64_t deg = 0;
        for (int i = f0 + threadIdx.x; i < f1; i += XT) {
            const int32_t u = s.nodes[i];
            deg += (int64_t)rowptr[u + 1] - (int64_t)rowptr[u];
        }
        const int64_t total = block_sum64(deg, red);
        if (edges + total > max_edges) return -1;        // uniform across the block
        edges += total;
        for (int i = f0 + w; i < f1; i += XT / 32) {
            const int32_t u = s.nodes[i];
            const int64_t e0 = rowptr[u], e1 = rowptr[u + 1];
            for (int64_t e = e0 + lane; e < e1; e += 32) {
                bool fresh;
                const int32_t v = __ldg(col + e);
                hash_claim(s, cap, v, d + 1, &fresh);
                if (fresh) s.nodes[atomicAdd(s_count, 1)] = v;
            }
        }
        __syncthreads();
        f0 = f1;
        f1 = *s_count;
        __syncthreads();
    }
    *edges_out = edges;
    return f1;
}

// ascending bitonic sort of s.nodes[0, n) (padded to a power of two with INT32_MAX)
__device__ void sort_nodes(int32_t* a, int n) {
    const int p = (int)pow2_at_least(n);
    for (int i = n + threadIdx.x; i < p; i += XT) a[i] = 0x7fffffff;
    __syncthreads();
    for (int k = 2; k <= p; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < p; i += XT) {
                const int l = i ^ j;
                if (l > i) {
                    const int32_t x = a[i], y = a[l];
                    if (((i & k) == 0) ? (x > y) : (x < y)) { a[i] = y; a[l] = x; }
                }
            }
            __syncthreads();
        }
}

template <typename RP>
__global__ void __launch_bounds__(XT) subgraph_count_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                            const int32_t* __restrict__ targets, int64_t n_targets, int hops,
                                                            int64_t max_edges, int64_t* __restrict__ counts, unsigned char* ws) {
    __shared__ int s_count;
    __shared__ int64_t red[XT / 32];
    int64_t cap, lcap;
    slot_sizes(max_edges, &cap, &lcap);
    const Slot s = slot_at(ws, max_edges, blockIdx.x);
    for (int64_t t = blockIdx.x; t < n_targets; t += gridDim.x) {
        int64_t edges = 0;
        const int n = bfs(rowptr, col, targets[t], hops, max_edges, s, cap, &edges, &s_count, red);
        if (threadIdx.x == 0) {
            counts[2 * t] = n < 0 ? -1 : n;
            counts[2 * t + 1] = n < 0 ? -1 : edges;
        }
        __syncthreads();
    }
}

template <typename RP>
__global__ void __launch_bounds__(XT) subgraph_fill_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                           const float* __restrict__ ew, const float* __restrict__ x, int F_in,
                                                           const int32_t* __restrict__ targets, int64_t n_targets, int hops,
                                                           int64_t max_edges, const int64_t* __restrict__ node_off,
                                                           const int64_t* __restrict__ edge_off, int64_t* __restrict__ out_rowptr,
                                                           int32_t* __restrict__ out_col, float* __restrict__ out_ew,
                                                           int64_t* __restrict__ out_epos, int32_t* __restrict__ out_node,
                                                           float* __restrict__ out_x, int32_t* __restrict__ out_target,
                                                           unsigned char* ws) {
    __shared__ int s_count;
    __shared__ int64_t red[XT / 32];
    __shared__ int32_t s_carry;
    int64_t cap, lcap;
    slot_sizes(max_edges, &cap, &lcap);
    const Slot s = slot_at(ws, max_edges, blockIdx.x);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < n_targets; t += gridDim.x) {
        int64_t edges = 0;
        const int n = bfs(rowptr, col, targets[t], hops, max_edges, s, cap, &edges, &s_count, red);
        if (n < 0) continue;                                          // over budget: the caller does not fill it (uniform)
        sort_nodes(s.nodes, n);
        for (int i = threadIdx.x; i < n; i += XT) s.loc[hash_find(s, cap, s.nodes[i])] = i;
        // exclusive prefix of the kept row lengths, XT rows at a time (lengths < 2^31: they sum to <= max_edges)
        if (threadIdx.x == 0) s_carry = 0;
        __syncthreads();
        for (int base = 0; base < n; base += XT) {
            const int i = base + threadIdx.x;
            int32_t len = 0;
            if (i < n) {
                const int32_t u = s.nodes[i];
                if (s.dist[hash_find(s, cap, u)] < hops) len = (int32_t)((int64_t)rowptr[u + 1] - (int64_t)rowptr[u]);
            }
            int32_t v = len;                                           // inclusive warp scan, then across warps
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t y = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += y;
            }
            __shared__ int32_t wsum[XT / 32];
            if (lane == 31) wsum[w] = v;
            __syncthreads();
            int32_t before = s_carry;
            for (int q = 0; q < w; ++q) before += wsum[q];
            if (i < n) s.pre[i] = before + v - len;
            __syncthreads();
            if (threadIdx.x == XT - 1) s_carry = before + v;
            __syncthreads();
        }
        const int64_t no = node_off[t], eo = edge_off[t];
        for (int i = threadIdx.x; i < n; i += XT) {
            out_rowptr[no + i] = eo + s.pre[i];
            out_node[no + i] = s.nodes[i];
        }
        if (threadIdx.x == 0) {
            out_rowptr[no + n] = eo + edges;                           // = the next block's first entry (same value)
            out_target[t] = (int32_t)(no + s.loc[hash_find(s, cap, targets[t])]);
        }
        for (int64_t q = threadIdx.x; q < (int64_t)n * (F_in / 4); q += XT) {
            const int i = (int)(q / (F_in / 4)), c = (int)(q % (F_in / 4));
            reinterpret_cast<float4*>(out_x + (no + i) * F_in)[c] = ldg4(x + (int64_t)s.nodes[i] * F_in + 4 * c);
        }
        for (int i = w; i < n; i += XT / 32) {                         // one warp per kept row, edges in original order
            const int32_t u = s.nodes[i];
            if (s.dist[hash_find(s, cap, u)] >= hops) continue;
            const int64_t e0 = rowptr[u], e1 = rowptr[u + 1];
            const int64_t o = eo + s.pre[i] - e0;
            for (int64_t e = e0 + lane; e < e1; e += 32) {
                out_col[o + e] = (int32_t)(no + s.loc[hash_find(s, cap, __ldg(col + e))]);
                out_ew[o + e] = __ldg(ew + e);
                out_epos[o + e] = e;
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(XT) topk_kernel(const int64_t* __restrict__ seg, const float* __restrict__ ew,
                                                  const float* __restrict__ d_ew, const int64_t* __restrict__ epos,
                                                  const int64_t* __restrict__ edge_event, int k, int64_t* __restrict__ out_edge,
                                                  float* __restrict__ out_attr, int64_t* __restrict__ out_pos,
                                                  int64_t* __restrict__ out_event) {
    __shared__ float rv[XT / 32];
    __shared__ int64_t ri[XT / 32];
    __shared__ float s_pv;
    __shared__ int64_t s_pi;
    const int64_t t = blockIdx.x;
    const int64_t e0 = seg[t], e1 = seg[t + 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float pv = __int_as_float(0x7f800000);       // +inf: every key is below the "previous pick" of round 0
    int64_t pi = -1;
    for (int r = 0; r < k; ++r) {
        float bv = -1.f;
        int64_t bi = -1;
        for (int64_t e = e0 + threadIdx.x; e < e1; e += XT) {
            const float v = rank_key(ew[e] * d_ew[e]);               // NaN: below every number, above "none"
            const int64_t i = e - e0;
            if (better(pv, pi, v, i) && (bi < 0 || better(v, i, bv, bi))) { bv = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || better(ov, oi, bv, bi))) { bv = ov; bi = oi; }
        }
        if (lane == 0) { rv[w] = bv; ri[w] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float v = -1.f;
            int64_t i = -1;
            for (int q = 0; q < XT / 32; ++q)
                if (ri[q] >= 0 && (i < 0 || better(rv[q], ri[q], v, i))) { v = rv[q]; i = ri[q]; }
            const int64_t o = t * k + r;
            out_edge[o] = i < 0 ? -1 : e0 + i;
            out_attr[o] = i < 0 ? 0.f : ew[e0 + i] * d_ew[e0 + i];
            const int64_t p = i < 0 ? -1 : (epos ? epos[e0 + i] : e0 + i);
            out_pos[o] = p;
            if (out_event) out_event[o] = (p < 0 || !edge_event) ? -1 : edge_event[p];
            s_pv = v; s_pi = i;
        }
        __syncthreads();
        pv = s_pv; pi = s_pi;
        __syncthreads();
        if (pi < 0) {                                                 // segment exhausted: the remaining picks are empty
            for (int q = r + 1 + threadIdx.x; q < k; q += XT) {
                const int64_t o = t * k + q;
                out_edge[o] = -1; out_attr[o] = 0.f; out_pos[o] = -1;
                if (out_event) out_event[o] = -1;
            }
            return;
        }
    }
}

constexpr int SW = 8;                 // sequences (one warp each) per CTA of the step kernel

// a_t of one step: the D products x[d] * g[d], each rounded, summed left to right (fixed order, no contraction)
__device__ __forceinline__ float step_attr(const float* __restrict__ x, const float* __restrict__ g, int D) {
    float s = __fmul_rn(__ldg(x), __ldg(g));
    for (int d = 1; d < D; ++d) s = __fadd_rn(s, __fmul_rn(__ldg(x + d), __ldg(g + d)));
    return s;
}

// argmax_d |x[d] * g[d]|, ties to the lower d; -1 when every term is 0 (a NaN term is never dominant)
__device__ __forceinline__ int dominant_feature(const float* __restrict__ x, const float* __restrict__ g, int D) {
    int best = -1;
    float bm = 0.f;
    for (int d = 0; d < D; ++d) {
        const float m = fabsf(__fmul_rn(__ldg(x + d), __ldg(g + d)));
        if (m > bm) { bm = m; best = d; }
    }
    return best;
}

__global__ void __launch_bounds__(32 * SW) explain_steps_kernel(const float* __restrict__ seq, const float* __restrict__ dseq,
                                                                const int32_t* __restrict__ len, int64_t B, int T, int D,
                                                                const int64_t* __restrict__ step_event, int k,
                                                                int32_t* __restrict__ out_step, float* __restrict__ out_attr,
                                                                int32_t* __restrict__ out_feature, int64_t* __restrict__ out_event) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * SW + (threadIdx.x >> 5);
    if (b >= B) return;                                               // warp-uniform
    const int lb = len[b];
    const int L = lb < 0 ? 0 : (lb > T ? T : lb);
    const float* X = seq + b * T * D;
    const float* G = dseq + b * T * D;
    float pv = __int_as_float(0x7f800000);                            // +inf: every key is below the "previous pick" of round 0
    int pi = -1;
    for (int r = 0; r < k; ++r) {
        float bv = -1.f;
        int bi = -1;
        for (int t = lane; t < L; t += 32) {
            const float v = rank_key(step_attr(X + (int64_t)t * D, G + (int64_t)t * D, D));
            if (better(pv, pi, v, t) && (bi < 0 || better(v, t, bv, bi))) { bv = v; bi = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {                            // a total order: every lane ends on the same pick
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || better(ov, oi, bv, bi))) { bv = ov; bi = oi; }
        }
        if (bi < 0) {                                                 // valid steps exhausted: the remaining picks are empty
            for (int q = r + lane; q < k; q += 32) {
                const int64_t o = b * k + q;
                out_step[o] = -1; out_attr[o] = 0.f; out_feature[o] = -1; out_event[o] = -1;
            }
            return;
        }
        if (lane == 0) {
            const int64_t o = b * k + r;
            const float* x = X + (int64_t)bi * D;
            const float* g = G + (int64_t)bi * D;
            out_step[o] = bi;
            out_attr[o] = step_attr(x, g, D);
            out_feature[o] = dominant_feature(x, g, D);
            out_event[o] = step_event ? step_event[b * T + bi] : -1;
        }
        pv = bv; pi = bi;
    }
}

int grid_slots(int64_t n_targets) {
    const int64_t g = 2 * (int64_t)sm_count();
    return (int)(n_targets < g ? (n_targets < 1 ? 1 : n_targets) : g);
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_explain_subgraph_workspace_bytes(int64_t n_targets, int64_t max_edges, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_targets >= 0, "bad argument");
    NERRF_REQUIRE(max_edges >= 0 && max_edges < (1ll << 28), "max_edges must lie in [0, 2^28) (got %lld)", (long long)max_edges);
    *bytes = slot_bytes(max_edges) * (size_t)grid_slots(n_targets);
    return NERRF_OK;
}

static int subgraph_check(const void* rowptr, const int32_t* col, int64_t n_nodes, const int32_t* targets, int64_t n_targets,
                          int hops, int64_t max_edges, void* workspace, size_t workspace_bytes) {
    NERRF_REQUIRE(n_nodes >= 0 && n_nodes < (1ll << 31), "node count must lie in [0, 2^31)");
    NERRF_REQUIRE(n_targets >= 0 && (n_targets == 0 || (rowptr && targets && workspace)), "null pointer");
    NERRF_REQUIRE(hops >= 1 && hops <= 16, "hops must lie in 1..16 (got %d)", hops);
    size_t need = 0;
    const int rc = nerrf_explain_subgraph_workspace_bytes(n_targets, max_edges, &need);
    if (rc) return rc;
    if (workspace_bytes < need) {
        set_error("explain workspace too small: need %zu bytes", need);
        return NERRF_ERR_WORKSPACE;
    }
    (void)col;
    return NERRF_OK;
}

extern "C" int nerrf_explain_subgraph_count(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes,
                                            const int32_t* targets, int64_t n_targets, int hops, int64_t max_edges,
                                            int64_t* counts, void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    const int rc = subgraph_check(rowptr, col, n_nodes, targets, n_targets, hops, max_edges, workspace, workspace_bytes);
    if (rc) return rc;
    if (n_targets == 0) return NERRF_OK;
    NERRF_REQUIRE(counts, "null counts");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_slots(n_targets);
    unsigned char* ws = (unsigned char*)workspace;
    if (rowptr_is64)
        subgraph_count_kernel<int64_t><<<grid, XT, 0, st>>>((const int64_t*)rowptr, col, targets, n_targets, hops, max_edges, counts, ws);
    else
        subgraph_count_kernel<int32_t><<<grid, XT, 0, st>>>((const int32_t*)rowptr, col, targets, n_targets, hops, max_edges, counts, ws);
    return launch_status("explain subgraph count");
}

extern "C" int nerrf_explain_subgraph_fill(const void* rowptr, int rowptr_is64, const int32_t* col, const float* ew,
                                           const float* x, int F_in, int64_t n_nodes, const int32_t* targets, int64_t n_targets,
                                           int hops, int64_t max_edges, const int64_t* node_off, const int64_t* edge_off,
                                           int64_t* out_rowptr, int32_t* out_col, float* out_ew, int64_t* out_epos,
                                           int32_t* out_node, float* out_x, int32_t* out_target, void* workspace,
                                           size_t workspace_bytes, nerrf_stream_t stream) {
    const int rc = subgraph_check(rowptr, col, n_nodes, targets, n_targets, hops, max_edges, workspace, workspace_bytes);
    if (rc) return rc;
    if (n_targets == 0) return NERRF_OK;
    NERRF_REQUIRE(F_in > 0 && F_in % 4 == 0, "F_in must be a positive multiple of 4 (got %d)", F_in);
    NERRF_REQUIRE(x && node_off && edge_off && out_rowptr && out_node && out_x && out_target, "null pointer");
    NERRF_REQUIRE((((uintptr_t)x | (uintptr_t)out_x) & 15) == 0, "x and out_x must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_slots(n_targets);
    unsigned char* ws = (unsigned char*)workspace;
    if (rowptr_is64)
        subgraph_fill_kernel<int64_t><<<grid, XT, 0, st>>>((const int64_t*)rowptr, col, ew, x, F_in, targets, n_targets, hops, max_edges,
                                                           node_off, edge_off, out_rowptr, out_col, out_ew, out_epos, out_node, out_x,
                                                           out_target, ws);
    else
        subgraph_fill_kernel<int32_t><<<grid, XT, 0, st>>>((const int32_t*)rowptr, col, ew, x, F_in, targets, n_targets, hops, max_edges,
                                                           node_off, edge_off, out_rowptr, out_col, out_ew, out_epos, out_node, out_x,
                                                           out_target, ws);
    return launch_status("explain subgraph fill");
}

extern "C" int nerrf_explain_topk(const int64_t* seg, int64_t n_seg, const float* ew, const float* d_ew, const int64_t* epos,
                                  const int64_t* edge_event, int k, int64_t* out_edge, float* out_attr, int64_t* out_pos,
                                  int64_t* out_event, nerrf_stream_t stream) {
    NERRF_REQUIRE(n_seg >= 0 && n_seg < (1ll << 31), "segment count must lie in [0, 2^31)");
    NERRF_REQUIRE(k >= 1 && k <= 1024, "k must lie in 1..1024 (got %d)", k);
    if (n_seg == 0) return NERRF_OK;
    NERRF_REQUIRE(seg && out_edge && out_attr && out_pos, "null pointer");
    topk_kernel<<<(unsigned)n_seg, XT, 0, (cudaStream_t)stream>>>(seg, ew, d_ew, epos, edge_event, k, out_edge, out_attr, out_pos,
                                                                   out_event);
    return launch_status("explain top-k");
}

extern "C" int nerrf_lstm_explain_steps(const float* seq, const float* dseq, const int32_t* len, int64_t B, int T, int D_in,
                                        const int64_t* step_event, int k, int32_t* out_step, float* out_attr,
                                        int32_t* out_feature, int64_t* out_event, nerrf_stream_t stream) {
    NERRF_REQUIRE(B >= 0, "negative sequence count");
    NERRF_REQUIRE(T >= 1 && D_in >= 1 && D_in <= 1024, "need T >= 1 and D_in in 1..1024 (got T = %d, D_in = %d)", T, D_in);
    NERRF_REQUIRE(k >= 1 && k <= 1024, "k must lie in 1..1024 (got %d)", k);
    if (B == 0) return NERRF_OK;
    NERRF_REQUIRE(seq && dseq && len && out_step && out_attr && out_feature && out_event, "null pointer");
    const int64_t grid = (B + SW - 1) / SW;
    NERRF_REQUIRE(grid < (1ll << 31), "too many sequences for one launch");
    explain_steps_kernel<<<(unsigned)grid, 32 * SW, 0, (cudaStream_t)stream>>>(seq, dseq, len, B, T, D_in, step_event, k, out_step,
                                                                               out_attr, out_feature, out_event);
    return launch_status("explain sequence steps");
}
