// Contamination (DESIGN.md 1.5): the time-respecting causal closure of a window graph from seeded nodes
// (nerrf_taint_closure), and the per-event information-flow class it runs on (nerrf_trace_flow_class_device; the host
// twin nerrf_trace_flow_class is in ingest.cu, both evaluate wire::flow_class).
//
//   validate: grid-stride passes over the nodes (kind), the edges (col range, flow byte) and the seeds (range, NaN time,
//             negative label; duplicates by a compare-and-swap on a per-node seed index) -> one wait.
//   phase 1:  Jacobi rounds, T double-buffered: one warp per row reduces the (t, position) minimum over the row's open
//             edges whose source arrived by t (a row of 10^5 edges costs 10^5 / 32 iterations of one warp); a row that
//             lowers its T stores the round number into a device flag -> one wait per round.
//   phase 2:  level-synchronous BFS over the tight edges: one warp per unlevelled reached row finds the lowest tight
//             position from the current level (a warp min); rows already levelled or unreached leave at once -> one
//             wait per level.  Levels are written in place: a reader tests level == k, which a node being levelled
//             k + 1 in the same launch never equals.
//   compact:  flags -> exclusive scan (scan.cuh) -> the levelled nodes in ascending node id.
// Every value is a function of the inputs (minima with fixed tie rules, no float atomics): two runs give the same bits.
#include <chrono>
#include <cmath>

#include "common.cuh"
#include "scan.cuh"
#include "wire.cuh"

namespace nerrf {
namespace {

constexpr int TW = 8;                 // warps per CTA of the per-row kernels
constexpr int ERR_KIND = 1, ERR_COL = 2, ERR_FLOW = 4, ERR_SEED_RANGE = 8, ERR_SEED_DUP = 16, ERR_SEED_TIME = 32,
              ERR_LABEL = 64;
constexpr int64_t NO_POS = INT64_MAX;

__host__ __device__ __forceinline__ int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

unsigned grid_for(int64_t n, int per_cta) {
    const int64_t cap = 4 * (int64_t)sm_count();
    const int64_t g = (n + per_cta - 1) / per_cta;
    return (unsigned)(g < 1 ? 1 : (g < cap ? g : cap));
}

// edge from a source of kind ku into a row of kind kv carries information in its direction
__device__ __forceinline__ bool flows(int ku, int kv, uint8_t f) {
    return (ku == 1 && kv == 0 && (f & wire::FLOW_P2F)) || (ku == 0 && kv == 1 && (f & wire::FLOW_F2P));
}

static __global__ void flow_kernel(const uint8_t* __restrict__ slot, const int32_t* __restrict__ flags,
                                   const int64_t* __restrict__ ret_val, int64_t n, uint8_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = wire::flow_class(slot[i], flags[i], ret_val[i]);
}

static __global__ void init_kernel(const int8_t* __restrict__ kind, int64_t n, double* __restrict__ T, int32_t* __restrict__ level,
                                   int64_t* __restrict__ pred, int32_t* __restrict__ label, int32_t* __restrict__ seed_idx,
                                   int32_t* __restrict__ err) {
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
        const int k = kind[v];
        if (k != 0 && k != 1) atomicOr(err, ERR_KIND);
        T[v] = INFINITY; level[v] = -1; pred[v] = -1; label[v] = -1; seed_idx[v] = -1;
    }
}

static __global__ void seed_kernel(const int64_t* __restrict__ seeds, const double* __restrict__ seed_time,
                                   const int32_t* __restrict__ seed_label, int64_t n_seeds, int64_t n, double* __restrict__ T,
                                   int32_t* __restrict__ seed_idx, int32_t* __restrict__ err) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_seeds; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = seeds[i];
        const double t = seed_time[i];
        if (isnan(t)) atomicOr(err, ERR_SEED_TIME);
        if (seed_label[i] < 0) atomicOr(err, ERR_LABEL);
        if (s < 0 || s >= n) { atomicOr(err, ERR_SEED_RANGE); continue; }
        if (atomicCAS(&seed_idx[s], -1, (int32_t)i) != -1) atomicOr(err, ERR_SEED_DUP);
        else T[s] = t;
    }
}

// every source id in [0, n) and every flow byte in [0, 3]: E = rowptr[n] is read on the device
template <typename RP>
static __global__ void edge_check_kernel(const RP* __restrict__ rowptr, int64_t n, const int32_t* __restrict__ col,
                                         const uint8_t* __restrict__ flow, int32_t* __restrict__ err) {
    const int64_t E = (int64_t)rowptr[n];
    bool bad_col = false, bad_flow = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t s = col[i];
        bad_col |= s < 0 || (int64_t)s >= n;
        bad_flow |= flow[i] > 3;
    }
    if (__syncthreads_or(bad_col) && threadIdx.x == 0) atomicOr(err, ERR_COL);
    if (__syncthreads_or(bad_flow) && threadIdx.x == 0) atomicOr(err, ERR_FLOW);
}

// (t1, p1) before (t2, p2): smaller time, ties to the lower position; NO_POS = none
__device__ __forceinline__ bool tp_before(double t1, int64_t p1, double t2, int64_t p2) {
    if (p1 == NO_POS) return false;
    if (p2 == NO_POS) return true;
    return t1 < t2 || (t1 == t2 && p1 < p2);
}

// one Jacobi round: Tout[v] = the (t, p)-smallest qualifying t_p of row v when it is below Tin[v], else Tin[v]
template <typename RP>
static __global__ void __launch_bounds__(32 * TW) round_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col, int64_t n,
                                                               const int8_t* __restrict__ kind, const uint8_t* __restrict__ flow,
                                                               const double* __restrict__ et, const double* __restrict__ Tin,
                                                               double* __restrict__ Tout, int32_t round, int32_t* __restrict__ changed) {
    const int lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu;
    for (int64_t v = (int64_t)blockIdx.x * TW + (threadIdx.x >> 5); v < n; v += (int64_t)gridDim.x * TW) {
        const int64_t b = (int64_t)rowptr[v], e = (int64_t)rowptr[v + 1];
        const int kv = kind[v];
        double bt = INFINITY; int64_t bp = NO_POS;
        for (int64_t p = b + lane; p < e; p += 32) {             // a lane's positions ascend: its first minimum is its lowest
            const int32_t u = col[p];
            if (u < 0 || (int64_t)u >= n || !flows(kind[u], kv, flow[p])) continue;
            const double t = et[p];
            if (!isnan(t) && Tin[u] <= t && (bp == NO_POS || t < bt)) { bt = t; bp = p; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ot = __shfl_xor_sync(full, bt, o);
            const int64_t op = __shfl_xor_sync(full, bp, o);
            if (tp_before(ot, op, bt, bp)) { bt = ot; bp = op; }
        }
        if (lane == 0) {
            const double tv = Tin[v];
            const bool lower = bp != NO_POS && bt < tv;
            Tout[v] = lower ? bt : tv;
            if (lower) atomicMax(changed, round);
        }
    }
}

static __global__ void level0_kernel(const int64_t* __restrict__ seeds, const double* __restrict__ seed_time,
                                     const int32_t* __restrict__ seed_label, int64_t n_seeds, const double* __restrict__ T,
                                     int32_t* __restrict__ level, int32_t* __restrict__ label, int32_t* __restrict__ found) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_seeds; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = seeds[i];
        if (T[s] == seed_time[i]) {                              // not reached before its own seed time: a root
            level[s] = 0; label[s] = seed_label[i];
            atomicMax(found, 1);
        }
    }
}

// level k + 1: an unlevelled reached row with a tight in-edge from a level-k node; pred = the lowest such position
template <typename RP>
static __global__ void __launch_bounds__(32 * TW) level_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col, int64_t n,
                                                               const int8_t* __restrict__ kind, const uint8_t* __restrict__ flow,
                                                               const double* __restrict__ et, const double* __restrict__ T,
                                                               int32_t k, int32_t* __restrict__ level, int64_t* __restrict__ pred,
                                                               int32_t* __restrict__ label, int32_t* __restrict__ found) {
    const int lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu;
    for (int64_t v = (int64_t)blockIdx.x * TW + (threadIdx.x >> 5); v < n; v += (int64_t)gridDim.x * TW) {
        const double tv = T[v];
        if (level[v] != -1 || !(tv < INFINITY)) continue;       // the same answer on every lane of the warp
        const int64_t b = (int64_t)rowptr[v], e = (int64_t)rowptr[v + 1];
        const int kv = kind[v];
        int64_t bp = NO_POS;
        for (int64_t p = b + lane; p < e && bp == NO_POS; p += 32) {
            const int32_t u = col[p];
            if (u < 0 || (int64_t)u >= n || !flows(kind[u], kv, flow[p])) continue;
            const double t = et[p];
            if (t == tv && level[u] == k && T[u] <= t) bp = p;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int64_t op = __shfl_xor_sync(full, bp, o);
            bp = op < bp ? op : bp;
        }
        if (lane == 0 && bp != NO_POS) {
            level[v] = k + 1; pred[v] = bp; label[v] = label[col[bp]];
            atomicMax(found, k + 2);
        }
    }
}

static __global__ void flag_kernel(const int32_t* __restrict__ level, int64_t n, int32_t* __restrict__ flag) {
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x)
        flag[v] = level[v] >= 0 ? 1 : 0;
}

static __global__ void compact_kernel(const int32_t* __restrict__ pos, int64_t n, const int32_t* __restrict__ total,
                                      const double* __restrict__ T, const int32_t* __restrict__ level,
                                      const int64_t* __restrict__ pred, const int32_t* __restrict__ label,
                                      int32_t* __restrict__ out_nodes, double* __restrict__ out_time, int32_t* __restrict__ out_level,
                                      int64_t* __restrict__ out_pred, int32_t* __restrict__ out_label) {
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
        const int32_t nxt = v + 1 < n ? pos[v + 1] : *total;
        if (nxt == pos[v]) continue;
        const int32_t q = pos[v];
        out_nodes[q] = (int32_t)v; out_time[q] = T[v]; out_level[q] = level[v]; out_pred[q] = pred[v]; out_label[q] = label[v];
    }
}

struct Ws {
    double *ta, *tb; int32_t *level, *label, *seed_idx, *pos, *sums, *ctl; int64_t* pred;
};

size_t ws_bytes(int64_t n, Ws* w, unsigned char* base) {
    const int64_t nn = n > 0 ? n : 1;
    int64_t off = 0;
    auto take = [&](int64_t bytes) { const int64_t o = off; off += align256(bytes); return base ? base + o : nullptr; };
    Ws t;
    t.ta = (double*)take(8 * nn); t.tb = (double*)take(8 * nn);
    t.pred = (int64_t*)take(8 * nn);
    t.level = (int32_t*)take(4 * nn); t.label = (int32_t*)take(4 * nn); t.seed_idx = (int32_t*)take(4 * nn);
    t.pos = (int32_t*)take(4 * nn);
    t.sums = (int32_t*)take(4 * ((nn + SCAN_TILE - 1) / SCAN_TILE + 2));
    t.ctl = (int32_t*)take(4 * 4);                               // [total, err, round flag, level flag]
    if (w) *w = t;
    return (size_t)off;
}

int wait_read(int32_t* h, const int32_t* d, int count, cudaStream_t st) {
    NERRF_CHECK_CUDA(cudaMemcpyAsync(h, d, 4 * count, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    return NERRF_OK;
}

template <typename RP>
int closure(const RP* rowptr, const int32_t* col, int64_t n, const int8_t* kind, const uint8_t* flow, const double* et,
            const int64_t* seeds, const double* seed_time, const int32_t* seed_label, int64_t n_seeds, int max_hops,
            int32_t* out_nodes, double* out_time, int32_t* out_level, int64_t* out_pred, int32_t* out_label,
            int64_t* n_tainted, int32_t* n_rounds, int32_t* n_levels, double* stage_ms, const Ws& w, cudaStream_t st) {
    // host clock at each stage's closing wait: validation, phase 1, phase 2, compaction (ms)
    auto clock = std::chrono::steady_clock::now();
    auto lap = [&](int i) {
        const auto now = std::chrono::steady_clock::now();
        if (stage_ms) stage_ms[i] = std::chrono::duration<double, std::milli>(now - clock).count();
        clock = now;
    };
    int32_t* err = w.ctl + 1;
    NERRF_CHECK_CUDA(cudaMemsetAsync(w.ctl, 0, 16, st));
    const unsigned gn = grid_for(n, 256), gr = grid_for(n, TW);
    init_kernel<<<gn, 256, 0, st>>>(kind, n, w.ta, w.level, w.pred, w.label, w.seed_idx, err);
    if (n_seeds) seed_kernel<<<grid_for(n_seeds, 256), 256, 0, st>>>(seeds, seed_time, seed_label, n_seeds, n, w.ta, w.seed_idx, err);
    edge_check_kernel<RP><<<grid_for(INT32_MAX, 256), 256, 0, st>>>(rowptr, n, col, flow, err);
    int rc = launch_status("taint validation");
    if (rc) return rc;
    int32_t h[4];
    if ((rc = wait_read(h, w.ctl, 4, st))) return rc;
    NERRF_REQUIRE(!(h[1] & ERR_KIND), "node_kind values must be 0 (file) or 1 (process)");
    NERRF_REQUIRE(!(h[1] & ERR_COL), "col holds node ids outside [0, %lld)", (long long)n);
    NERRF_REQUIRE(!(h[1] & ERR_FLOW), "edge_flow bytes must lie in [0, 3]");
    NERRF_REQUIRE(!(h[1] & ERR_SEED_RANGE), "seed node ids must lie in [0, %lld)", (long long)n);
    NERRF_REQUIRE(!(h[1] & ERR_SEED_DUP), "seed node ids must be distinct");
    NERRF_REQUIRE(!(h[1] & ERR_SEED_TIME), "a seed time is NaN");
    NERRF_REQUIRE(!(h[1] & ERR_LABEL), "seed labels must be >= 0");
    lap(0);
    // phase 1
    double *tin = w.ta, *tout = w.tb;
    int32_t rounds = 0;
    for (int32_t r = 1; max_hops < 0 || r <= max_hops; ++r) {
        round_kernel<RP><<<gr, 32 * TW, 0, st>>>(rowptr, col, n, kind, flow, et, tin, tout, r, w.ctl + 2);
        if ((rc = launch_status("taint round"))) return rc;
        rounds = r;
        double* t_ = tin; tin = tout; tout = t_;
        if ((rc = wait_read(h, w.ctl + 2, 1, st))) return rc;
        if (h[0] != r) break;                                    // the round changed nothing
    }
    lap(1);
    // phase 2 over the final T (tin)
    int32_t levels = 0;
    if (n_seeds) {
        level0_kernel<<<grid_for(n_seeds, 256), 256, 0, st>>>(seeds, seed_time, seed_label, n_seeds, tin, w.level, w.label, w.ctl + 3);
        if ((rc = launch_status("taint level 0"))) return rc;
        if ((rc = wait_read(h, w.ctl + 3, 1, st))) return rc;
        if (h[0] == 1) {
            levels = 1;
            for (int32_t k = 0;; ++k) {
                level_kernel<RP><<<gr, 32 * TW, 0, st>>>(rowptr, col, n, kind, flow, et, tin, k, w.level, w.pred, w.label, w.ctl + 3);
                if ((rc = launch_status("taint level"))) return rc;
                if ((rc = wait_read(h, w.ctl + 3, 1, st))) return rc;
                if (h[0] != k + 2) break;                        // level k + 1 is empty
                levels = k + 2;
            }
        }
    }
    lap(2);
    // compaction
    flag_kernel<<<gn, 256, 0, st>>>(w.level, n, w.pos);
    exclusive_scan_i32(w.pos, n, w.sums, w.ctl, st);
    compact_kernel<<<gn, 256, 0, st>>>(w.pos, n, w.ctl, tin, w.level, w.pred, w.label, out_nodes, out_time, out_level, out_pred,
                                       out_label);
    if ((rc = launch_status("taint compact"))) return rc;
    if ((rc = wait_read(h, w.ctl, 1, st))) return rc;
    lap(3);
    *n_tainted = h[0]; *n_rounds = rounds; *n_levels = levels;
    return NERRF_OK;
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_taint_closure_workspace_bytes(int64_t n_nodes, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_nodes >= 0 && n_nodes < (1ll << 31), "node count must lie in [0, 2^31)");
    *bytes = ws_bytes(n_nodes, nullptr, nullptr) + 256;
    return NERRF_OK;
}

extern "C" int nerrf_taint_closure(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes, const int8_t* node_kind,
                                   const uint8_t* edge_flow, const double* edge_time, const int64_t* seeds, const double* seed_time,
                                   const int32_t* seed_label, int64_t n_seeds, int max_hops, int32_t* out_nodes, double* out_time,
                                   int32_t* out_level, int64_t* out_pred, int32_t* out_label, int64_t* n_tainted, int32_t* n_rounds,
                                   int32_t* n_levels, double* stage_ms, void* workspace, size_t workspace_bytes,
                                   nerrf_stream_t stream) {
    NERRF_REQUIRE(n_nodes >= 0 && n_nodes < (1ll << 31), "node count must lie in [0, 2^31)");
    NERRF_REQUIRE(n_seeds >= 0, "negative seed count");
    NERRF_REQUIRE(max_hops >= -1, "max_hops must be -1 (until nothing changes) or >= 0");
    NERRF_REQUIRE(n_tainted && n_rounds && n_levels, "null count pointer");
    *n_tainted = 0; *n_rounds = 0; *n_levels = 0;
    if (n_nodes == 0) {
        NERRF_REQUIRE(n_seeds == 0, "seed node ids must lie in [0, 0)");
        return NERRF_OK;
    }
    NERRF_REQUIRE(rowptr && col && node_kind && edge_flow && edge_time && out_nodes && out_time && out_level && out_pred &&
                  out_label && workspace && (n_seeds == 0 || (seeds && seed_time && seed_label)), "null pointer");
    const size_t need = ws_bytes(n_nodes, nullptr, nullptr) + 256;
    if (workspace_bytes < need) {
        set_error("taint workspace too small: need %zu bytes", need);
        return NERRF_ERR_WORKSPACE;
    }
    Ws w;
    ws_bytes(n_nodes, &w, (unsigned char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255));
    cudaStream_t st = (cudaStream_t)stream;
    if (rowptr_is64)
        return closure((const int64_t*)rowptr, col, n_nodes, node_kind, edge_flow, edge_time, seeds, seed_time, seed_label, n_seeds,
                       max_hops, out_nodes, out_time, out_level, out_pred, out_label, n_tainted, n_rounds, n_levels, stage_ms, w, st);
    return closure((const int32_t*)rowptr, col, n_nodes, node_kind, edge_flow, edge_time, seeds, seed_time, seed_label, n_seeds,
                   max_hops, out_nodes, out_time, out_level, out_pred, out_label, n_tainted, n_rounds, n_levels, stage_ms, w, st);
}

extern "C" int nerrf_trace_flow_class_device(const uint8_t* event_slot, const int32_t* flags, const int64_t* ret_val, int64_t n,
                                             uint8_t* flow_out, nerrf_stream_t stream) {
    NERRF_REQUIRE(n >= 0, "negative event count");
    if (n == 0) return NERRF_OK;
    NERRF_REQUIRE(event_slot && flags && ret_val && flow_out, "null pointer");
    flow_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(event_slot, flags, ret_val, n, flow_out);
    return launch_status("flow class");
}
