// Incidents (DESIGN.md 1.4): the flagged files of a window graph, each file's owning process and the span of its
// owner's events in the file's row (nerrf_incident_files), and the files grouped by (source, owner) into incident
// records (nerrf_incident_group).
//
//   files:  flag pass (kind == 0 && score >= tau, plus the seeds) -> exclusive scan (scan.cuh) -> compaction in ascending
//           node id -> one warp per flagged row: owner (writer rule: scan back from the row's end in steps of 32; edge
//           rule: a warp arg-max of P(attack) over the row's process sources), then the owner's first / last position
//           (warp min / max) and the count of later events of other processes (warp sum).  A row of 10^5 edges costs
//           3 * 10^5 / 32 iterations of one warp, none of them on one lane alone.
//   group:  key (source << 32 | (uint32)owner; owner -1 sorts last) radix-sorted (radix_sort.cuh, stable: files stay in
//           ascending node id inside a key) -> segment heads by scan -> one warp per incident reduces its files in a fixed
//           lane order (no float atomics) -> a second stable radix sort by onset orders the incidents by
//           (onset, source, owner).
#include "common.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"

namespace nerrf {
namespace {

constexpr int IW = 8;                 // warps per CTA of the per-row and per-incident kernels
constexpr int ERR_KIND = 1, ERR_SEED_RANGE = 2, ERR_SEED_KIND = 4, ERR_COL_RANGE = 8;
constexpr int FILE_INT = 6;           // per flagged file: owner, first, last, later, onset event, end event
constexpr int FILE_REAL = 2;          //                   onset, end
constexpr int INC_INT = 7;            // per incident: source, owner, file offset, n_files, onset event, end event, later
constexpr int INC_REAL = 4;           //               onset, end, size_mb, max_score

__host__ __device__ __forceinline__ int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

static __global__ void flag_kernel(const int8_t* __restrict__ kind, const float* __restrict__ score, float tau, int64_t n,
                                   int32_t* __restrict__ flag, int32_t* __restrict__ err) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = kind[i];
        if (k != 0 && k != 1) atomicOr(err, ERR_KIND);
        flag[i] = (k == 0 && score[i] >= tau) ? 1 : 0;          // NaN compares false: never flagged by its score
    }
}

static __global__ void seed_kernel(const int64_t* __restrict__ seeds, int64_t n_seeds, const int8_t* __restrict__ kind, int64_t n,
                                   int32_t* __restrict__ flag, int32_t* __restrict__ err) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_seeds; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = seeds[i];
        if (s < 0 || s >= n) atomicOr(err, ERR_SEED_RANGE);
        else if (kind[s] != 0) atomicOr(err, ERR_SEED_KIND);
        else flag[s] = 1;                                       // duplicates write the same value
    }
}

// every source id of the graph in [0, n): E = rowptr[n] is read on the device, so the check needs no host copy
template <typename RP>
static __global__ void col_check_kernel(const RP* __restrict__ rowptr, int64_t n, const int32_t* __restrict__ col,
                                        int32_t* __restrict__ err) {
    const int64_t E = (int64_t)rowptr[n];
    bool bad = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t s = col[i];
        bad |= s < 0 || (int64_t)s >= n;
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(err, ERR_COL_RANGE);
}

// pos = exclusive scan of the flags: node i is flagged iff the next prefix (or the total) is larger
static __global__ void compact_kernel(const int32_t* __restrict__ pos, int64_t n, const int32_t* __restrict__ total,
                                      int32_t* __restrict__ files) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t nxt = i + 1 < n ? pos[i + 1] : *total;
        if (nxt != pos[i]) files[pos[i]] = (int32_t)i;
    }
}

// (a1, p1) ranks above (a2, p2): numpy's float order (NaN above every number), ties to the later position
__device__ __forceinline__ bool attack_above(float a1, int64_t p1, float a2, int64_t p2) {
    const bool n1 = isnan(a1), n2 = isnan(a2);
    if (n1 != n2) return n1;
    if (!n1 && a1 != a2) return a1 > a2;
    return p1 > p2;
}

template <typename RP>
static __global__ void __launch_bounds__(32 * IW) owner_kernel(const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                               const int8_t* __restrict__ kind, int64_t n,
                                                               const float* __restrict__ edge_attack,
                                                               const double* __restrict__ edge_time,
                                                               const int64_t* __restrict__ edge_event,
                                                               const int32_t* __restrict__ files, const int32_t* __restrict__ count,
                                                               int64_t* __restrict__ file_int, double* __restrict__ file_real) {
    const int lane = threadIdx.x & 31;
    const int64_t n_files = *count;
    const unsigned full = 0xffffffffu;
    for (int64_t f = (int64_t)blockIdx.x * IW + (threadIdx.x >> 5); f < n_files; f += (int64_t)gridDim.x * IW) {
        const int32_t v = files[f];
        const int64_t b = (int64_t)rowptr[v], e = (int64_t)rowptr[v + 1];
        auto src_at = [&](int64_t p) -> int32_t {               // source of position p; -1 out of range (col_check_kernel
            const int32_t s = col[p];                            // reports it; this keeps the kind[] read in bounds)
            return (s < 0 || (int64_t)s >= n) ? -1 : s;
        };
        int32_t own = -1;
        if (edge_attack == nullptr) {                            // writer rule: the last process source of the row
            for (int64_t base = e; base > b && own < 0; base -= 32) {
                const int64_t p = base - 1 - lane;
                const int32_t s = p >= b ? src_at(p) : -1;
                const unsigned m = __ballot_sync(full, s >= 0 && kind[s] == 1);
                if (m) own = __shfl_sync(full, s, __ffs(m) - 1);
            }
        } else {                                                 // edge rule: highest P(attack), ties to the later position
            float ba = 0.0f; int64_t bp = -1;
            for (int64_t p = b + lane; p < e; p += 32) {
                const int32_t s = src_at(p);
                if (s >= 0 && kind[s] == 1) {
                    const float a = edge_attack[p];
                    if (bp < 0 || attack_above(a, p, ba, bp)) { ba = a; bp = p; }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float oa = __shfl_xor_sync(full, ba, o);
                const int64_t op = __shfl_xor_sync(full, bp, o);
                if (op >= 0 && (bp < 0 || attack_above(oa, op, ba, bp))) { ba = oa; bp = op; }
            }
            if (bp >= 0) own = col[bp];
        }
        int64_t first = -1, last = -1, later = 0;
        if (e > b && own < 0) {
            first = b; last = e - 1;
        } else if (own >= 0) {
            int64_t lo = INT64_MAX, hi = -1;
            for (int64_t p = b + lane; p < e; p += 32)
                if (col[p] == own) { lo = p < lo ? p : lo; hi = p; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const int64_t ol = __shfl_xor_sync(full, lo, o), oh = __shfl_xor_sync(full, hi, o);
                lo = ol < lo ? ol : lo; hi = oh > hi ? oh : hi;
            }
            first = lo; last = hi;
            int64_t c = 0;
            for (int64_t p = first + 1 + lane; p < e; p += 32) {
                const int32_t s = src_at(p);
                c += (s >= 0 && s != own && kind[s] == 1) ? 1 : 0;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(full, c, o);
            later = c;
        }
        if (lane == 0) {
            int64_t* fi = file_int + f * FILE_INT;
            double* fr = file_real + f * FILE_REAL;
            fi[0] = own; fi[1] = first; fi[2] = last; fi[3] = later;
            fi[4] = (first >= 0 && edge_event) ? edge_event[first] : -1;
            fi[5] = (last >= 0 && edge_event) ? edge_event[last] : -1;
            fr[0] = (first >= 0 && edge_time) ? edge_time[first] : __longlong_as_double(0x7ff8000000000000ll);
            fr[1] = (last >= 0 && edge_time) ? edge_time[last] : __longlong_as_double(0x7ff8000000000000ll);
        }
    }
}

// ---- grouping
static __global__ void key_kernel(const int32_t* __restrict__ files, const int64_t* __restrict__ file_int,
                                  const int32_t* __restrict__ node_source, int64_t m, uint64_t* __restrict__ keys,
                                  uint32_t* __restrict__ vals) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = node_source ? (uint32_t)node_source[files[i]] & 0xffffu : 0u;
        keys[i] = ((uint64_t)s << 32) | (uint32_t)(int32_t)file_int[i * FILE_INT];
        vals[i] = (uint32_t)i;
    }
}

static __global__ void head_kernel(const uint64_t* __restrict__ keys, int64_t m, int32_t* __restrict__ head) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
        head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// pos = exclusive scan of the heads -> segment of sorted position q, its first position, the grouped file list
static __global__ void segment_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                      const int32_t* __restrict__ pos, int64_t m, const int32_t* __restrict__ files,
                                      int32_t* __restrict__ seg_of, int32_t* __restrict__ start, int32_t* __restrict__ grouped) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) {
        const bool h = q == 0 || keys[q] != keys[q - 1];
        const int32_t s = h ? pos[q] : pos[q] - 1;
        if (h) start[s] = (int32_t)q;
        seg_of[vals[q]] = s;
        grouped[q] = files[vals[q]];
    }
}

__device__ __forceinline__ uint64_t onset_key(double x) {   // ascending double order; -0 == +0; NaN after every number
    if (isnan(x)) return ~1ull;
    if (x == 0.0) x = 0.0;
    const uint64_t u = (uint64_t)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

// (t1, v1) before (t2, v2) for the onset: smaller time, ties to the lower node; NaN never wins
__device__ __forceinline__ bool onset_before(double t1, int32_t v1, double t2, int32_t v2) {
    if (isnan(t1)) return false;
    if (isnan(t2)) return true;
    return t1 < t2 || (t1 == t2 && v1 < v2);
}
__device__ __forceinline__ bool end_before(double t1, int32_t v1, double t2, int32_t v2) {
    if (isnan(t1)) return false;
    if (isnan(t2)) return true;
    return t1 > t2 || (t1 == t2 && v1 < v2);
}

static __global__ void __launch_bounds__(32 * IW) reduce_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                                const int32_t* __restrict__ start, const int32_t* __restrict__ n_inc_p,
                                                                int64_t m, const int32_t* __restrict__ files,
                                                                const int64_t* __restrict__ file_int, const double* __restrict__ file_real,
                                                                const float* __restrict__ size_mb, const float* __restrict__ score,
                                                                int64_t* __restrict__ inc_int, double* __restrict__ inc_real,
                                                                uint64_t* __restrict__ okeys, uint32_t* __restrict__ ovals) {
    const int lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu;
    const int64_t n_inc = *n_inc_p;
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    for (int64_t j = (int64_t)blockIdx.x * IW + (threadIdx.x >> 5); j < m; j += (int64_t)gridDim.x * IW) {
        if (j >= n_inc) {                                        // padding: sorts after every incident
            if (lane == 0) { okeys[j] = ~0ull; ovals[j] = (uint32_t)j; }
            continue;
        }
        const int64_t a = start[j], z = j + 1 < n_inc ? start[j + 1] : m;
        double on = qnan, en = qnan, sz = 0.0;
        int32_t onv = -1, env = -1;
        int64_t onev = -1, enev = -1, later = 0;
        float ms = __int_as_float(0x7fc00000);
        for (int64_t q = a + lane; q < z; q += 32) {              // each lane: its files in ascending node id
            const uint32_t i = vals[q];
            const int32_t v = files[i];
            const double t0 = file_real[(int64_t)i * FILE_REAL], t1 = file_real[(int64_t)i * FILE_REAL + 1];
            if (onv < 0 ? !isnan(t0) : onset_before(t0, v, on, onv)) { on = t0; onv = v; onev = file_int[(int64_t)i * FILE_INT + 4]; }
            if (env < 0 ? !isnan(t1) : end_before(t1, v, en, env)) { en = t1; env = v; enev = file_int[(int64_t)i * FILE_INT + 5]; }
            sz += (double)size_mb[v];
            later += file_int[(int64_t)i * FILE_INT + 3];
            ms = fmaxf(ms, score[v]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {                       // fixed tree: the same bits on every run
            const double oon = __shfl_xor_sync(full, on, o), oen = __shfl_xor_sync(full, en, o);
            const int32_t oonv = __shfl_xor_sync(full, onv, o), oenv = __shfl_xor_sync(full, env, o);
            const int64_t oonev = __shfl_xor_sync(full, onev, o), oenev = __shfl_xor_sync(full, enev, o);
            if (oonv >= 0 && (onv < 0 || onset_before(oon, oonv, on, onv))) { on = oon; onv = oonv; onev = oonev; }
            if (oenv >= 0 && (env < 0 || end_before(oen, oenv, en, env))) { en = oen; env = oenv; enev = oenev; }
            sz += __shfl_xor_sync(full, sz, o);
            later += __shfl_xor_sync(full, later, o);
            ms = fmaxf(ms, __shfl_xor_sync(full, ms, o));
        }
        if (lane == 0) {
            const uint64_t k = keys[a];
            int64_t* ii = inc_int + j * INC_INT;
            double* ir = inc_real + j * INC_REAL;
            ii[0] = (int64_t)(k >> 32); ii[1] = (int32_t)(uint32_t)k; ii[2] = a; ii[3] = z - a; ii[4] = onev; ii[5] = enev; ii[6] = later;
            ir[0] = on; ir[1] = en; ir[2] = sz; ir[3] = (double)ms;
            okeys[j] = onset_key(on); ovals[j] = (uint32_t)j;
        }
    }
}

static __global__ void order_kernel(const uint32_t* __restrict__ sorted, const int32_t* __restrict__ n_inc_p,
                                    const int64_t* __restrict__ inc_int, const double* __restrict__ inc_real,
                                    int64_t* __restrict__ out_int, double* __restrict__ out_real, int32_t* __restrict__ rank) {
    const int64_t n_inc = *n_inc_p;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_inc; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t j = sorted[r];
        rank[j] = (int32_t)r;
#pragma unroll
        for (int c = 0; c < INC_INT; ++c) out_int[r * INC_INT + c] = inc_int[(int64_t)j * INC_INT + c];
#pragma unroll
        for (int c = 0; c < INC_REAL; ++c) out_real[r * INC_REAL + c] = inc_real[(int64_t)j * INC_REAL + c];
    }
}

static __global__ void file_incident_kernel(const int32_t* __restrict__ seg_of, const int32_t* __restrict__ rank, int64_t m,
                                            int32_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = rank[seg_of[i]];
}

unsigned grid_for(int64_t n, int per_cta) {
    const int64_t cap = 4 * (int64_t)sm_count();
    const int64_t g = (n + per_cta - 1) / per_cta;
    return (unsigned)(g < 1 ? 1 : (g < cap ? g : cap));
}

size_t files_ws_bytes(int64_t n) {
    return (size_t)(align256(4 * (n > 0 ? n : 1)) + align256(4 * ((n + SCAN_TILE - 1) / SCAN_TILE + 4)) + 256);
}

struct GroupWs {
    uint64_t *ka, *kb; uint32_t *va, *vb; int32_t *pos, *seg_of, *start, *rank, *n_inc; int64_t* inc_int; double* inc_real;
    int32_t* sums; void* rs;
};

size_t group_ws_bytes(int64_t m, GroupWs* w, unsigned char* base) {
    const int64_t mm = m > 0 ? m : 1;
    int64_t off = 0;
    auto take = [&](int64_t bytes) { const int64_t o = off; off += align256(bytes); return base ? base + o : nullptr; };
    GroupWs t;
    t.ka = (uint64_t*)take(8 * mm); t.kb = (uint64_t*)take(8 * mm);
    t.va = (uint32_t*)take(4 * mm); t.vb = (uint32_t*)take(4 * mm);
    t.pos = (int32_t*)take(4 * mm); t.seg_of = (int32_t*)take(4 * mm); t.start = (int32_t*)take(4 * mm);
    t.rank = (int32_t*)take(4 * mm); t.n_inc = (int32_t*)take(8);
    t.inc_int = (int64_t*)take(8 * INC_INT * mm); t.inc_real = (double*)take(8 * INC_REAL * mm);
    t.sums = (int32_t*)take(4 * ((mm + SCAN_TILE - 1) / SCAN_TILE + 2));
    t.rs = take((int64_t)rs_scratch_bytes(mm));
    if (w) *w = t;
    return (size_t)off;
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_incident_files_workspace_bytes(int64_t n_nodes, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_nodes >= 0 && n_nodes < (1ll << 31), "node count must lie in [0, 2^31)");
    *bytes = files_ws_bytes(n_nodes);
    return NERRF_OK;
}

extern "C" int nerrf_incident_files(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes,
                                    const int8_t* node_kind, const float* score, float tau, const int64_t* seeds, int64_t n_seeds,
                                    const float* edge_attack, const double* edge_time, const int64_t* edge_event,
                                    int32_t* out_files, int64_t* out_int, double* out_real, int64_t* n_flagged,
                                    void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    NERRF_REQUIRE(n_nodes >= 0 && n_nodes < (1ll << 31), "node count must lie in [0, 2^31)");
    NERRF_REQUIRE(n_seeds >= 0, "negative seed count");
    NERRF_REQUIRE(!isnan(tau), "tau is NaN");
    NERRF_REQUIRE(n_flagged, "null n_flagged");
    *n_flagged = 0;
    if (n_nodes == 0) {
        NERRF_REQUIRE(n_seeds == 0, "seed node ids must lie in [0, 0)");
        return NERRF_OK;
    }
    NERRF_REQUIRE(rowptr && col && node_kind && score && out_files && out_int && out_real && workspace && (n_seeds == 0 || seeds),
                  "null pointer");
    if (workspace_bytes < files_ws_bytes(n_nodes)) {
        set_error("incident workspace too small: need %zu bytes", files_ws_bytes(n_nodes));
        return NERRF_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* ws = (unsigned char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    int32_t* pos = (int32_t*)ws;
    int32_t* sums = (int32_t*)(ws + align256(4 * n_nodes));
    int32_t* total = sums + (n_nodes + SCAN_TILE - 1) / SCAN_TILE + 1;   // [total, err]
    NERRF_CHECK_CUDA(cudaMemsetAsync(total + 1, 0, 4, st));
    flag_kernel<<<grid_for(n_nodes, 256), 256, 0, st>>>(node_kind, score, tau, n_nodes, pos, total + 1);
    if (n_seeds) seed_kernel<<<grid_for(n_seeds, 256), 256, 0, st>>>(seeds, n_seeds, node_kind, n_nodes, pos, total + 1);
    exclusive_scan_i32(pos, n_nodes, sums, total, st);
    compact_kernel<<<grid_for(n_nodes, 256), 256, 0, st>>>(pos, n_nodes, total, out_files);
    const unsigned g = grid_for(n_nodes, IW);
    if (rowptr_is64)
        col_check_kernel<int64_t><<<grid_for(INT32_MAX, 256), 256, 0, st>>>((const int64_t*)rowptr, n_nodes, col, total + 1);
    else
        col_check_kernel<int32_t><<<grid_for(INT32_MAX, 256), 256, 0, st>>>((const int32_t*)rowptr, n_nodes, col, total + 1);
    if (rowptr_is64)
        owner_kernel<int64_t><<<g, 32 * IW, 0, st>>>((const int64_t*)rowptr, col, node_kind, n_nodes, edge_attack, edge_time, edge_event,
                                                     out_files, total, out_int, out_real);
    else
        owner_kernel<int32_t><<<g, 32 * IW, 0, st>>>((const int32_t*)rowptr, col, node_kind, n_nodes, edge_attack, edge_time, edge_event,
                                                     out_files, total, out_int, out_real);
    int rc = launch_status("incident files");
    if (rc) return rc;
    // the one wait of this call: the flagged count sizes the caller's next step, and bad input must be an error code
    int32_t h[2];
    NERRF_CHECK_CUDA(cudaMemcpyAsync(h, total, 8, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    NERRF_REQUIRE(!(h[1] & ERR_KIND), "node_kind values must be 0 (file) or 1 (process)");
    NERRF_REQUIRE(!(h[1] & ERR_SEED_RANGE), "seed node ids must lie in [0, %lld)", (long long)n_nodes);
    NERRF_REQUIRE(!(h[1] & ERR_SEED_KIND), "a seed is not a file node");
    NERRF_REQUIRE(!(h[1] & ERR_COL_RANGE), "col holds node ids outside [0, %lld)", (long long)n_nodes);
    *n_flagged = h[0];
    return NERRF_OK;
}

extern "C" int nerrf_incident_group_workspace_bytes(int64_t n_flagged, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_flagged >= 0 && n_flagged < (1ll << 31), "flagged count must lie in [0, 2^31)");
    *bytes = group_ws_bytes(n_flagged, nullptr, nullptr) + 256;
    return NERRF_OK;
}

extern "C" int nerrf_incident_group(const int32_t* files, const int64_t* file_int, const double* file_real, int64_t n_flagged,
                                    const int32_t* node_source, const float* size_mb, const float* score,
                                    int32_t* n_incidents, int64_t* inc_int, double* inc_real, int32_t* grouped_files,
                                    int32_t* file_incident, void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    NERRF_REQUIRE(n_flagged >= 0 && n_flagged < (1ll << 31), "flagged count must lie in [0, 2^31)");
    NERRF_REQUIRE(n_incidents, "null n_incidents");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_flagged == 0) {
        NERRF_CHECK_CUDA(cudaMemsetAsync(n_incidents, 0, 4, st));
        return NERRF_OK;
    }
    NERRF_REQUIRE(files && file_int && file_real && size_mb && score && inc_int && inc_real && grouped_files && file_incident && workspace,
                  "null pointer");
    const size_t need = group_ws_bytes(n_flagged, nullptr, nullptr) + 256;
    if (workspace_bytes < need) {
        set_error("incident group workspace too small: need %zu bytes", need);
        return NERRF_ERR_WORKSPACE;
    }
    GroupWs w;
    group_ws_bytes(n_flagged, &w, (unsigned char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255));
    const int64_t m = n_flagged;
    const unsigned g = grid_for(m, 256);
    key_kernel<<<g, 256, 0, st>>>(files, file_int, node_source, m, w.ka, w.va);
    const int cur = radix_sort_pairs(w.ka, w.kb, w.va, w.vb, m, 0, 48, w.rs, st);
    const uint64_t* keys = cur ? w.kb : w.ka;
    const uint32_t* vals = cur ? w.vb : w.va;
    head_kernel<<<g, 256, 0, st>>>(keys, m, w.pos);
    exclusive_scan_i32(w.pos, m, w.sums, w.n_inc, st);
    segment_kernel<<<g, 256, 0, st>>>(keys, vals, w.pos, m, files, w.seg_of, w.start, grouped_files);
    // the per-incident sort keys take the pair of sort buffers the file sort left free; the file keys / values are not
    // read after reduce_kernel, so the second sort may use their buffers
    uint64_t* ok_a = cur ? w.ka : w.kb;
    uint32_t* ov_a = cur ? w.va : w.vb;
    reduce_kernel<<<grid_for(m, IW), 32 * IW, 0, st>>>(keys, vals, w.start, w.n_inc, m, files, file_int, file_real, size_mb, score,
                                                       w.inc_int, w.inc_real, ok_a, ov_a);
    // stable: incidents enter in (source, owner) order, so the result is ordered by (onset, source, owner)
    uint64_t* kb2 = (uint64_t*)(cur ? w.kb : w.ka);
    uint32_t* vb2 = (uint32_t*)(cur ? w.vb : w.va);
    const int cur2 = radix_sort_pairs(ok_a, kb2, ov_a, vb2, m, 0, 64, w.rs, st);
    const uint32_t* sorted = cur2 ? vb2 : ov_a;
    order_kernel<<<g, 256, 0, st>>>(sorted, w.n_inc, w.inc_int, w.inc_real, inc_int, inc_real, w.rank);
    file_incident_kernel<<<g, 256, 0, st>>>(w.seg_of, w.rank, m, file_incident);
    NERRF_CHECK_CUDA(cudaMemcpyAsync(n_incidents, w.n_inc, 4, cudaMemcpyDeviceToDevice, st));
    return launch_status("incident group");
}
