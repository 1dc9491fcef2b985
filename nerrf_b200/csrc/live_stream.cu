// The live event stream on the device: EventBatch records decoded in HBM as they arrive, appended to device columns
// the caller owns, and the resident events re-ordered, resolved and trimmed after every append.  Host side:
// nerrf_b200/stream.py DeviceStream.live / append / compact.
//
//   nerrf_trace_decode_device   one thread per record parses the Event body with the shared wire parser (csrc/wire.cuh,
//                               the same code as the host decoder) and writes the scalars at row n_old + k and each
//                               string's (start, length) into staging; one exclusive scan turns the lengths into string
//                               offsets; one warp per record copies the bytes and computes path_flags over them.  A
//                               malformed record does an atomicMin of its byte offset into the status word.
//   nerrf_trace_stream_order    stable time order (LSD radix sort of the orderable float64 bits, radix_sort.cuh); the
//                               columnar resolve_columns of nerrf_b200/ingest.py: a stable regroup by (source, pid) (radix
//                               sort of the pid, or of (source << 32) | pid in 6 digit passes instead of 4 when some
//                               source is nonzero, over the time order), then a segmented "last event with a path so far" max-scan
//                               gives the source event of every path-less write, or drops it; the survivors' time order;
//                               the resolved path offsets; and the rows to keep at a retention horizon.
//   nerrf_trace_stream_columns  the resolved path column (warp per event) and the per-event flags / slots the window
//                               graph reads.
//   nerrf_trace_gather_rows     a subset of rows of every column, stored order kept (retention).
#include "common.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "wire.cuh"

namespace nerrf {
namespace {

constexpr int N_COLS = 17;     // ts_sec, ts_nanos, pid, tid, flags, ret_val, bytes, event_slot, path_flags, 4 x (off, data)
constexpr int32_t NEG = -2147483647 - 1;

inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---- inclusive max-scan of int32 [m] in place (the segmented "last so far" scans): per-tile scan + tile maxima, exclusive
// scan of the maxima by one CTA, combine.  Same three-launch shape as scan.cuh.
__global__ void __launch_bounds__(256) maxscan_tiles_kernel(int32_t* __restrict__ v, int64_t m, int32_t* __restrict__ sums) {
    __shared__ int32_t warp_tot[8];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + threadIdx.x * 4;
    int32_t x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = (base + k < m) ? v[base + k] : NEG;
    const int32_t mine = max(max(x[0], x[1]), max(x[2], x[3]));
    int32_t inc = mine;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc = max(inc, t); }
    int32_t prev = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) prev = NEG;
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    int32_t wbase = NEG;
    for (int w = 0; w < warp; ++w) wbase = max(wbase, warp_tot[w]);
    int32_t run = max(wbase, prev);
#pragma unroll
    for (int k = 0; k < 4; ++k) { run = max(run, x[k]); if (base + k < m) v[base + k] = run; }
    if (threadIdx.x == 255) sums[blockIdx.x] = max(wbase, inc);
}
__global__ void __launch_bounds__(1024) maxscan_sums_kernel(int32_t* __restrict__ sums, int64_t nb) {
    __shared__ int32_t warp_tot[32];
    __shared__ int32_t carry_s;
    if (threadIdx.x == 0) carry_s = NEG;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t b0 = 0; b0 < nb; b0 += 1024) {
        const int64_t i = b0 + threadIdx.x;
        const int32_t x = i < nb ? sums[i] : NEG;
        int32_t inc = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc = max(inc, t); }
        int32_t prev = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 0) prev = NEG;
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        int32_t wbase = NEG;
        for (int w = 0; w < warp; ++w) wbase = max(wbase, warp_tot[w]);
        const int32_t carry = carry_s;
        if (i < nb) sums[i] = max(carry, max(wbase, prev));              // exclusive: the maximum of the tiles before
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = max(carry, max(wbase, inc));
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) maxscan_add_kernel(int32_t* __restrict__ v, int64_t m, const int32_t* __restrict__ sums) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + threadIdx.x * 4;
    const int32_t c = sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < 4; ++k) if (base + k < m) v[base + k] = max(v[base + k], c);
}
inline void inclusive_max_scan_i32(int32_t* v, int64_t m, int32_t* sums, cudaStream_t st) {
    const int64_t nb = (m + SCAN_TILE - 1) / SCAN_TILE;
    maxscan_tiles_kernel<<<(unsigned)nb, 256, 0, st>>>(v, m, sums);
    maxscan_sums_kernel<<<1, 1024, 0, st>>>(sums, nb);
    maxscan_add_kernel<<<(unsigned)nb, 256, 0, st>>>(v, m, sums);
}

// ---- columns: the 17 pointers of nerrf_trace_decode's outputs, in its argument order
struct Cols {
    int64_t* ts_sec; int32_t* ts_nanos; uint32_t* pid; uint32_t* tid; int32_t* flags; int64_t* ret_val; uint64_t* bytes;
    uint8_t* event_slot; uint8_t* path_flags;
    int64_t* off[4]; uint8_t* data[4];
    uint16_t* source;            // source id per row (not one of the 17; NULL = not stored)
};
Cols make_cols(void* const* p) {
    Cols c;
    c.ts_sec = (int64_t*)p[0]; c.ts_nanos = (int32_t*)p[1]; c.pid = (uint32_t*)p[2]; c.tid = (uint32_t*)p[3];
    c.flags = (int32_t*)p[4]; c.ret_val = (int64_t*)p[5]; c.bytes = (uint64_t*)p[6]; c.event_slot = (uint8_t*)p[7];
    c.path_flags = (uint8_t*)p[8];
    for (int k = 0; k < 4; ++k) { c.off[k] = (int64_t*)p[9 + 2 * k]; c.data[k] = (uint8_t*)p[10 + 2 * k]; }
    c.source = nullptr;
    return c;
}
bool cols_ok(void* const* p) {
    if (!p) return false;
    for (int k = 0; k < N_COLS; ++k) if (!p[k]) return false;
    return true;
}

// ---- decode: thread per record
__global__ void __launch_bounds__(256) decode_records_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ rec_at,
                                                             const int64_t* __restrict__ body_off, const int64_t* __restrict__ body_len,
                                                             int64_t m, int64_t n_old, Cols c, uint16_t source, int64_t* __restrict__ start,
                                                             int32_t* __restrict__ len, unsigned long long* __restrict__ status) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += stride) {
        wire::EventView e;
        const uint8_t* s = buf + body_off[k];
        if (!wire::parse_event(s, (uint64_t)body_len[k], &e)) {
            atomicMin(status, (unsigned long long)rec_at[k]);
            for (int q = 0; q < 4; ++q) { start[q * m + k] = 0; len[q * m + k] = 0; }
            continue;
        }
        const int64_t row = n_old + k;
        c.ts_sec[row] = e.ts_sec; c.ts_nanos[row] = e.ts_nanos; c.pid[row] = e.pid; c.tid[row] = e.tid; c.flags[row] = e.flags;
        c.ret_val[row] = e.ret_val; c.bytes[row] = e.bytes;
        if (c.source) c.source[row] = source;
        c.event_slot[row] = (uint8_t)wire::event_slot(e.syscall, e.syscall_n);
        const uint8_t* str[4] = {e.comm, e.syscall, e.path, e.new_path};
        const uint64_t sn[4] = {e.comm_n, e.syscall_n, e.path_n, e.new_path_n};
#pragma unroll
        for (int q = 0; q < 4; ++q) { start[q * m + k] = sn[q] ? str[q] - buf : 0; len[q * m + k] = (int32_t)sn[q]; }
    }
}

// NERRF_PATH_* bits of s[0..n) by one warp (the rules of wire::path_flags; every lane gets the result)
__device__ __forceinline__ uint8_t warp_path_flags(const uint8_t* __restrict__ s, int64_t n, int lane) {
    bool lock = false, note = false;
    for (int64_t i = lane; i + 6 <= n; i += 32) {
        if (i + 8 <= n && wire::matches_at(s + i, ".lockbit", 8)) lock = true;
        if (wire::note_word_at(s + i)) note = true;
    }
    uint8_t pf = 0;
    if (__any_sync(0xffffffffu, lock)) pf |= NERRF_PATH_LOCKBIT;
    if (__any_sync(0xffffffffu, note)) pf |= NERRF_PATH_NOTE;
    if (wire::starts_with(s, (uint64_t)n, "/tmp", 4) || wire::starts_with(s, (uint64_t)n, "/proc", 5)) pf |= NERRF_PATH_TMP;
    if (wire::ends_with(s, (uint64_t)n, ".lockbit3", 9)) pf |= NERRF_PATH_ENCRYPTED;
    return pf;
}

// ---- string copy: warp per row k; string q of row k = src[q] + start[q*m + k], length from the scanned lengths; written
// at data[q] + off[q][n_old] + (relative offset), off[q][n_old + k + 1] set.  pf_out != NULL: path_flags of column 2.
struct StrSrc { const uint8_t* base[4]; };
__global__ void __launch_bounds__(256) copy_strings_kernel(StrSrc src, const int64_t* __restrict__ start, const int32_t* __restrict__ scan,
                                                           const int32_t* __restrict__ total, int64_t m, int64_t n_old, Cols c,
                                                           uint8_t* __restrict__ pf_out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t m4 = 4 * m;
    for (int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < m; k += warps) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {                                  // unrolled: the column pointers stay in registers
            const int64_t idx = q * m + k;
            const int32_t s0 = scan[idx];
            const int64_t n = (int64_t)((idx + 1 < m4 ? scan[idx + 1] : *total) - s0);
            const int64_t rel = (int64_t)(s0 - scan[q * m]);
            const int64_t base = c.off[q][n_old];
            const uint8_t* s = src.base[q] + start[idx];
            uint8_t* d = c.data[q] + base + rel;
            for (int64_t i = lane; i < n; i += 32) d[i] = s[i];
            if (q == 2 && pf_out) {
                const uint8_t pf = warp_path_flags(s, n, lane);
                if (lane == 0) pf_out[n_old + k] = pf;
            }
            if (lane == 0) c.off[q][n_old + k + 1] = base + rel + n;
        }
    }
}

struct DecodeWs { size_t start, scan, sums, total, bytes; };
DecodeWs decode_layout(int64_t m) {
    DecodeWs L;
    const int64_t m4 = 4 * (m > 0 ? m : 1);
    size_t o = 0;
    L.start = o; o += up256((size_t)m4 * 8);
    L.scan = o; o += up256((size_t)m4 * 4);
    L.sums = o; o += up256((size_t)((m4 + SCAN_TILE - 1) / SCAN_TILE + 1) * 4);
    L.total = o; o += 256;
    L.bytes = o;
    return L;
}

// ---- gather: scalars thread per row, strings via copy_strings_kernel
__global__ void __launch_bounds__(256) gather_scalars_kernel(Cols in, const int64_t* __restrict__ rows, int64_t m, Cols out,
                                                             int64_t* __restrict__ start, int32_t* __restrict__ len) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += stride) {
        const int64_t r = rows[k];
        out.ts_sec[k] = in.ts_sec[r]; out.ts_nanos[k] = in.ts_nanos[r]; out.pid[k] = in.pid[r]; out.tid[k] = in.tid[r];
        out.flags[k] = in.flags[r]; out.ret_val[k] = in.ret_val[r]; out.bytes[k] = in.bytes[r];
        out.event_slot[k] = in.event_slot[r]; out.path_flags[k] = in.path_flags[r];
        if (out.source) out.source[k] = in.source ? in.source[r] : (uint16_t)0;
#pragma unroll
        for (int q = 0; q < 4; ++q) { start[q * m + k] = in.off[q][r]; len[q * m + k] = (int32_t)(in.off[q][r + 1] - in.off[q][r]); }
    }
}

// ---- order / resolve / retain
struct OrderArgs {
    int64_t n;
    const int64_t* ts_sec; const int32_t* ts_nanos; const uint32_t* pid; const int64_t* path_off;
    const uint16_t* source;      // [n] source id per event, read only when key_bits == 48 (NULL: all 0)
    int key_bits;                // 32: regroup by pid; 48: by (source << 32) | pid
    double horizon;
    double* ts;                  // [n] float64 timestamps by stored index
    uint32_t* tord;              // [n] stored index by time rank
    uint32_t* byp;               // [n] stored index by position in the pid regroup
    int32_t *A, *G, *C;          // [n] max-scans over the regroup: last named, group start, last named at or before the horizon
    int32_t *F, *R, *L;          // [n] keep flags by time rank, retain flags / resolved path lengths by stored index
    int64_t* src;                // [n] source event of the path (-1: dropped)
    unsigned long long* res_bytes;   // the sum of L in 64 bits: L is scanned in int32, and the caller checks this first
};

__device__ __forceinline__ uint64_t orderable(double t) {
    uint64_t b = (uint64_t)__double_as_longlong(t);
    if (b == 0x8000000000000000ull) b = 0;                                   // -0.0 sorts with +0.0 (numpy compares equal)
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__global__ void __launch_bounds__(256) order_keys_kernel(OrderArgs a, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.res_bytes = 0ull;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
        // seconds + nanos * 1e-9 rounded exactly like numpy (two roundings, no FMA contraction)
        const double t = __dadd_rn((double)a.ts_sec[i], __dmul_rn((double)a.ts_nanos[i], 1e-9));
        a.ts[i] = t;
        key[i] = orderable(t);
        val[i] = (uint32_t)i;
        a.R[i] = t > a.horizon ? 1 : 0;
    }
}
// time rank k: remember the time order, key the (source, pid) for the stable regroup (in place: same index read and written)
__global__ void __launch_bounds__(256) order_pid_keys_kernel(OrderArgs a, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        const uint32_t e = val[k];
        a.tord[k] = e;
        key[k] = (a.key_bits > 32 && a.source) ? ((uint64_t)a.source[e] << 32) | a.pid[e] : (uint64_t)a.pid[e];
        val[k] = (uint32_t)k;
    }
}
__global__ void __launch_bounds__(256) order_segments_kernel(OrderArgs a, const uint64_t* __restrict__ key, const uint32_t* __restrict__ val) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.n; j += stride) {
        const uint32_t e = a.tord[val[j]];
        a.byp[j] = e;
        const bool start = j == 0 || key[j] != key[j - 1];
        const bool named = a.path_off[e + 1] > a.path_off[e];
        a.A[j] = named ? (int32_t)j : NEG;
        a.G[j] = start ? (int32_t)j : 0;
        a.C[j] = (named && !(a.ts[e] > a.horizon)) ? (int32_t)j : NEG;
    }
}
__global__ void __launch_bounds__(256) order_resolve_kernel(OrderArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.n; j += stride) {
        const uint32_t e = a.byp[j];
        const int32_t g = a.G[j];
        a.src[e] = a.A[j] >= g ? (int64_t)a.byp[a.A[j]] : -1;
        const bool last = j + 1 == a.n || a.G[j + 1] != g;
        if (last && a.C[j] >= g) a.R[a.byp[a.C[j]]] = 1;                   // the (source, pid)'s latest named event at the horizon
    }
}
__global__ void __launch_bounds__(256) order_flags_kernel(OrderArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned long long bytes = 0ull;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        a.F[k] = a.src[a.tord[k]] >= 0 ? 1 : 0;
        const int64_t s = a.src[k];
        const int64_t len = s >= 0 ? a.path_off[s + 1] - a.path_off[s] : 0;
        a.L[k] = (int32_t)len;
        bytes += (unsigned long long)len;
    }
    // a path is repeated for every path-less write that resolves to it, so the stored bytes do not bound this sum
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bytes += __shfl_down_sync(0xffffffffu, bytes, o);
    if ((threadIdx.x & 31) == 0 && bytes) atomicAdd(a.res_bytes, bytes);
}
// exclusive-scanned flags -> compacted lists
__global__ void __launch_bounds__(256) order_compact_kernel(OrderArgs a, const int32_t* __restrict__ totals, int64_t* __restrict__ order,
                                                            double* __restrict__ ts_sorted, int64_t* __restrict__ retain,
                                                            int64_t* __restrict__ res_off) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        const int32_t f_next = k + 1 < a.n ? a.F[k + 1] : totals[0];
        if (f_next != a.F[k]) { const uint32_t e = a.tord[k]; order[a.F[k]] = e; ts_sorted[a.F[k]] = a.ts[e]; }
        const int32_t r_next = k + 1 < a.n ? a.R[k + 1] : totals[1];
        if (retain && r_next != a.R[k]) retain[a.R[k]] = k;
        res_off[k] = a.L[k];
        if (k + 1 == a.n) res_off[a.n] = totals[2];
    }
}

struct OrderWs { size_t ka, kb, va, vb, tord, byp, A, G, C, F, R, L, sums, totals, rs, bytes; };
OrderWs order_layout(int64_t n) {
    OrderWs L;
    const size_t n8 = up256((size_t)n * 8), n4 = up256((size_t)n * 4);
    size_t o = 0;
    L.ka = o; o += n8; L.kb = o; o += n8;
    L.va = o; o += n4; L.vb = o; o += n4; L.tord = o; o += n4; L.byp = o; o += n4;
    L.A = o; o += n4; L.G = o; o += n4; L.C = o; o += n4; L.F = o; o += n4; L.R = o; o += n4; L.L = o; o += n4;
    L.sums = o; o += up256((size_t)((n + SCAN_TILE - 1) / SCAN_TILE + 1) * 4);
    L.totals = o; o += 256;
    L.rs = o; o += up256(rs_scratch_bytes(n));
    L.bytes = o;
    return L;
}

// ---- resolved columns: warp per stored event
__global__ void __launch_bounds__(256) stream_columns_kernel(int64_t n, const int64_t* __restrict__ src, const int64_t* __restrict__ path_off,
                                                             const uint8_t* __restrict__ path_data, const uint8_t* __restrict__ path_flags,
                                                             const int64_t* __restrict__ gpath_off, const uint8_t* __restrict__ gpath_data,
                                                             const uint8_t* __restrict__ event_slot, const uint8_t* __restrict__ slot_map,
                                                             const int64_t* __restrict__ res_off, int merge, uint8_t* __restrict__ res_data,
                                                             uint8_t* __restrict__ pf_out, uint8_t* __restrict__ pf_raw_out,
                                                             uint8_t* __restrict__ slot_out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int64_t s = src[i];
        if (s >= 0) {
            const uint8_t* p = path_data + path_off[s];
            uint8_t* d = res_data + res_off[i];
            const int64_t len = res_off[i + 1] - res_off[i];
            for (int64_t k = lane; k < len; k += 32) d[k] = p[k];
        }
        bool lock = false;
        if (merge) {                                                   // the renamed twin is the same node: its .lockbit bit counts
            const uint8_t* g = gpath_data + gpath_off[i];
            const int64_t gn = gpath_off[i + 1] - gpath_off[i];
            for (int64_t k = lane; k + 8 <= gn; k += 32)
                if (wire::matches_at(g + k, ".lockbit", 8)) lock = true;
        }
        lock = __any_sync(0xffffffffu, lock);
        if (lane == 0) {
            const uint8_t raw = s >= 0 ? path_flags[s] : 0;
            pf_raw_out[i] = raw;
            pf_out[i] = raw | (lock ? (uint8_t)NERRF_PATH_LOCKBIT : (uint8_t)0);
            const uint8_t sl = event_slot[i];
            slot_out[i] = slot_map ? slot_map[sl & 7] : sl;
        }
    }
}

int grid_for(int64_t n, int per_block) {
    const int64_t b = (n + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_trace_decode_device_workspace_bytes(int64_t n_records, int64_t* bytes) {
    NERRF_REQUIRE(bytes && n_records >= 0 && n_records < ((int64_t)1 << 28), "bad arguments");
    *bytes = (int64_t)decode_layout(n_records).bytes;
    return NERRF_OK;
}

extern "C" int nerrf_trace_decode_device_ex(const uint8_t* buf, const int64_t* rec_at, const int64_t* body_off, const int64_t* body_len,
                                            int64_t n_records, int64_t n_old, void* const* cols, uint16_t* source_col, int source,
                                            uint64_t* status, void* workspace, int64_t workspace_bytes, void* stream) {
    NERRF_REQUIRE(status, "null status");
    NERRF_REQUIRE(n_records >= 0 && n_records < ((int64_t)1 << 28) && n_old >= 0, "bad record count");
    NERRF_REQUIRE(source >= 0 && source < (1 << 16), "source=%d out of range [0, 65536)", source);
    cudaStream_t st = (cudaStream_t)stream;
    NERRF_CHECK_CUDA(cudaMemsetAsync(status, 0xff, 8, st));                  // all ones: no record failed
    if (n_records == 0) return NERRF_OK;
    NERRF_REQUIRE(buf && rec_at && body_off && body_len && workspace, "null pointer");
    NERRF_REQUIRE(cols_ok(cols), "null column pointer");
    const DecodeWs L = decode_layout(n_records);
    NERRF_REQUIRE(workspace_bytes >= (int64_t)L.bytes, "workspace too small: %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)L.bytes);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    char* ws = (char*)workspace;
    Cols c = make_cols(cols);
    c.source = source_col;
    int64_t* start = (int64_t*)(ws + L.start);
    int32_t* scan = (int32_t*)(ws + L.scan);
    int32_t* total = (int32_t*)(ws + L.total);
    decode_records_kernel<<<grid_for(n_records, 256), 256, 0, st>>>(buf, rec_at, body_off, body_len, n_records, n_old, c,
                                                                     (uint16_t)source, start, scan, (unsigned long long*)status);
    exclusive_scan_i32(scan, 4 * n_records, (int32_t*)(ws + L.sums), total, st);
    StrSrc s;
    for (int q = 0; q < 4; ++q) s.base[q] = buf;
    copy_strings_kernel<<<grid_for(n_records, 8), 256, 0, st>>>(s, start, scan, total, n_records, n_old, c, c.path_flags);
    return launch_status("device decoder kernels");
}

extern "C" int nerrf_trace_decode_device(const uint8_t* buf, const int64_t* rec_at, const int64_t* body_off, const int64_t* body_len,
                                         int64_t n_records, int64_t n_old, void* const* cols, uint64_t* status, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
    return nerrf_trace_decode_device_ex(buf, rec_at, body_off, body_len, n_records, n_old, cols, nullptr, 0, status, workspace,
                                        workspace_bytes, stream);
}

extern "C" int nerrf_trace_stream_order_workspace_bytes(int64_t n_events, int64_t* bytes) {
    NERRF_REQUIRE(bytes && n_events >= 0 && n_events < ((int64_t)1 << 30), "bad arguments");
    *bytes = (int64_t)order_layout(n_events > 0 ? n_events : 1).bytes;
    return NERRF_OK;
}

extern "C" int nerrf_trace_stream_order_ex(int64_t n_events, const int64_t* ts_sec, const int32_t* ts_nanos, const uint32_t* pid,
                                           const uint16_t* source, int key_bits, const int64_t* path_off, double horizon,
                                           double* ts_out, int64_t* order_out, double* ts_sorted_out, int64_t* src_out,
                                           int64_t* res_path_off, int64_t* retain_out, int64_t* counts, void* workspace,
                                           int64_t workspace_bytes, void* stream) {
    NERRF_REQUIRE(counts, "null counts");
    counts[0] = counts[1] = counts[2] = 0;
    NERRF_REQUIRE(key_bits == 32 || (key_bits == 48 && source), "key_bits=%d: 32, or 48 with a source column", key_bits);
    NERRF_REQUIRE(n_events >= 0 && n_events < ((int64_t)1 << 30), "n_events=%lld out of range", (long long)n_events);
    if (n_events == 0) return NERRF_OK;
    NERRF_REQUIRE(ts_sec && ts_nanos && pid && path_off && ts_out && order_out && ts_sorted_out && src_out && res_path_off && workspace,
                  "null pointer");
    const OrderWs L = order_layout(n_events);
    NERRF_REQUIRE(workspace_bytes >= (int64_t)L.bytes, "workspace too small: %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)L.bytes);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    OrderArgs a;
    a.n = n_events; a.ts_sec = ts_sec; a.ts_nanos = ts_nanos; a.pid = pid; a.path_off = path_off; a.horizon = horizon;
    a.source = source; a.key_bits = key_bits;
    a.ts = ts_out; a.tord = (uint32_t*)(ws + L.tord); a.byp = (uint32_t*)(ws + L.byp);
    a.A = (int32_t*)(ws + L.A); a.G = (int32_t*)(ws + L.G); a.C = (int32_t*)(ws + L.C);
    a.F = (int32_t*)(ws + L.F); a.R = (int32_t*)(ws + L.R); a.L = (int32_t*)(ws + L.L); a.src = src_out;
    a.res_bytes = (unsigned long long*)(ws + L.totals + 16);               // after the three int32 scan totals
    uint64_t *ka = (uint64_t*)(ws + L.ka), *kb = (uint64_t*)(ws + L.kb);
    uint32_t *va = (uint32_t*)(ws + L.va), *vb = (uint32_t*)(ws + L.vb);
    int32_t* sums = (int32_t*)(ws + L.sums);
    int32_t* totals = (int32_t*)(ws + L.totals);
    const int grid = grid_for(n_events, 256);
    order_keys_kernel<<<grid, 256, 0, st>>>(a, ka, va);
    if (radix_sort_pairs(ka, kb, va, vb, n_events, 0, 64, ws + L.rs, st)) { uint64_t* t = ka; ka = kb; kb = t; uint32_t* u = va; va = vb; vb = u; }
    order_pid_keys_kernel<<<grid, 256, 0, st>>>(a, ka, va);
    if (radix_sort_pairs(ka, kb, va, vb, n_events, 0, key_bits, ws + L.rs, st)) { uint64_t* t = ka; ka = kb; kb = t; uint32_t* u = va; va = vb; vb = u; }
    order_segments_kernel<<<grid, 256, 0, st>>>(a, ka, va);
    inclusive_max_scan_i32(a.A, n_events, sums, st);
    inclusive_max_scan_i32(a.G, n_events, sums, st);
    inclusive_max_scan_i32(a.C, n_events, sums, st);
    order_resolve_kernel<<<grid, 256, 0, st>>>(a);
    order_flags_kernel<<<grid, 256, 0, st>>>(a);
    exclusive_scan_i32(a.F, n_events, sums, totals + 0, st);
    exclusive_scan_i32(a.R, n_events, sums, totals + 1, st);
    exclusive_scan_i32(a.L, n_events, sums, totals + 2, st);
    order_compact_kernel<<<grid, 256, 0, st>>>(a, totals, order_out, ts_sorted_out, retain_out, res_path_off);
    int rc = launch_status("stream order kernels");
    if (rc) return rc;
    struct { int32_t scan[4]; unsigned long long res_bytes; } h;
    NERRF_CHECK_CUDA(cudaMemcpyAsync(&h, totals, sizeof(h), cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    // the resolved path offsets come from an int32 scan: past 2^31 - 1 bytes they have wrapped and nothing may read them
    NERRF_REQUIRE(h.res_bytes < (1ull << 31),
                  "resolved paths of %llu bytes: at most 2^31 - 1 per stream (a path counts once for every path-less event "
                  "that resolves to it); compact the stream or split it", h.res_bytes);
    counts[0] = h.scan[0]; counts[1] = h.scan[1]; counts[2] = h.scan[2];
    return NERRF_OK;
}

extern "C" int nerrf_trace_stream_order(int64_t n_events, const int64_t* ts_sec, const int32_t* ts_nanos, const uint32_t* pid,
                                        const int64_t* path_off, double horizon, double* ts_out, int64_t* order_out,
                                        double* ts_sorted_out, int64_t* src_out, int64_t* res_path_off, int64_t* retain_out,
                                        int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream) {
    return nerrf_trace_stream_order_ex(n_events, ts_sec, ts_nanos, pid, nullptr, 32, path_off, horizon, ts_out, order_out,
                                       ts_sorted_out, src_out, res_path_off, retain_out, counts, workspace, workspace_bytes, stream);
}

extern "C" int nerrf_trace_stream_columns(int64_t n_events, const int64_t* src, const int64_t* path_off, const uint8_t* path_data,
                                          const uint8_t* path_flags, const int64_t* new_path_off, const uint8_t* new_path_data,
                                          const uint8_t* event_slot, const uint8_t* slot_map, const int64_t* res_path_off,
                                          int merge_renames, uint8_t* res_path_data, uint8_t* pf_out, uint8_t* pf_raw_out,
                                          uint8_t* slot_out, void* stream) {
    NERRF_REQUIRE(n_events >= 0, "negative event count");
    if (n_events == 0) return NERRF_OK;
    NERRF_REQUIRE(src && path_off && path_data && path_flags && new_path_off && new_path_data && event_slot && res_path_off &&
                      res_path_data && pf_out && pf_raw_out && slot_out,
                  "null pointer");
    stream_columns_kernel<<<grid_for(n_events, 8), 256, 0, (cudaStream_t)stream>>>(
        n_events, src, path_off, path_data, path_flags, new_path_off, new_path_data, event_slot, slot_map, res_path_off,
        merge_renames ? 1 : 0, res_path_data, pf_out, pf_raw_out, slot_out);
    return launch_status("stream_columns_kernel");
}

extern "C" int nerrf_trace_gather_rows_workspace_bytes(int64_t n_rows, int64_t* bytes) {
    return nerrf_trace_decode_device_workspace_bytes(n_rows, bytes);
}

extern "C" int nerrf_trace_gather_rows_ex(void* const* cols_in, const uint16_t* source_in, const int64_t* rows, int64_t n_rows,
                                          void* const* cols_out, uint16_t* source_out, void* workspace, int64_t workspace_bytes,
                                          void* stream) {
    NERRF_REQUIRE(n_rows >= 0 && n_rows < ((int64_t)1 << 28), "bad row count");
    NERRF_REQUIRE(cols_ok(cols_in) && cols_ok(cols_out), "null column pointer");
    cudaStream_t st = (cudaStream_t)stream;
    Cols in = make_cols(cols_in), out = make_cols(cols_out);
    in.source = (uint16_t*)source_in; out.source = source_out;
    for (int q = 0; q < 4; ++q) NERRF_CHECK_CUDA(cudaMemsetAsync(out.off[q], 0, 8, st));
    if (n_rows == 0) return NERRF_OK;
    NERRF_REQUIRE(rows && workspace, "null pointer");
    const DecodeWs L = decode_layout(n_rows);
    NERRF_REQUIRE(workspace_bytes >= (int64_t)L.bytes, "workspace too small: %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)L.bytes);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    char* ws = (char*)workspace;
    int64_t* start = (int64_t*)(ws + L.start);
    int32_t* scan = (int32_t*)(ws + L.scan);
    int32_t* total = (int32_t*)(ws + L.total);
    gather_scalars_kernel<<<grid_for(n_rows, 256), 256, 0, st>>>(in, rows, n_rows, out, start, scan);
    exclusive_scan_i32(scan, 4 * n_rows, (int32_t*)(ws + L.sums), total, st);
    StrSrc s;
    for (int q = 0; q < 4; ++q) s.base[q] = in.data[q];
    copy_strings_kernel<<<grid_for(n_rows, 8), 256, 0, st>>>(s, start, scan, total, n_rows, 0, out, nullptr);
    return launch_status("gather kernels");
}

extern "C" int nerrf_trace_gather_rows(void* const* cols_in, const int64_t* rows, int64_t n_rows, void* const* cols_out,
                                       void* workspace, int64_t workspace_bytes, void* stream) {
    return nerrf_trace_gather_rows_ex(cols_in, nullptr, rows, n_rows, cols_out, nullptr, workspace, workspace_bytes, stream);
}
