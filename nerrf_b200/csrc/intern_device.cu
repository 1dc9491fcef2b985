// Node interning ON THE DEVICE: "node merging (inode deduplication)" of the temporal-graph constructor
// (docs/content/docs/architecture.mdx:39-41; SURVEY.md 8f rank 1 "inode/path dedup via hash").  Same nodes, same
// numbering, same names as the host routine nerrf_trace_intern (csrc/ingest.cu) -- the spec -- for events given in
// processing (time) order, but as data-parallel passes over the event columns resident in HBM:
//
//   1  hash     thread per event: 64-bit hash of the pid, of the path's merge key (the path without its last extension when
//               merge_renames, the whole path otherwise) and of the rename target's; find-or-insert into an open-addressing
//               table (atomicCAS on the 64-bit key); every key keeps its FIRST MENTION = min over 2*event + role
//               (role 0 = path, 1 = rename target) with atomicMin -- order-independent, hence deterministic
//   2  verify   thread per mention: the bytes of the key equal the bytes of the key's first mention (a 64-bit collision
//               would otherwise merge two files silently; it raises an error instead)
//   3  roots    the host loop binds a key at its first mention: as a path it makes a node, as a rename target
//               (merge_renames) it aliases the node of the same event's path.  First mentions are final after pass 1, so
//               "alias of" is a static forest; every key follows its parents to the root (chains = rename chains)
//   4  number   nodes are numbered in order of first appearance over the interleaved (pid, path, target) mentions:
//               flag the creating mentions in a [3n] array, exclusive scan (own kernels), node id = scan value
//   5  assign   per event: node_p / node_f / node_g; per node: kind, naming event (the creation, overridden by the LAST event
//               that touches the node under a name ending in ".lockbit3" -- atomicMax over 2*event + which)
//
// Bound: HBM / L2 latency of the table probes; ~100 B of traffic per event.  No string ever goes back to the host.
#include "common.cuh"
#include "scan.cuh"

namespace nerrf {
namespace {

constexpr uint64_t FNV_OFF = 0xcbf29ce484222325ull, FNV_PRIME = 0x100000001b3ull;

__device__ __forceinline__ uint64_t mix64(uint64_t h) {      // murmur3 finaliser: avalanche, then never 0 (0 = empty slot)
    h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
    return h ? h : 1ull;
}
__device__ __forceinline__ uint64_t hash_bytes(const uint8_t* __restrict__ s, int64_t n) {
    uint64_t h = FNV_OFF ^ (uint64_t)n;
    for (int64_t i = 0; i < n; ++i) { h ^= s[i]; h *= FNV_PRIME; }
    return mix64(h);
}
// source-qualified key and name hashes: the identity at source 0, so a single-source stream hashes as it always did
__device__ __forceinline__ uint64_t qualify(uint64_t h, uint32_t s) { return s ? mix64(h + (uint64_t)s * 0x9E3779B97F4A7C15ull) : h; }
__device__ __forceinline__ uint64_t pid_hash(uint32_t pid, uint32_t s) { return mix64((((uint64_t)s << 32) | pid) + 0x9E3779B97F4A7C15ull); }
__device__ __forceinline__ uint32_t source_at(const uint16_t* __restrict__ source, int64_t i) { return source ? source[i] : 0u; }
// csrc/ingest.cu stem_len: the path without its last extension (graph.py _stem)
__device__ __forceinline__ int64_t stem_len_dev(const uint8_t* __restrict__ s, int64_t n) {
    int64_t slash = -1, dot = -1;
    for (int64_t i = n - 1; i >= 0; --i) {
        if (s[i] == '.' && dot < 0) dot = i;
        if (s[i] == '/') { slash = i; break; }
    }
    return (dot > slash) ? dot : n;
}
__device__ __forceinline__ bool ends_lockbit3(const uint8_t* __restrict__ s, int64_t n) {
    const char suf[9] = {'.', 'l', 'o', 'c', 'k', 'b', 'i', 't', '3'};
    if (n < 9) return false;
    for (int k = 0; k < 9; ++k)
        if (s[n - 9 + k] != (uint8_t)suf[k]) return false;
    return true;
}

struct Table {
    unsigned long long* key;    // 0 = empty
    int32_t* first;             // first mention (file keys: 2*event + role; pids: event), INT_MAX = none yet
    uint32_t mask;
};
__device__ __forceinline__ int32_t table_insert(const Table t, uint64_t h, int32_t mention) {
    uint32_t s = (uint32_t)(h >> 17) & t.mask;
    for (uint32_t probe = 0; probe <= t.mask; ++probe) {
        const unsigned long long prev = atomicCAS(t.key + s, 0ull, (unsigned long long)h);
        if (prev == 0ull || prev == h) { atomicMin(t.first + s, mention); return (int32_t)s; }
        s = (s + 1) & t.mask;
    }
    return -1;                                                   // table full (cannot happen: capacity >= 2x the keys)
}

struct InternArgs {
    int64_t n;                             // events processed (ranks 0..n-1)
    int64_t n_total;                       // events stored (the columns' length): order[] indexes into [0, n_total)
    const int64_t* order;                  // processing order: rank k handles stored event order[k] (NULL: identity)
    const uint32_t* pid;
    const uint16_t* source;                // NULL: every event from source 0
    const int64_t *path_off, *gpath_off;
    const uint8_t *path_data, *gpath_data;
    int merge;
    Table files, pids;
    int32_t *slot_p, *slot_f, *slot_g;     // [n] BY RANK: table slots of the event's keys (slot_g = -1: no rename target)
    int32_t* flags;                        // [3n] creating mentions -> exclusive scan in place
    int32_t* err;                          // [0] != 0: 1 = table full, 2 = hash collision, 3 = node capacity
    int32_t *node_p, *node_f, *node_g;     // [n] by STORED event index, like the host routine
    int8_t* kind;
    int64_t* name_event;
    int8_t* name_which;
    long long* name_code;                  // [cap] -1, or max over renaming mentions of 2*event + which
    int64_t cap;
};

__device__ __forceinline__ int64_t stored(const InternArgs& a, int64_t k) { return a.order ? a.order[k] : k; }

// mentions are numbered by RANK k (processing order); the data of rank k is stored event stored(a, k)
__global__ void __launch_bounds__(256) intern_hash_kernel(InternArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        const int64_t i = stored(a, k);
        if (i < 0 || i >= a.n_total) { *a.err = 4; a.slot_p[k] = a.slot_f[k] = 0; a.slot_g[k] = -1; continue; }
        const uint32_t src = source_at(a.source, i);
        const int32_t sp = table_insert(a.pids, pid_hash(a.pid[i], src), (int32_t)k);
        const uint8_t* s = a.path_data + a.path_off[i];
        const int64_t n = a.path_off[i + 1] - a.path_off[i];
        const int32_t sf = table_insert(a.files, qualify(hash_bytes(s, a.merge ? stem_len_dev(s, n) : n), src), (int32_t)(2 * k));
        int32_t sg = -1;
        const int64_t gn = a.gpath_off[i + 1] - a.gpath_off[i];
        if (gn > 0) {
            const uint8_t* g = a.gpath_data + a.gpath_off[i];
            sg = table_insert(a.files, qualify(hash_bytes(g, a.merge ? stem_len_dev(g, gn) : gn), src), (int32_t)(2 * k + 1));
            if (sg < 0) *a.err = 1;
        }
        if (sp < 0 || sf < 0) *a.err = 1;
        a.slot_p[k] = sp; a.slot_f[k] = sf; a.slot_g[k] = sg;
    }
}

// key bytes of mention m (2*event + role)
__device__ __forceinline__ const uint8_t* mention_key(const InternArgs& a, int32_t m, int64_t* len) {
    const int64_t e = stored(a, m >> 1);
    const uint8_t* s; int64_t n;
    if (m & 1) { s = a.gpath_data + a.gpath_off[e]; n = a.gpath_off[e + 1] - a.gpath_off[e]; }
    else { s = a.path_data + a.path_off[e]; n = a.path_off[e + 1] - a.path_off[e]; }
    *len = a.merge ? stem_len_dev(s, n) : n;
    return s;
}
__device__ __forceinline__ void verify_mention(const InternArgs& a, int32_t slot, int32_t m) {
    const int32_t f = a.files.first[slot];
    if (f == m) return;
    int64_t n0, n1;
    const uint8_t* s0 = mention_key(a, f, &n0);
    const uint8_t* s1 = mention_key(a, m, &n1);
    bool same = n0 == n1 && source_at(a.source, stored(a, f >> 1)) == source_at(a.source, stored(a, m >> 1));
    for (int64_t k = 0; same && k < n0; ++k) same = s0[k] == s1[k];
    if (!same) *a.err = 2;
}
__global__ void __launch_bounds__(256) intern_verify_kernel(InternArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (*a.err) return;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        const int32_t pf = a.pids.first[a.slot_p[k]];
        if (pf != (int32_t)k && (a.pid[stored(a, pf)] != a.pid[stored(a, k)] ||
                                 source_at(a.source, stored(a, pf)) != source_at(a.source, stored(a, k))))
            *a.err = 2;
        verify_mention(a, a.slot_f[k], (int32_t)(2 * k));
        if (a.slot_g[k] >= 0) verify_mention(a, a.slot_g[k], (int32_t)(2 * k + 1));
    }
}

// root of a file key: follow "first mentioned as the rename target of event e -> the path key of e" to a key that was
// first mentioned as a path (it made the node).  Non-merge mode: every key is its own root.
__device__ __forceinline__ int32_t root_of(const InternArgs& a, int32_t slot) {
    if (!a.merge) return slot;
    for (int hop = 0; hop < (1 << 20); ++hop) {
        const int32_t f = a.files.first[slot];
        if (!(f & 1)) return slot;
        slot = a.slot_f[f >> 1];                                  // strictly earlier first mention: the walk terminates
    }
    return slot;
}

__global__ void __launch_bounds__(256) intern_flags_kernel(InternArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (*a.err) return;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
        a.flags[3 * i] = a.pids.first[a.slot_p[i]] == (int32_t)i;
        a.flags[3 * i + 1] = a.files.first[a.slot_f[i]] == (int32_t)(2 * i);
        a.flags[3 * i + 2] = (!a.merge && a.slot_g[i] >= 0 && a.files.first[a.slot_g[i]] == (int32_t)(2 * i + 1)) ? 1 : 0;
    }
}

// node id of the node made by creating mention c (index into the [3n] scan)
__global__ void __launch_bounds__(256) intern_assign_kernel(InternArgs a, const int32_t* __restrict__ total) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t N = *total;
    if (*a.err) return;
    if (N > a.cap) { if (blockIdx.x == 0 && threadIdx.x == 0) *a.err = 3; return; }
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) {
        const int64_t i = stored(a, k);
        const int32_t pe = a.pids.first[a.slot_p[k]];
        const int32_t np_ = a.flags[3 * (int64_t)pe];
        a.node_p[i] = np_;
        if (pe == (int32_t)k) { a.kind[np_] = 1; a.name_event[np_] = i; a.name_which[np_] = 2; }
        const int32_t rf = root_of(a, a.slot_f[k]);
        const int32_t ff = a.files.first[rf];
        const int32_t nf = a.flags[3 * (int64_t)(ff >> 1) + 1 + (ff & 1)];
        a.node_f[i] = nf;
        if (ff == (int32_t)(2 * k)) { a.kind[nf] = 0; a.name_event[nf] = i; a.name_which[nf] = 0; }
        const uint8_t* s = a.path_data + a.path_off[i];
        if (ends_lockbit3(s, a.path_off[i + 1] - a.path_off[i])) atomicMax(a.name_code + nf, (long long)(2 * k));
        int32_t ng = -1;
        const int32_t sg = a.slot_g[k];
        if (sg >= 0) {
            const uint8_t* g = a.gpath_data + a.gpath_off[i];
            const int64_t gn = a.gpath_off[i + 1] - a.gpath_off[i];
            if (a.merge) {
                if (ends_lockbit3(g, gn)) atomicMax(a.name_code + nf, (long long)(2 * k + 1));   // the rollback target's name
            } else {
                const int32_t fg = a.files.first[sg];
                ng = a.flags[3 * (int64_t)(fg >> 1) + 1 + (fg & 1)];
                if (fg == (int32_t)(2 * k + 1)) { a.kind[ng] = 0; a.name_event[ng] = i; a.name_which[ng] = 1; }
            }
        }
        a.node_g[i] = ng;
    }
}
__global__ void __launch_bounds__(256) intern_names_kernel(InternArgs a, const int32_t* __restrict__ total) {
    const int64_t N = *total < a.cap ? *total : a.cap;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (*a.err) return;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < N; v += stride) {
        const long long c = a.name_code[v];
        if (c >= 0) { a.name_event[v] = stored(a, c >> 1); a.name_which[v] = (int8_t)(c & 1); }
    }
}

// 64-bit hash of every node's NAME (the string its naming event gives it; pid nodes: their pid): lets a caller match
// nodes against a set of names (e.g. the files an earlier tick already reverted) without bringing a million strings
// to the host.  Same function as nerrf_b200/ingest.py name_hash.
__global__ void __launch_bounds__(256) name_hash_kernel(int64_t n_nodes, const int64_t* __restrict__ name_event,
                                                        const int8_t* __restrict__ name_which, const uint32_t* __restrict__ pid,
                                                        const uint16_t* __restrict__ source, const int64_t* __restrict__ path_off, const uint8_t* __restrict__ path_data,
                                                        const int64_t* __restrict__ gpath_off, const uint8_t* __restrict__ gpath_data,
                                                        unsigned long long* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_nodes; v += stride) {
        const int64_t e = name_event[v];
        const int w = name_which[v];
        const uint32_t src = source_at(source, e);
        unsigned long long h;
        if (w == 2) h = pid_hash(pid[e], src);
        else if (w == 1) h = qualify(hash_bytes(gpath_data + gpath_off[e], gpath_off[e + 1] - gpath_off[e]), src);
        else h = qualify(hash_bytes(path_data + path_off[e], path_off[e + 1] - path_off[e]), src);
        out[v] = h;
    }
}

// 64-bit hash of every node's parent DIRECTORY: the name hash of the bytes of its name up to (not including) the last
// '/' (no '/': the empty string); pid nodes hash their pid as in name_hash_kernel.  Groups file nodes by directory for the
// planner's "restore from backup" candidates.  Same function as nerrf_b200/stream.py dir_hash.
__device__ __forceinline__ int64_t dir_len_dev(const uint8_t* __restrict__ s, int64_t n) {
    for (int64_t i = n - 1; i >= 0; --i)
        if (s[i] == '/') return i;
    return 0;
}
__global__ void __launch_bounds__(256) dir_hash_kernel(int64_t n_nodes, const int64_t* __restrict__ name_event,
                                                       const int8_t* __restrict__ name_which, const uint32_t* __restrict__ pid,
                                                       const uint16_t* __restrict__ source, const int64_t* __restrict__ path_off, const uint8_t* __restrict__ path_data,
                                                       const int64_t* __restrict__ gpath_off, const uint8_t* __restrict__ gpath_data,
                                                       unsigned long long* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_nodes; v += stride) {
        const int64_t e = name_event[v];
        const int w = name_which[v];
        const uint32_t src = source_at(source, e);
        unsigned long long h;
        if (w == 2) {
            h = pid_hash(pid[e], src);
        } else {
            const uint8_t* s = w == 1 ? gpath_data + gpath_off[e] : path_data + path_off[e];
            const int64_t n = w == 1 ? gpath_off[e + 1] - gpath_off[e] : path_off[e + 1] - path_off[e];
            h = qualify(hash_bytes(s, dir_len_dev(s, n)), src);
        }
        out[v] = h;
    }
}

struct InternWs {
    size_t fkey, ffirst, pkey, pfirst, slot_p, slot_f, slot_g, flags, sums, total, err, name_code, bytes;
    uint32_t fcap, pcap;
    int64_t nb;
};
inline size_t up256i(size_t x) { return (x + 255) & ~(size_t)255; }
InternWs intern_layout(int64_t n, int64_t cap) {
    InternWs L;
    uint64_t fc = 1024, pc = 1024;
    while (fc < (uint64_t)(4 * n)) fc <<= 1;                      // <= 2n file keys: load factor <= 1/2
    while (pc < (uint64_t)(2 * n)) pc <<= 1;
    L.fcap = (uint32_t)fc; L.pcap = (uint32_t)pc;
    L.nb = (3 * n + SCAN_TILE - 1) / SCAN_TILE;
    size_t o = 0;
    L.fkey = o; o += up256i(fc * 8);
    L.ffirst = o; o += up256i(fc * 4);
    L.pkey = o; o += up256i(pc * 8);
    L.pfirst = o; o += up256i(pc * 4);
    L.slot_p = o; o += up256i((size_t)n * 4);
    L.slot_f = o; o += up256i((size_t)n * 4);
    L.slot_g = o; o += up256i((size_t)n * 4);
    L.flags = o; o += up256i((size_t)3 * n * 4 + 16);
    L.sums = o; o += up256i((size_t)(L.nb + 1) * 4);
    L.total = o; o += 256;
    L.err = o; o += 256;
    L.name_code = o; o += up256i((size_t)cap * 8);
    L.bytes = o;
    return L;
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_trace_intern_device_workspace_bytes(int64_t n_events, int64_t node_capacity, int64_t* bytes) {
    NERRF_REQUIRE(bytes && n_events >= 0 && n_events < ((int64_t)1 << 29) && node_capacity >= 0, "bad arguments");
    *bytes = (int64_t)intern_layout(n_events > 0 ? n_events : 1, node_capacity).bytes;
    return NERRF_OK;
}

extern "C" int nerrf_trace_intern_device_ex(int64_t n_events, int64_t n_stored, const int64_t* order, const uint32_t* pid,
                                            const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                                            const int64_t* new_path_off, const uint8_t* new_path_data, int merge_renames,
                                            int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes, int8_t* node_kind,
                                            int64_t* node_name_event, int8_t* node_name_which, int64_t node_capacity,
                                            void* workspace, int64_t workspace_bytes, void* stream) {
    NERRF_REQUIRE(n_nodes, "null n_nodes");
    *n_nodes = 0;
    if (n_events == 0) return NERRF_OK;
    NERRF_REQUIRE(n_events > 0 && n_events < ((int64_t)1 << 29), "n_events=%lld out of range", (long long)n_events);
    NERRF_REQUIRE(n_stored >= n_events || (order && n_stored >= 1), "n_stored=%lld < n_events without an order", (long long)n_stored);
    NERRF_REQUIRE(pid && path_off && path_data && new_path_off && new_path_data && node_p && node_f && node_g && node_kind &&
                      node_name_event && node_name_which && workspace,
                  "null pointer");
    const InternWs L = intern_layout(n_events, node_capacity);
    NERRF_REQUIRE(workspace_bytes >= (int64_t)L.bytes, "workspace too small: %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)L.bytes);
    NERRF_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    InternArgs a;
    a.n = n_events; a.n_total = n_stored; a.order = order; a.pid = pid; a.source = source; a.path_off = path_off; a.gpath_off = new_path_off; a.path_data = path_data; a.gpath_data = new_path_data;
    a.merge = merge_renames ? 1 : 0;
    a.files.key = (unsigned long long*)(ws + L.fkey); a.files.first = (int32_t*)(ws + L.ffirst); a.files.mask = L.fcap - 1;
    a.pids.key = (unsigned long long*)(ws + L.pkey); a.pids.first = (int32_t*)(ws + L.pfirst); a.pids.mask = L.pcap - 1;
    a.slot_p = (int32_t*)(ws + L.slot_p); a.slot_f = (int32_t*)(ws + L.slot_f); a.slot_g = (int32_t*)(ws + L.slot_g);
    a.flags = (int32_t*)(ws + L.flags); a.err = (int32_t*)(ws + L.err);
    a.node_p = node_p; a.node_f = node_f; a.node_g = node_g; a.kind = node_kind; a.name_event = node_name_event;
    a.name_which = node_name_which; a.name_code = (long long*)(ws + L.name_code); a.cap = node_capacity;
    int32_t* sums = (int32_t*)(ws + L.sums);
    int32_t* total = (int32_t*)(ws + L.total);
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.fkey, 0, (size_t)L.fcap * 8, st));
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.ffirst, 0x7f, (size_t)L.fcap * 4, st));      // 0x7f7f7f7f > any mention index
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.pkey, 0, (size_t)L.pcap * 8, st));
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.pfirst, 0x7f, (size_t)L.pcap * 4, st));
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.err, 0, 4, st));
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.name_code, 0xff, (size_t)node_capacity * 8, st));
    const int grid = sm_count() * 8;
    intern_hash_kernel<<<grid, 256, 0, st>>>(a);
    intern_verify_kernel<<<grid, 256, 0, st>>>(a);
    intern_flags_kernel<<<grid, 256, 0, st>>>(a);
    const int64_t m = 3 * n_events;
    exclusive_scan_i32(a.flags, m, sums, total, st);
    intern_assign_kernel<<<grid, 256, 0, st>>>(a, total);
    intern_names_kernel<<<grid, 256, 0, st>>>(a, total);
    int rc = launch_status("device interning kernels");
    if (rc) return rc;
    int32_t h[2] = {0, 0};
    NERRF_CHECK_CUDA(cudaMemcpyAsync(&h[0], total, 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(&h[1], a.err, 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    NERRF_REQUIRE(h[1] != 4, "order[] holds an index outside [0, n_stored)");
    NERRF_REQUIRE(h[1] != 1, "interning table full (internal sizing error)");
    NERRF_REQUIRE(h[1] != 2, "64-bit hash collision between two different paths: use the host interning for this batch");
    NERRF_REQUIRE(h[1] != 3 && h[0] <= node_capacity, "node_capacity=%lld too small (%d nodes)", (long long)node_capacity, h[0]);
    *n_nodes = h[0];
    return NERRF_OK;
}

extern "C" int nerrf_trace_intern_device(int64_t n_events, int64_t n_stored, const int64_t* order, const uint32_t* pid, const int64_t* path_off, const uint8_t* path_data,
                                         const int64_t* new_path_off, const uint8_t* new_path_data, int merge_renames,
                                         int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes, int8_t* node_kind,
                                         int64_t* node_name_event, int8_t* node_name_which, int64_t node_capacity,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
    return nerrf_trace_intern_device_ex(n_events, n_stored, order, pid, nullptr, path_off, path_data, new_path_off, new_path_data,
                                        merge_renames, node_p, node_f, node_g, n_nodes, node_kind, node_name_event, node_name_which,
                                        node_capacity, workspace, workspace_bytes, stream);
}

extern "C" int nerrf_trace_name_hash_ex(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                                        const uint32_t* pid, const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                                        const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream) {
    NERRF_REQUIRE(n_nodes >= 0, "negative node count");
    if (n_nodes == 0) return NERRF_OK;
    NERRF_REQUIRE(node_name_event && node_name_which && pid && path_off && path_data && new_path_off && new_path_data && hash_out,
                  "null pointer");
    name_hash_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(n_nodes, node_name_event, node_name_which, pid, source, path_off,
                                                                        path_data, new_path_off, new_path_data, (unsigned long long*)hash_out);
    return launch_status("name_hash_kernel");
}

extern "C" int nerrf_trace_name_hash(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                                     const uint32_t* pid, const int64_t* path_off, const uint8_t* path_data,
                                     const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream) {
    return nerrf_trace_name_hash_ex(n_nodes, node_name_event, node_name_which, pid, nullptr, path_off, path_data, new_path_off,
                                    new_path_data, hash_out, stream);
}

extern "C" int nerrf_trace_dir_hash_ex(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                                       const uint32_t* pid, const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                                       const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream) {
    NERRF_REQUIRE(n_nodes >= 0, "negative node count");
    if (n_nodes == 0) return NERRF_OK;
    NERRF_REQUIRE(node_name_event && node_name_which && pid && path_off && path_data && new_path_off && new_path_data && hash_out,
                  "null pointer");
    dir_hash_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(n_nodes, node_name_event, node_name_which, pid, source, path_off,
                                                                       path_data, new_path_off, new_path_data, (unsigned long long*)hash_out);
    return launch_status("dir_hash_kernel");
}

extern "C" int nerrf_trace_dir_hash(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                                    const uint32_t* pid, const int64_t* path_off, const uint8_t* path_data,
                                    const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream) {
    return nerrf_trace_dir_hash_ex(n_nodes, node_name_event, node_name_which, pid, nullptr, path_off, path_data, new_path_off,
                                   new_path_data, hash_out, stream);
}
