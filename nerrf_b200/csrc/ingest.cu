// nerrf.trace.EventBatch ingest (SURVEY.md 8f rank 2): protobuf wire bytes -> columnar arrays, plus the
// pid / path interning ("inode dedup") the graph constructor needs.  HOST code (no kernels): it is the data format
// on the input side of the hot path, native like the rest of the boundary, compiled into the same C-ABI library.
//
// Wire schema = proto/trace.proto:11-49 (Event: ts=1 Timestamp{seconds=1, nanos=2}, pid=2, tid=3, comm=4,
// syscall=5, path=6, new_path=7, flags=8 enum, ret_val=9 sint64, bytes=10, inode=11, mode=12, uid=13, gid=14,
// dependencies=15) and :47-49 (EventBatch: repeated Event events=1).  Producer: tracker/cmd/tracker/main.go:229-252.
// Concatenated serialized EventBatch messages are one valid EventBatch (repeated fields append), so a client that
// buffers the gRPC stream hands the bytes over unchanged.  Unknown fields are skipped by wire type.
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <string.h>
#include <string>
#include <unordered_map>
#include <vector>
#include "common.cuh"
#include "wire.cuh"

namespace nerrf {
namespace {

using wire::EventView;
using wire::Reader;

// calls f(EventView&) for every Event of the batch; returns the byte offset of the first malformed record or -1
template <typename Fn>
int64_t for_each_event(const uint8_t* buf, int64_t len, Fn&& f) {
    Reader r{buf, buf + len};
    while (r.p < r.end) {
        const uint8_t* at = r.p;
        bool event; const uint8_t* s; uint64_t n;
        if (!wire::next_record(&r, &event, &s, &n)) return at - buf;
        if (event) {
            EventView e;
            if (!wire::parse_event(s, n, &e)) return at - buf;
            f(e);
        }
    }
    return -1;
}

// merge key of a file and its renamed / encrypted twin: the path without its last extension (graph.py _stem)
uint64_t stem_len(const uint8_t* s, uint64_t n) {
    int64_t slash = -1, dot = -1;
    for (int64_t i = (int64_t)n - 1; i >= 0; --i) {
        if (s[i] == '.' && dot < 0) dot = i;
        if (s[i] == '/') { slash = i; break; }
    }
    return (dot > slash) ? (uint64_t)dot : n;
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_trace_scan(const uint8_t* buf, int64_t len, int64_t* n_events, int64_t* string_bytes) {
    NERRF_REQUIRE((buf != nullptr || len == 0) && len >= 0, "null buffer");
    NERRF_REQUIRE(n_events && string_bytes, "null output");
    // top-level hop only (tag + length per Event): the Events themselves are parsed once, by nerrf_trace_decode.
    // string_bytes[k] is therefore an UPPER BOUND for column k (no string column can exceed the Event payload bytes).
    int64_t n = 0, payload = 0;
    Reader r{buf, buf + len};
    while (r.p < r.end) {
        const uint8_t* at = r.p;
        uint64_t tag, m; const uint8_t* s;
        bool ok = r.varint(&tag);
        if (ok && (tag >> 3) == 1 && (tag & 7) == 2) { ok = r.len_delim(&s, &m); ++n; payload += (int64_t)m; }
        else if (ok) ok = r.skip((uint32_t)(tag & 7));
        NERRF_REQUIRE(ok, "malformed EventBatch at byte offset %lld", (long long)(at - buf));
    }
    *n_events = n;
    for (int i = 0; i < 4; ++i) string_bytes[i] = payload;
    return NERRF_OK;
}

// top-level varint for the framing walk: 1 = read, 0 = the bytes ran out first (cut off), -1 = more than 10 bytes
static int frame_varint(const uint8_t** p, const uint8_t* end, uint64_t* v) {
    uint64_t r = 0;
    for (int shift = 0; shift < 70; shift += 7) {
        if (*p >= end) return 0;
        const uint8_t b = *(*p)++;
        if (shift < 64) r |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) { *v = r; return 1; }
    }
    return -1;
}

extern "C" int nerrf_trace_frame(const uint8_t* buf, int64_t len, int partial, int64_t max_records, int64_t* rec_at,
                                 int64_t* body_off, int64_t* body_len, int64_t* n_records, int64_t* consumed) {
    NERRF_REQUIRE((buf != nullptr || len == 0) && len >= 0 && max_records >= 0, "bad buffer");
    NERRF_REQUIRE(n_records && consumed && (max_records == 0 || (rec_at && body_off && body_len)), "null output");
    // the walk of for_each_event (tag + length per record, unknown fields skipped by wire type) without parsing the Events
    const uint8_t* p = buf;
    const uint8_t* end = buf + len;
    int64_t n = 0;
    int state = 1;                                          // 1 ok, 0 cut off, -1 malformed
    const uint8_t* at = p;
    while (p < end) {
        at = p;
        uint64_t tag, m = 0;
        state = frame_varint(&p, end, &tag);
        if (state < 1) break;
        const uint32_t wt = (uint32_t)(tag & 7);
        const bool event = (tag >> 3) == 1 && wt == 2;
        if (wt == 0) state = frame_varint(&p, end, &m);
        else if (wt == 1 || wt == 5) { const int64_t w = wt == 1 ? 8 : 4; state = end - p < w ? 0 : 1; if (state) p += w; }
        else if (wt == 2) {
            state = frame_varint(&p, end, &m);
            if (state == 1 && m > (uint64_t)(end - p)) state = 0;
        } else state = -1;                                  // groups are malformed
        if (state < 1) break;
        if (event) {
            if (n < max_records) { rec_at[n] = at - buf; body_off[n] = p - buf; body_len[n] = (int64_t)m; }
            ++n;
        }
        if (wt == 2) p += m;
    }
    *n_records = n;
    *consumed = (state == 1 ? p : at) - buf;
    // a malformed record, or (whole-buffer mode) a cut-off one: the outputs still describe the records before it
    NERRF_REQUIRE(state == 1 || (state == 0 && partial), "malformed EventBatch at byte offset %lld", (long long)(at - buf));
    return NERRF_OK;
}

extern "C" int nerrf_trace_decode(const uint8_t* buf, int64_t len, int64_t n_events, int64_t* ts_sec, int32_t* ts_nanos,
                                  uint32_t* pid, uint32_t* tid, int32_t* flags, int64_t* ret_val, uint64_t* bytes,
                                  uint8_t* event_slot_out, uint8_t* path_flags, int64_t* comm_off, uint8_t* comm_data,
                                  int64_t* syscall_off, uint8_t* syscall_data, int64_t* path_off, uint8_t* path_data,
                                  int64_t* new_path_off, uint8_t* new_path_data) {
    NERRF_REQUIRE((buf != nullptr || len == 0) && len >= 0 && n_events >= 0, "bad buffer");
    NERRF_REQUIRE(ts_sec && ts_nanos && pid && tid && flags && ret_val && bytes && event_slot_out && path_flags,
                  "null scalar column");
    NERRF_REQUIRE(comm_off && syscall_off && path_off && new_path_off, "null offsets column");
    int64_t i = 0, o[4] = {0, 0, 0, 0};
    bool overflow = false;
    comm_off[0] = syscall_off[0] = path_off[0] = new_path_off[0] = 0;
    auto put = [](uint8_t* dst, int64_t* off, int64_t i, int64_t* cursor, const uint8_t* s, uint64_t n) {
        if (n) memcpy(dst + *cursor, s, n);
        *cursor += (int64_t)n;
        off[i + 1] = *cursor;
    };
    const int64_t bad = for_each_event(buf, len, [&](const EventView& e) {
        if (i >= n_events) { overflow = true; return; }
        ts_sec[i] = e.ts_sec; ts_nanos[i] = e.ts_nanos; pid[i] = e.pid; tid[i] = e.tid; flags[i] = e.flags;
        ret_val[i] = e.ret_val; bytes[i] = e.bytes;
        event_slot_out[i] = (uint8_t)wire::event_slot(e.syscall, e.syscall_n);
        path_flags[i] = wire::path_flags(e.path, e.path_n);
        put(comm_data, comm_off, i, &o[0], e.comm, e.comm_n);
        put(syscall_data, syscall_off, i, &o[1], e.syscall, e.syscall_n);
        put(path_data, path_off, i, &o[2], e.path, e.path_n);
        put(new_path_data, new_path_off, i, &o[3], e.new_path, e.new_path_n);
        ++i;
    });
    NERRF_REQUIRE(bad < 0, "malformed EventBatch at byte offset %lld", (long long)bad);
    NERRF_REQUIRE(!overflow && i == n_events, "n_events=%lld does not match the buffer (nerrf_trace_scan)", (long long)n_events);
    return NERRF_OK;
}

// NERRF_PATH_* bits of every string of a packed string column (same rules as the path_flags column of
// nerrf_trace_decode); used for new_path, whose flags the decoder does not emit.
extern "C" int nerrf_trace_path_flags(const int64_t* off, const uint8_t* data, int64_t n, uint8_t* flags_out) {
    NERRF_REQUIRE(n >= 0 && off && flags_out && (data || n == 0 || off[n] == 0), "null pointer");
    for (int64_t i = 0; i < n; ++i) {
        NERRF_REQUIRE(off[i + 1] >= off[i], "offsets must be non-decreasing (string %lld)", (long long)i);
        const uint8_t* s = data + off[i];
        const uint64_t m = (uint64_t)(off[i + 1] - off[i]);
        flags_out[i] = wire::path_flags(s, m);
    }
    return NERRF_OK;
}

// information-flow class of every event (wire::flow_class; DESIGN.md 1.5) from host columns
extern "C" int nerrf_trace_flow_class(const uint8_t* event_slot, const int64_t* flags, const int64_t* ret_val, int64_t n,
                                      uint8_t* flow_out) {
    NERRF_REQUIRE(n >= 0 && (n == 0 || (event_slot && flags && ret_val && flow_out)), "null pointer");
    for (int64_t i = 0; i < n; ++i) flow_out[i] = wire::flow_class(event_slot[i], flags[i], ret_val[i]);
    return NERRF_OK;
}

// Node interning in event order `order` (NULL = identity): one node per pid and one per file identity, ids in
// order of first appearance over the interleaved (process, file[, rename target]) sequence -- exactly the numbering
// of graph.py graph_from_events.  merge_renames: a file and its renamed / encrypted twin share the node (key = path
// without its last extension), a non-empty new_path ALIASES its own key to that node (and names it when it ends in
// .lockbit3) instead of making a node; else every distinct path is a node and a non-empty
// new_path gets one too (node_g, -1 when absent).
// source (NULL: every event from source 0): a process is (source, pid) and a file (source, merge key), so a rename target
// aliases within its own source only.
extern "C" int nerrf_trace_intern_ex(int64_t n_events, const int64_t* order, const uint32_t* pid, const uint16_t* source,
                                     const int64_t* path_off, const uint8_t* path_data, const int64_t* new_path_off,
                                     const uint8_t* new_path_data, int merge_renames, int32_t* node_p, int32_t* node_f,
                                     int32_t* node_g, int64_t* n_nodes, int8_t* node_kind, int64_t* node_name_event,
                                     int8_t* node_name_which, int64_t node_capacity) {
    NERRF_REQUIRE(n_events >= 0 && pid && path_off && new_path_off && node_p && node_f && node_g && n_nodes && node_kind &&
                      node_name_event && node_name_which,
                  "null pointer");
    NERRF_REQUIRE(n_events < ((int64_t)1 << 30), "too many events for 32-bit node ids");
    std::unordered_map<uint64_t, int32_t> pids;
    std::unordered_map<std::string, int32_t> files;
    pids.reserve((size_t)n_events / 8 + 16);
    files.reserve((size_t)n_events / 2 + 16);
    int64_t nn = 0;
    auto new_node = [&](int8_t kind, int64_t ev, int8_t which) -> int32_t {
        if (nn >= node_capacity) return -1;
        node_kind[nn] = kind; node_name_event[nn] = ev; node_name_which[nn] = which;
        return (int32_t)nn++;
    };
    std::string key;
    char sk[2] = {0, 0};                                                 // the source id, appended to every file key
    auto set_key = [&](const uint8_t* s, uint64_t n) { key.assign((const char*)s, n); key.append(sk, 2); };
    for (int64_t k = 0; k < n_events; ++k) {
        const int64_t i = order ? order[k] : k;
        NERRF_REQUIRE(i >= 0 && i < n_events, "order[%lld]=%lld out of range", (long long)k, (long long)i);
        const uint16_t src = source ? source[i] : (uint16_t)0;
        sk[0] = (char)(src & 0xff); sk[1] = (char)(src >> 8);
        const uint64_t pkey = ((uint64_t)src << 32) | pid[i];
        auto pit = pids.find(pkey);
        if (pit == pids.end()) {
            const int32_t id = new_node(1, i, 2);
            NERRF_REQUIRE(id >= 0, "node_capacity=%lld too small", (long long)node_capacity);
            pit = pids.emplace(pkey, id).first;
        }
        node_p[i] = pit->second;
        const uint8_t* s = path_data + path_off[i];
        const uint64_t n = (uint64_t)(path_off[i + 1] - path_off[i]);
        set_key(s, merge_renames ? stem_len(s, n) : n);
        auto fit = files.find(key);
        if (fit == files.end()) {
            const int32_t id = new_node(0, i, 0);
            NERRF_REQUIRE(id >= 0, "node_capacity=%lld too small", (long long)node_capacity);
            fit = files.emplace(key, id).first;
        }
        node_f[i] = fit->second;
        if (wire::ends_with(s, n, ".lockbit3", 9)) { node_name_event[fit->second] = i; node_name_which[fit->second] = 0; }   // rollback target
        node_g[i] = -1;
        const uint64_t gn = (uint64_t)(new_path_off[i + 1] - new_path_off[i]);
        if (gn && merge_renames) {
            // a real rename `a.dat -> a.dat.lockbit3`: the target is the same file identity whatever its stem (merge by
            // inode); later events on the new name land on this node, and an encrypted target names the rollback
            const uint8_t* g = new_path_data + new_path_off[i];
            set_key(g, stem_len(g, gn));
            files.emplace(key, fit->second);                              // no-op when the key is already known
            if (wire::ends_with(g, gn, ".lockbit3", 9)) { node_name_event[fit->second] = i; node_name_which[fit->second] = 1; }
        }
        if (gn && !merge_renames) {
            set_key(new_path_data + new_path_off[i], gn);
            auto git = files.find(key);
            if (git == files.end()) {
                const int32_t id = new_node(0, i, 1);
                NERRF_REQUIRE(id >= 0, "node_capacity=%lld too small", (long long)node_capacity);
                git = files.emplace(key, id).first;
            }
            node_g[i] = git->second;
        }
    }
    *n_nodes = nn;
    return NERRF_OK;
}

extern "C" int nerrf_trace_intern(int64_t n_events, const int64_t* order, const uint32_t* pid, const int64_t* path_off,
                                  const uint8_t* path_data, const int64_t* new_path_off, const uint8_t* new_path_data,
                                  int merge_renames, int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes,
                                  int8_t* node_kind, int64_t* node_name_event, int8_t* node_name_which, int64_t node_capacity) {
    return nerrf_trace_intern_ex(n_events, order, pid, nullptr, path_off, path_data, new_path_off, new_path_data, merge_renames,
                                 node_p, node_f, node_g, n_nodes, node_kind, node_name_event, node_name_which, node_capacity);
}
