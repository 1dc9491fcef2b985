// The nerrf.trace.Event wire parser, shared by the host decoder (csrc/ingest.cu: nerrf_trace_decode) and the device
// decoder (csrc/live_stream.cu: nerrf_trace_decode_device): one definition of the protobuf rules, so the two cannot drift.
// Plain loops only (no libc, no std::): every function compiles for the host and for sm_90a.
//
// Wire schema = proto/trace.proto:11-49 (Event: ts=1 Timestamp{seconds=1, nanos=2}, pid=2, tid=3, comm=4, syscall=5,
// path=6, new_path=7, flags=8 enum, ret_val=9 sint64, bytes=10, inode=11, mode=12, uid=13, gid=14, dependencies=15).
// Rules: a varint is at most 10 bytes; repeated `ts` sub-messages merge; for string fields the last occurrence wins; a
// known field with another wire type is skipped by that wire type; groups (wire types 3, 4) are malformed; pid / tid /
// flags are truncated to 32 bits; ret_val is zigzag-decoded; strings are kept as bytes (no UTF-8 check).
#pragma once
#include <stdint.h>
#include "../../include/nerrf_b200.h"

#define NERRF_HD __host__ __device__ __forceinline__

namespace nerrf {
namespace wire {

struct Reader {
    const uint8_t* p;
    const uint8_t* end;
    NERRF_HD bool varint(uint64_t* v) {
        uint64_t r = 0;
        for (int shift = 0; shift < 70; shift += 7) {
            if (p >= end) return false;
            const uint8_t b = *p++;
            if (shift < 64) r |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) { *v = r; return true; }
        }
        return false;   // > 10 bytes
    }
    NERRF_HD bool len_delim(const uint8_t** s, uint64_t* n) {
        if (!varint(n)) return false;
        if (*n > (uint64_t)(end - p)) return false;
        *s = p; p += *n;
        return true;
    }
    NERRF_HD bool skip(uint32_t wire) {
        uint64_t v; const uint8_t* s;
        switch (wire) {
            case 0: return varint(&v);
            case 1: if (end - p < 8) return false; p += 8; return true;
            case 2: return len_delim(&s, &v);
            case 5: if (end - p < 4) return false; p += 4; return true;
            default: return false;   // groups (3, 4) are not used by this schema
        }
    }
};

struct EventView {
    int64_t ts_sec = 0; int32_t ts_nanos = 0;
    uint32_t pid = 0, tid = 0; int32_t flags = 0; int64_t ret_val = 0; uint64_t bytes = 0;
    const uint8_t *comm = nullptr, *syscall = nullptr, *path = nullptr, *new_path = nullptr;
    uint64_t comm_n = 0, syscall_n = 0, path_n = 0, new_path_n = 0;
};

NERRF_HD bool parse_timestamp(const uint8_t* s, uint64_t n, EventView* e) {
    Reader r{s, s + n};
    while (r.p < r.end) {
        uint64_t tag, v;
        if (!r.varint(&tag)) return false;
        const uint32_t field = (uint32_t)(tag >> 3), wire = (uint32_t)(tag & 7);
        if (field == 1 && wire == 0) { if (!r.varint(&v)) return false; e->ts_sec = (int64_t)v; }
        else if (field == 2 && wire == 0) { if (!r.varint(&v)) return false; e->ts_nanos = (int32_t)v; }
        else if (!r.skip(wire)) return false;
    }
    return true;
}

NERRF_HD bool parse_event(const uint8_t* s, uint64_t n, EventView* e) {
    Reader r{s, s + n};
    while (r.p < r.end) {
        uint64_t tag, v; const uint8_t* q;
        if (!r.varint(&tag)) return false;
        const uint32_t field = (uint32_t)(tag >> 3), wire = (uint32_t)(tag & 7);
        if (wire == 0 && (field == 2 || field == 3 || field == 8 || field == 9 || field == 10)) {
            if (!r.varint(&v)) return false;
            if (field == 2) e->pid = (uint32_t)v;
            else if (field == 3) e->tid = (uint32_t)v;
            else if (field == 8) e->flags = (int32_t)v;
            else if (field == 9) e->ret_val = (int64_t)(v >> 1) ^ -(int64_t)(v & 1);      // zigzag
            else e->bytes = v;
        } else if (wire == 2 && (field == 1 || (field >= 4 && field <= 7))) {
            if (!r.len_delim(&q, &v)) return false;
            if (field == 1) { if (!parse_timestamp(q, v, e)) return false; }             // repeated occurrence merges
            else if (field == 4) { e->comm = q; e->comm_n = v; }
            else if (field == 5) { e->syscall = q; e->syscall_n = v; }
            else if (field == 6) { e->path = q; e->path_n = v; }
            else { e->new_path = q; e->new_path_n = v; }
        } else if (!r.skip(wire)) return false;
    }
    return true;
}

// one top-level record of an EventBatch at r.p: *event = true and (body, n) for an Event (field 1, wire type 2); any other
// field is skipped by its wire type.  false = malformed or cut off.
NERRF_HD bool next_record(Reader* r, bool* event, const uint8_t** body, uint64_t* n) {
    uint64_t tag;
    if (!r->varint(&tag)) return false;
    *event = (tag >> 3) == 1 && (tag & 7) == 2;
    if (*event) return r->len_delim(body, n);
    return r->skip((uint32_t)(tag & 7));
}

NERRF_HD bool equals(const uint8_t* s, uint64_t n, const char* lit, uint64_t m) {
    if (n != m) return false;
    for (uint64_t i = 0; i < m; ++i)
        if (s[i] != (uint8_t)lit[i]) return false;
    return true;
}
NERRF_HD bool matches_at(const uint8_t* s, const char* lit, uint64_t m) {
    for (uint64_t i = 0; i < m; ++i)
        if (s[i] != (uint8_t)lit[i]) return false;
    return true;
}
NERRF_HD bool contains(const uint8_t* s, uint64_t n, const char* lit, uint64_t m) {
    if (n < m) return false;
    for (uint64_t i = 0; i + m <= n; ++i)
        if (s[i] == (uint8_t)lit[0] && matches_at(s + i, lit, m)) return true;
    return false;
}
NERRF_HD bool starts_with(const uint8_t* s, uint64_t n, const char* lit, uint64_t m) { return n >= m && matches_at(s, lit, m); }
NERRF_HD bool ends_with(const uint8_t* s, uint64_t n, const char* lit, uint64_t m) { return n >= m && matches_at(s + n - m, lit, m); }

// "README" or "RANSOM" starting at s[i] (i + 6 <= n), ASCII case-insensitive: both start with R
NERRF_HD bool note_word_at(const uint8_t* s) {
    if ((s[0] | 0x20) != 'r') return false;
    uint8_t w[5];
    for (int k = 0; k < 5; ++k) { const uint8_t c = s[1 + k]; w[k] = (c >= 'a' && c <= 'z') ? (uint8_t)(c - 32) : c; }
    return matches_at(w, "EADME", 5) || matches_at(w, "ANSOM", 5);
}
NERRF_HD bool has_note_word(const uint8_t* s, uint64_t n) {
    if (n < 6) return false;
    for (uint64_t i = 0; i + 6 <= n; ++i)
        if (note_word_at(s + i)) return true;
    return false;
}

// NERRF_PATH_* bits of one path
NERRF_HD uint8_t path_flags(const uint8_t* s, uint64_t n) {
    uint8_t pf = 0;
    if (contains(s, n, ".lockbit", 8)) pf |= NERRF_PATH_LOCKBIT;
    if (has_note_word(s, n)) pf |= NERRF_PATH_NOTE;
    if (starts_with(s, n, "/tmp", 4) || starts_with(s, n, "/proc", 5)) pf |= NERRF_PATH_TMP;
    if (ends_with(s, n, ".lockbit3", 9)) pf |= NERRF_PATH_ENCRYPTED;
    return pf;
}

// event-kind slots of nerrf_b200/graph.py (_EVENT_SLOT); slot 7 = anything else
NERRF_HD int event_slot(const uint8_t* s, uint64_t n) {
    if (equals(s, n, "file_created", 12)) return 0;
    if (equals(s, n, "file_encrypt_start", 18)) return 1;
    if (equals(s, n, "file_encrypt_complete", 21)) return 2;
    if (equals(s, n, "ransom_note_created", 19)) return 3;
    if (equals(s, n, "openat", 6)) return 4;
    if (equals(s, n, "write", 5)) return 5;
    if (equals(s, n, "rename", 6)) return 6;
    return 7;
}

// information-flow class of an event (DESIGN.md 1.5) from its raw slot (event_slot above, not the observable fold), its
// open flags and its return value: bit 0 = process -> file, bit 1 = file -> process.  The one definition of the table:
// the host columns (nerrf_trace_flow_class) and the live stream's device columns (nerrf_trace_flow_class_device) use it.
constexpr uint8_t FLOW_P2F = 1, FLOW_F2P = 2;
NERRF_HD uint8_t flow_class(int slot, int64_t flags, int64_t ret_val) {
    if (ret_val < 0) return 0;                                   // the syscall failed: nothing moved
    switch (slot) {
    case 0: case 1: case 2: case 3: case 5: case 6: return FLOW_P2F;   // created, encrypt_*, note, write, rename
    case 4: return flags == 0 ? FLOW_F2P : flags == 1 ? FLOW_P2F : (uint8_t)(FLOW_P2F | FLOW_F2P);   // openat
    default: return 0;                                           // slot 7: recon *_enum, unlink, ...
    }
}

}  // namespace wire
}  // namespace nerrf
