// Fused GraphSAGE-T layer on Hopper tensor cores (wgmma), sm_90a.
//
//   out[v, :] = act( [x_v || m_v] @ W + b ),   m_v = weighted mean of gathered source rows
//
// computed TRANSPOSED so that the gathered tile is the shared-memory operand and the weights travel in registers:
//
//   D^T[H=128 features, rows] = W^T[128, K=2F] . X^T[K, rows]      (one m64n32k16 wgmma half per consumer warpgroup)
//     A operand = W^T, register fragments split into bf16 terms once per launch.  F = 32, and F = 128 without hub rows:
//                 loaded once per CTA by the consumer warpgroups and kept in their registers (KSTEPS x NS x 4 per thread,
//                 NS = 3: 48 at F = 32, 96 at F = 128, whose layer kernel runs only the mean half, below).  F = 64, and
//                 F = 128 with hub rows: read from L2 one K step ahead of the MMAs
//     F = 64 / 128: the self half x_v . W[0:F] needs no gather; a prep kernel (sage_self_prep_kernel) computes it over
//                 contiguous rows of x with W resident in registers and stores the raw accumulators in out, and the
//                 layer kernel starts from them and runs only the mean half (K = F), which halves its weight traffic.
//                 F = 32 keeps K = 2F in the layer kernel (split_w_kernel).
//     B operand = the gathered tile X[rows, K] exactly as the gather warps produce it: row-major, K contiguous ==
//                 the wgmma "K-major" canonical layout (128-byte swizzle), bf16 terms
//     D         = fp32 accumulators in the consumer warpgroups' registers
//
// fp32-level accuracy from bf16 tensor cores (the 1e-4 bound rules out plain TF32/bf16): every fp32 value v is split
// v = hi + lo (hi = bf16(v), lo = bf16(v - hi)) and the products x_hi.w_hi + x_lo.w_hi + x_hi.w_lo are accumulated in
// fp32 (error ~1e-5 relative); NS = 3 terms with six products is fp32-equivalent.
//
// The aggregate never round-trips HBM: gather warps write hi/lo bf16 straight into the shared memory B operand.
// Warp roles in one CTA per SM:
//   warps 0-7   two consumer warpgroups (output features 0-63 and 64-127): wgmma (A in registers, B from shared
//               memory), then the epilogue from the accumulator registers: + bias, ReLU, row stores, fused node head.
//               At F = 64 / 128 they take the tiles two at a time (F = 128 without hub rows: both tiles' MMAs in
//               one commit group)
//   warp  8     edge-block loader: stages each tile's rowptr words and its col / ew slices into shared memory --
//               the slices as two bulk async copies (cp.async.bulk, byte count on the stage's mbarrier) --
//               running up to IDX_STAGES tiles ahead; the next tile's rowptr words are prefetched before it
//               waits for a free stage
//   warps 9-..  gather: one CSR row per warp at a time (four at F=32), rows round-robin; source rows are copied into the
//               warp's shared-memory ring with cp.async (LDGSTS, 16 B per lane), NQ-1 sub-batches in flight;
//               indices come from shared memory, so the only global latency a row exposes is its x rows.
//               F = 32: warps 9-23 (six warpgroups; consumers 112 registers per thread, producers 64).  F = 128 without
//               hub rows: warps 9-19 (five warpgroups; consumers 168, producers 48).  Otherwise warps 9-22 and a spare
//               warp 23 (six warpgroups; consumers 128, producers 56)
// Pipelines: idx stages full/empty (loader <-> gather), smem operand stages full/empty (gather <-> consumer).
#include <map>
#include <mutex>
#include <utility>
#include "common.cuh"
#include "ptx.cuh"
#include "sage_gather.cuh"

namespace nerrf {

namespace {

constexpr int TN = 32;                 // destination rows per tile (wgmma N)
constexpr int UM = 128;                // hidden width = two wgmma M=64 halves
constexpr int EPI_WARPS = 8;           // two consumer warpgroups, one per 64-feature half of the output
constexpr int LOADER_WARP = 8;
constexpr int GATHER_WARP0 = 9;
constexpr int EMAX = 512;              // staged edges per tile (4 KB); the rest of a heavier tile is read from global
constexpr int EPAD = EMAX + 4;         // a slice is copied as its 16-byte aligned superset: up to 3 leading + 3 trailing elements
constexpr int IDX_STAGE_BYTES = EPAD * 8 + 512;      // col[EPAD] | ew[EPAD] | rp[TN+1] (relative) | e_lo (int64) | col_off, ew_off
// items (source rows) per sub-batch (= one cp.async group): 4 warp-wide copy instructions, i.e. 4 * (32 / (F/4))
template <int F> constexpr int qs_for() { return 4 * (32 / (F / 4)); }

// NS = number of bf16 terms each fp32 value is split into (v = p0 + p1 [+ p2], p_i = bf16 of the
// running residual).  NS = 3 with the six products (x0w0, x1w0, x0w1, x1w1, x2w0, x0w2) drops only
// terms below 2^-24: fp32-equivalent.  NS = 2 with three products is ~1e-5 relative.
// LONG: the launch has hub-row scratch (the kernel's pre-aggregated partial items); it picks the CTA shape at F = 128.
template <int F, int NS, bool LONG = false>
struct UmmaCfg {
    // RESIDENT: the consumers keep all of the split W^T of the K steps they run in registers (KSTEPS x NS x 4: 48 at F = 32
    // (K = 2F), 96 at F = 128, NS = 3).  At F = 128 that takes a CTA of five warpgroups with 11 gather warps, which
    // measured faster without hub rows but slower on the hub-destination graph, whose gather (hub-row partial items) sets
    // the pace with fewer warps, and slower at F = 64, where there is less weight traffic to save: there the layer keeps
    // 14 gather warps and reads the fragments from L2 one K step ahead of the MMAs (DESIGN 2.1, 5).
    static constexpr bool RESIDENT = F == 32 || (F == 128 && !LONG);
    // F = 32: 15 gather warps (the quad gather needs the TLP).  F = 64 / 128 resident: 11 gather warps with deeper rings
    // (NQ = 5: 4 sub-batches in flight per warp, ~the bytes in flight of 14 warps x 3); otherwise 14 and NQ = 4
    static constexpr int GATHER_WARPS = (F == 32) ? 15 : RESIDENT ? 11 : 14;
    static constexpr int NQ = (F != 32 && RESIDENT) ? 5 : 4; // sub-batch slots in a warp's ring; NQ-1 groups are in flight
    // The CTA is whole warpgroups (14 gather warps: one spare warp after them), so that setmaxnreg can
    // move registers from the producer warpgroups (loader, gather) to the two consumer warpgroups: THREADS x LAUNCH_REGS
    // >= 2 x 128 x CONSUMER_REGS + (WARPS / 4 - 2) x 128 x PRODUCER_REGS.  768 x 80 = 2 x 128 x 112 + 4 x 128 x 64 (F = 32),
    // 640 x 96 = 2 x 128 x 168 + 3 x 128 x 48 (F = 128 resident: W^T and two tiles' accumulators),
    // 768 x 80 = 2 x 128 x 128 + 4 x 128 x 56 (F = 64, F = 128 with hub rows: two tiles' accumulators, two fragment sets)
    static constexpr int WARPS = (GATHER_WARP0 + GATHER_WARPS + 3) / 4 * 4;
    static constexpr int THREADS = WARPS * 32;
    static constexpr int LAUNCH_REGS = (65536 / THREADS) & ~7;   // one CTA per SM, allocated in 8-register steps
    static constexpr int CONSUMER_REGS = (F == 32) ? 112 : RESIDENT ? 168 : 128;
    static constexpr int PRODUCER_REGS = (F == 32) ? 64 : RESIDENT ? 48 : 56;
    static_assert((EPI_WARPS * CONSUMER_REGS + (WARPS - EPI_WARPS) * PRODUCER_REGS) * 32 <= THREADS * LAUNCH_REGS,
                  "register budget at launch");
    // F = 32 (quad-mode gather): a warp runs up to 3 units = ~7 tiles ahead of what it has consumed and holds a tile's edge
    // block from issue to completion, so the look-ahead is bounded by the number of edge-block stages, not by the rings
    // (with 4 stages most issue-side polls find the next tile not yet staged)
    static constexpr int IDX_STAGES = (F == 32) ? 9 : 3;
    // F = 64 / 128: the self half x_v . W[0:F] is computed by the prep kernel (sage_self_prep_kernel) and the layer kernel
    // starts its accumulators from it, so a tile carries only the mean columns (K = F).  At F = 32 a mean-only row
    // (64 B) would be less than one 128-byte swizzle block, so the tile keeps [x_v || m_v] (K = 2F).
    static constexpr bool SELF_SPLIT = F != 32;
    static constexpr int K = SELF_SPLIT ? F : 2 * F;
    static constexpr int KB = K / 64;                        // 128-byte K blocks
    static constexpr int KSTEPS = K / 16;                    // MMAs (K=16) per product
    static constexpr int PART_BYTES = KB * TN * 128;         // one bf16 term of one stage
    static constexpr int STAGE_BYTES = NS * PART_BYTES;
    static constexpr int QS = qs_for<F>();                    // 4 (F=128), 8 (F=64), 16 (F=32): always 2 KB per sub-batch
    static constexpr int RING_BYTES = NQ * QS * F * 4;       // per gather warp: NQ sub-batches x QS source rows (8 / 10 KB)
    static constexpr int STAGES = 4;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + IDX_STAGES * IDX_STAGE_BYTES +
                                   (size_t)GATHER_WARPS * RING_BYTES + 2048 /*head reduce*/ + 1024 /*align*/ + 1024 /*barriers*/;
    static_assert(SMEM <= 227 * 1024, "shared memory budget");
    static_assert(STAGES >= 2, "need at least two smem stages");
};

template <int NS>
__device__ __forceinline__ void split4(const float4 v, uint2 (&parts)[NS]) {
    uint32_t lo[NS], hi[NS];
    split_pair<NS>(v.x, v.y, lo);
    split_pair<NS>(v.z, v.w, hi);
#pragma unroll
    for (int p = 0; p < NS; ++p) parts[p] = make_uint2(lo[p], hi[p]);
}

// the products of one K step over the split terms (a = W^T terms, xb = descriptors of the x terms), in the fixed order
// x0w0, x1w0, x0w1 [, x1w1, x2w0, x0w2]; scale_d 0 on the first product starts the accumulator
template <int NS>
__device__ __forceinline__ void wgmma_split_products(float (&d)[16], const uint32_t (&a)[NS][4], const uint64_t (&xb)[NS],
                                                     uint32_t scale_d) {
    wgmma_rs(d, a[0], xb[0], scale_d);
    wgmma_rs(d, a[0], xb[1], 1u);
    wgmma_rs(d, a[1], xb[0], 1u);
    if constexpr (NS == 3) {
        wgmma_rs(d, a[1], xb[1], 1u);
        wgmma_rs(d, a[0], xb[2], 1u);
        wgmma_rs(d, a[2], xb[0], 1u);
    }
}

// ---------------------------------------------------------------- fused exchange (multi-GPU)
// Peer-mapped [n_nodes, 128] embedding buffers of the other ranks (NVLink P2P, CUDA IPC / symmetric memory).
// The epilogue stores every output row slice to the local buffer AND to each peer buffer, so the per-layer
// embedding exchange of the 1-D sharded forward happens inside the layer kernel, overlapped tile by tile.
constexpr int MAX_PEERS = 7;
struct Peers {
    float* out[MAX_PEERS];
    int n;
    const uint8_t* need;  // optional [n_nodes]: bit pr set <=> peer slot pr references this row as a source; rows a
                          // peer never reads are not sent to it (nullptr: send every row to every peer)
    float* mc;            // NVSwitch multicast address of the same buffer on ALL ranks (incl. this one), or nullptr:
                          // one multimem.st per element, replicated by the switch (egress 1x instead of (G-1)x)
};
__device__ __forceinline__ void multimem_st2(float* addr, const float2 v) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(v.x), "f"(v.y) : "memory");
}
// ---------------------------------------------------------------- long rows (hub destinations)
// A destination row with more than LONG_T in-edges would be gathered by ONE warp.  A deterministic pre-pass
// cuts every such row into fixed chunks of LONG_CH edges; one CTA per chunk computes the unnormalised
// weighted sum + weight sum (fixed order: 8 warps x 64 edges, then warp 0 adds the 8 warp partials in order)
// into a side buffer.  The main kernel then sees the row as the items [partial_0 .. partial_{nc-1}] (F=32:
// [self, partial_0 ..]; weight 1 each, weight-sum from pw[]).  The workspace is capacity driven: rows that do not fit stay inline.
// Threshold: a row of a few hundred edges gathered by one warp takes many times as long as the other 31 rows of its tile,
// and a trace graph has exactly such a row every 64 nodes (the process node of each component, in-degree = events of
// its files).
constexpr int LONG_T = 128;
constexpr int LONG_CH = 256;

struct LongWs {
    int* hdr;              // [0] = number of chunk items claimed (may exceed cap), [1] = cap
    int* hash_key;         // row + 1, 0 = empty
    int* hash_val;         // first item of the row
    int2* queue;           // per chunk item: (absolute row, chunk index within the row)
    float* partial;        // [cap][128]
    float* pw;             // [cap]
    int cap;
    int hash_mask;         // slots - 1 (slots = power of two >= 2 * cap)
};

__host__ __device__ inline size_t long_ws_bytes_for(int cap, int slots) {
    return 256 + (size_t)slots * 8 + (size_t)cap * (8 + 128 * 4 + 4);
}
static LongWs long_ws_carve(void* ws, size_t bytes) {
    LongWs L{};
    if (!ws || bytes < 8192) return L;
    int cap = (int)((bytes - 256) / (8 + 128 * 4 + 4 + 32));        // 32 B/item covers the hash (>= 2 slots x 8 B, rounded up)
    cap &= ~3;                                                       // keeps every sub-array 16-byte aligned
    if (cap < 4) return L;
    int slots = 1;
    while (slots < 2 * cap) slots <<= 1;
    while (long_ws_bytes_for(cap, slots) > bytes && cap > 4) { cap = (cap * 3 / 4) & ~3; slots = 1; while (slots < 2 * cap) slots <<= 1; }
    if (long_ws_bytes_for(cap, slots) > bytes) return L;
    unsigned char* b = (unsigned char*)ws;
    L.hdr = (int*)b; b += 256;
    L.hash_key = (int*)b; b += (size_t)slots * 4;
    L.hash_val = (int*)b; b += (size_t)slots * 4;
    L.queue = (int2*)b; b += (size_t)cap * 8;
    L.partial = (float*)b; b += (size_t)cap * 128 * 4;
    L.pw = (float*)b;
    L.cap = cap; L.hash_mask = slots - 1;
    return L;
}
__device__ __forceinline__ int long_hash(int64_t row, int mask) { return (int)(((uint64_t)row * 0x9E3779B97F4A7C15ull) >> 40) & mask; }
__device__ __forceinline__ int long_lookup(const LongWs& L, int64_t row) {      // first item of `row`, or -1
    int h = long_hash(row, L.hash_mask);
    const int key = (int)row + 1;
    for (int probe = 0; probe <= L.hash_mask; ++probe) {
        const int k = L.hash_key[h];
        if (k == key) return L.hash_val[h];
        if (k == 0) return -1;
        h = (h + 1) & L.hash_mask;
    }
    return -1;
}

template <typename RP>
__global__ void __launch_bounds__(256) long_scan_kernel(const RP* __restrict__ rowptr, int64_t row_begin, int64_t row_end, LongWs L) {
    for (int64_t row = row_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < row_end; row += (int64_t)gridDim.x * blockDim.x) {
        const int64_t deg = (int64_t)rowptr[row + 1] - (int64_t)rowptr[row];
        if (deg <= LONG_T) continue;
        const int nch = (int)((deg + LONG_CH - 1) / LONG_CH);
        const int first = atomicAdd(L.hdr, nch);
        if (first + nch > L.cap) continue;                               // does not fit: the row stays inline
        for (int c = 0; c < nch; ++c) L.queue[first + c] = make_int2((int)row, c);
        int h = long_hash(row, L.hash_mask);
        const int key = (int)row + 1;
        while (atomicCAS(L.hash_key + h, 0, key) != 0) h = (h + 1) & L.hash_mask;
        L.hash_val[h] = first;
    }
}

template <int F, typename RP>
__global__ void __launch_bounds__(256) long_chunk_kernel(const float* __restrict__ x, const RP* __restrict__ rowptr,
                                                         const int32_t* __restrict__ col, const float* __restrict__ ew, LongWs L) {
    __shared__ float4 s_acc[8][32];
    __shared__ float s_w[8];
    constexpr int LPR = F / 4;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int n_items = L.hdr[0];
    if (n_items > L.cap) n_items = L.cap;                                // items past cap were never queued ...
    for (int i = blockIdx.x; i < n_items; i += gridDim.x) {
        const int2 it = L.queue[i];
        if (it.x < 0) continue;                                          // claimed by a row that did not fit (never queued)
        const int64_t e0 = (int64_t)rowptr[it.x], e1 = (int64_t)rowptr[it.x + 1];
        const int64_t c0 = e0 + (int64_t)it.y * LONG_CH;
        const int64_t c1 = (c0 + LONG_CH < e1) ? c0 + LONG_CH : e1;
        const int64_t a = c0 + warp * (LONG_CH / 8);
        int64_t b = a + LONG_CH / 8;
        if (b > c1) b = c1;
        float wsum = 0.f;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a < b) acc = gather_row<F>(x, col, ew, a, b, lane, &wsum);
        if (lane < LPR) s_acc[warp][lane] = acc;
        if (lane == 0) s_w[warp] = wsum;
        __syncthreads();
        if (warp == 0) {
            if (lane < LPR) {
                float4 t = s_acc[0][lane];
#pragma unroll
                for (int k = 1; k < 8; ++k) { t.x += s_acc[k][lane].x; t.y += s_acc[k][lane].y; t.z += s_acc[k][lane].z; t.w += s_acc[k][lane].w; }
                *reinterpret_cast<float4*>(L.partial + (size_t)i * 128 + 4 * lane) = t;
            }
            if (lane == 0) {
                float t = s_w[0];
#pragma unroll
                for (int k = 1; k < 8; ++k) t += s_w[k];
                L.pw[i] = t;
            }
        }
        __syncthreads();
    }
}

// LONG: compiled with the hub-row (pre-aggregated partial items) paths; the plain variant is used when the
// launch has no hub-row scratch, so graphs without hub rows pay nothing for the feature.
template <int F, int NS, typename RP, bool LONG>
__global__ void __launch_bounds__((UmmaCfg<F, NS, LONG>::THREADS), 1)
sage_layer_umma_kernel(const float* __restrict__ x, const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                       const float* __restrict__ ew, const float* __restrict__ W, const float* __restrict__ bias,
                       float* __restrict__ out, int64_t row_begin, int64_t row_end, int relu,
                       const float* __restrict__ node_w, float node_b, float* __restrict__ score, const LongWs lw,
                       const Peers peers, unsigned* __restrict__ tile_ctr, const uint4* __restrict__ wsplit,
                       int l2_policy) {
    using C = UmmaCfg<F, NS, LONG>;
    constexpr int LPR = F / 4;
    // L2 policy, F = 64 / 128 (l2_policy == 0: every access at normal priority): the gathered source rows, S, the output rows
    // and the col / ew slices are evict-first; the F = 32 layer (QUAD below) gives no hints (measured, DESIGN 2.1).
    // Created where it is used, so that it holds no register across the roles.
    auto pol = [l2_policy]() { return l2_policy ? l2_policy_evict_first() : l2_policy_evict_normal(); };
    constexpr int GATHER_WARPS = C::GATHER_WARPS, IDX_STAGES = C::IDX_STAGES, NQ = C::NQ;
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;          // SWIZZLE_128B needs 1024-B alignment
    unsigned char* smem_gen = smem_dyn + (smem_base - smem_u32(smem_dyn));
    const uint32_t idx_base = smem_base + C::STAGES * C::STAGE_BYTES;
    // 1 KB barrier area, then the gather rings: the stage mbarriers in the first 256 B, end_tl and the tile-id ring in
    // the last 72 B, the bytes in between unused
    const uint32_t bar_base = idx_base + IDX_STAGES * IDX_STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
    auto idxf_bar = [&](int q) { return bar_base + 8u * (2 * C::STAGES + q); };
    auto idxe_bar = [&](int q) { return bar_base + 8u * (2 * C::STAGES + IDX_STAGES + q); };
    static_assert(8 * (2 * C::STAGES + 2 * IDX_STAGES) <= 256, "barrier area");
    // DYNAMIC TILE SCHEDULE: the loader warp claims tiles from a global counter (tile_ctr, zero at launch) and publishes
    // the id of the CTA's tl-th tile in this ring (-1 = end of stream) before it releases the tile's edge block; every
    // role reads it after the mbarrier wait that orders it behind that release.  Rows are not equally expensive (hub
    // destinations: a 32-row tile can hold 50x the edges of an average one), a static round-robin left whole SMs idle.
    constexpr int TILE_RING = 16;                  // > IDX_STAGES + STAGES: an entry outlives its tile
    volatile int* tile_ids = reinterpret_cast<volatile int*>(smem_gen + (bar_base + 1024 - 64 - smem_base));
    // QUAD mode (F = 32): a gather warp works on FOUR rows at a time, one per 8-lane group (a 128-byte source row is 8 lanes
    // x 16 B), so the per-row overhead -- row setup, the cross-group combine, the bf16 split, the operand stores, the barrier
    // arrivals -- is paid once per four rows and by all 32 lanes (one row per warp leaves the F=32 layer issue-bound on
    // this overhead).  Units of 4 rows are dealt round-robin to the warps; a warp need not
    // own a unit in every tile, so the end of the tile stream is also published in `end_tl` (the closing tile's index).
    constexpr bool QUAD = F == 32;
    volatile int* end_tl = reinterpret_cast<volatile int*>(smem_gen + (bar_base + 1024 - 64 - 8 - smem_base));
    unsigned char* idx_gen = smem_gen + (idx_base - smem_base);
    const uint32_t ring_base = bar_base + 1024;
    float* head_red = reinterpret_cast<float*>(smem_gen + (ring_base - smem_base) + (size_t)GATHER_WARPS * C::RING_BYTES);   // [2][8][32]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t rows = row_end - row_begin;
    const int64_t n_tiles = (rows + TN - 1) / TN;

    if (warp == LOADER_WARP) {
        if (lane == 0) {
            // operand stage full: one arrival per row (per 4-row unit in QUAD mode); empty: one per consumer warp
            for (int s = 0; s < C::STAGES; ++s) { mbar_init(full_bar(s), QUAD ? TN / 4 : TN); mbar_init(empty_bar(s), EPI_WARPS); }
            *end_tl = 0x7fffffff;
            for (int i = 0; i < TILE_RING; ++i) tile_ids[i] = -1;        // (the consumers peek at entries ahead)
            // idx full: ONE arrive.expect_tx by the loader (publishes the rowptr words, counts the bytes of the two bulk
            // copies); empty: one per gather warp (per 4-row unit in QUAD mode)
            for (int q = 0; q < IDX_STAGES; ++q) { mbar_init(idxf_bar(q), 1); mbar_init(idxe_bar(q), QUAD ? TN / 4 : GATHER_WARPS); }
            fence_barrier_init();
        }
        __syncwarp();
    }
    __syncthreads();

    if (warp >= GATHER_WARP0) {
      if constexpr (QUAD) {
        // =========================================================== gather warps, QUAD mode (F = 32): see above
        constexpr int UPT = TN / 4;                                       // units (4 rows) per tile
        constexpr int SLOT_BYTES = 4 * 4 * F * 4;                         // a sub-batch = 4 steps x 4 rows x 128 B = 2 KB
        static_assert(SLOT_BYTES * NQ == C::RING_BYTES, "ring layout");
        setmaxnreg_dec<C::PRODUCER_REGS>();
        const int g = warp - GATHER_WARP0;
        const int grp = lane >> 3, sub = lane & 7;
        // ring slot layout [step][group][8 lanes x 16 B] = lane-linear: conflict-free 16-byte shared loads
        const uint32_t ring_u32 = ring_base + (uint32_t)(g * C::RING_BYTES) + (uint32_t)(lane * 16);
        const float* ring_gen = reinterpret_cast<const float*>(smem_gen + (ring_base - smem_base) + (size_t)g * C::RING_BYTES) + lane * 4;
        const float* xs = x + 4 * sub;
        int stream_end = 0x7fffff00;                                      // in units

        // per-unit state; e0 / items / row / long are per GROUP (each 8-lane group has its own row), nb is warp-uniform
        int iu = g, ib = 0, inb = 1, ie0 = 0, iitems = 0, ilong = -1, itl = -1, itile = 0;  uint32_t irow = 0;  bool ifast = true;
        const int32_t* icol = nullptr; int64_t ielo = 0;
        int cu = g, cb = 0, cnb = 1, ce0 = 0, citems = 0, clong = -1, ctl = -1, ctile = 0;  bool cfast = true;
        const float* cew = nullptr; int64_t celo = 0;

        // Set up unit `iu` for issuing.  NEVER blocks: a warp runs up to NQ-1 sub-batches = up to 3 units = ~7 tiles ahead of
        // what it has consumed, more than there are edge-block stages, so blocking here for a stage that is waiting for this
        // very warp's consumption would deadlock.  false = the unit's tile is not staged yet (the caller emits an empty
        // "bubble" group and retries at its next call) or the stream ended before it (stream_end shrinks to iu).
        auto try_setup_issue_unit = [&]() -> bool {
            const int tl = iu / UPT, r = (iu % UPT) * 4 + grp;
            if (tl != itl) {
                uint32_t done;
                // test_wait, not try_wait: the latter may suspend the warp for a hardware time limit, and this poll sits in front of
                // the consumption of data that has already landed
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(done) : "r"(idxf_bar(tl % IDX_STAGES)), "r"((uint32_t)(tl / IDX_STAGES) & 1u) : "memory");
                if (!__all_sync(0xffffffffu, done != 0)) {               // every lane must have acquired the loader's writes
                    if (__any_sync(0xffffffffu, *end_tl < tl)) stream_end = iu;    // the tile will never come
                    return false;
                }
                itl = tl;
                itile = tile_ids[tl % TILE_RING];
                if (itile < 0) stream_end = (tl + 1) * UPT;              // the closing tile: its units carry the end of stream on
            }
            const unsigned char* ibp = idx_gen + (size_t)(tl % IDX_STAGES) * IDX_STAGE_BYTES;
            const int32_t* rp_s = reinterpret_cast<const int32_t*>(ibp + EPAD * 8);
            // (the closing tile's stage holds no rowptr words: its slack reads must not follow a stale offset)
            icol = reinterpret_cast<const int32_t*>(ibp) + (itile >= 0 ? rp_s[96 + 2] : 0);
            ielo = *reinterpret_cast<const int64_t*>(ibp + EPAD * 8 + 384);
            const int64_t row = row_begin + (int64_t)itile * TN + r;
            ib = 0; iitems = 0; ilong = -1; ifast = true;
            if (itile < 0) ie0 = 1;
            if (itile >= 0 && row < row_end) {
                irow = (uint32_t)row;
                ie0 = rp_s[r];
                const int deg = rp_s[r + 1] - ie0;
                iitems = deg + 1;                                        // [self, edges...]
                if (LONG && deg > LONG_T && lw.cap > 0) {
                    ilong = long_lookup(lw, row);
                    if (ilong >= 0) iitems = 1 + (deg + LONG_CH - 1) / LONG_CH;
                }
                ifast = ilong < 0 && ie0 + deg <= EMAX;
            }
            inb = __reduce_max_sync(0xffffffffu, (iitems + 3) >> 2);
            inb = inb > 0 ? inb : 1;                                     // an all-invalid unit still travels as one empty sub-batch
            ifast = __all_sync(0xffffffffu, ifast);
            return true;
        };
        auto setup_consume_unit = [&]() {                                // cu < stream_end, tile already staged
            const int tl = cu / UPT, r = (cu % UPT) * 4 + grp;
            if (tl != ctl) ctile = tile_ids[tl % TILE_RING];
            ctl = tl;
            const unsigned char* ibp = idx_gen + (size_t)(tl % IDX_STAGES) * IDX_STAGE_BYTES;
            const int32_t* rp_s = reinterpret_cast<const int32_t*>(ibp + EPAD * 8);
            cew = reinterpret_cast<const float*>(ibp + EPAD * 4) + (ctile >= 0 ? rp_s[96 + 3] : 0);
            celo = *reinterpret_cast<const int64_t*>(ibp + EPAD * 8 + 384);
            const int64_t row = row_begin + (int64_t)ctile * TN + r;
            cb = 0; citems = 0; clong = -1; cfast = true;
            if (ctile < 0) ce0 = 1;
            if (ctile >= 0 && row < row_end) {
                ce0 = rp_s[r];
                const int deg = rp_s[r + 1] - ce0;
                citems = deg + 1;
                if (LONG && deg > LONG_T && lw.cap > 0) {
                    clong = long_lookup(lw, row);
                    if (clong >= 0) citems = 1 + (deg + LONG_CH - 1) / LONG_CH;
                }
                cfast = clong < 0 && ce0 + deg <= EMAX;
            }
            cnb = __reduce_max_sync(0xffffffffu, (citems + 3) >> 2);
            cnb = cnb > 0 ? cnb : 1;
            cfast = __all_sync(0xffffffffu, cfast);
        };
        // one cp.async group = sub-batch `ib` of the issue unit: 4 steps, step s = item ib*4+s of each of the 4 rows
        bool iready = false, cready = false;
        uint32_t bubbles = 0;                                             // bit q: nothing was issued into ring slot q
        auto issue = [&](int slot) {
            if (iu < stream_end && !iready) iready = try_setup_issue_unit();       // may shrink stream_end
            bubbles |= 1u << slot;
            if (iu < stream_end && iready) {
                bubbles &= ~(1u << slot);
                const int first = ib * 4;
                const uint32_t dst = ring_u32 + (uint32_t)(slot * SLOT_BYTES);
                if (ifast) {                                             // every row of the unit staged in full: branch free
                    uint32_t src[4];
#pragma unroll
                    for (int st = 0; st < 4; ++st) src[st] = (uint32_t)icol[ie0 + first + st - 1];   // slack reads stay in smem
                    if (first == 0) src[0] = irow;                       // item 0 of every row is its self row
#pragma unroll
                    for (int st = 0; st < 4; ++st)
                        cp_async16_pred(dst + (uint32_t)(st * 512), xs + (size_t)src[st] * F, first + st < iitems);
                } else {
#pragma unroll
                    for (int st = 0; st < 4; ++st) {
                        const int it = first + st;
                        if (it < iitems) {
                            const float* srcp;
                            if (it == 0) srcp = xs + (size_t)irow * F;
                            else if (LONG && ilong >= 0) srcp = lw.partial + (size_t)(ilong + it - 1) * 128 + 4 * sub;
                            else {
                                const int k = ie0 + it - 1;
                                srcp = xs + (size_t)(uint32_t)((k < EMAX) ? icol[k] : __ldg(col + ielo + k)) * F;
                            }
                            cp_async16(dst + (uint32_t)(st * 512), srcp);
                        }
                    }
                }
                if (++ib >= inb) { iu += GATHER_WARPS; iready = false; }
            }
            cp_async_commit();                                            // (possibly empty) group keeps the count in step
        };

        int islot = 0, cslot = 0;
#pragma unroll
        for (int d = 0; d < NQ - 1; ++d) { issue(islot); islot = (islot + 1) % NQ; }
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f), self = acc;
        float wsum = 0.f;
        int last_tl = -1;
        while (cu < stream_end) {
            cp_async_wait<NQ - 2>();
            __syncwarp();
            issue(islot);
            islot = (islot + 1) % NQ;
            if ((bubbles >> cslot) & 1u) {                                // a bubble: the unit's tile was not staged yet
                cslot = (cslot + 1) % NQ;
                __nanosleep(64);
                continue;
            }
            if (!cready) { setup_consume_unit(); cready = true; }         // first sub-batch of the unit (its tile is staged: the
                                                                          // issue side saw it, and this warp has not released it)
            {
                const int first = cb * 4;
                const float* rs = ring_gen + cslot * (SLOT_BYTES / 4);
                if (cfast) {
                    float4 v[4];
                    float w[4];
#pragma unroll
                    for (int st = 0; st < 4; ++st) {
                        v[st] = *reinterpret_cast<const float4*>(rs + st * 128);
                        w[st] = cew[ce0 + first + st - 1];
                    }
                    if (first == 0) { self = v[0]; w[0] = 0.f; v[0] = make_float4(0.f, 0.f, 0.f, 0.f); }
#pragma unroll
                    for (int st = 0; st < 4; ++st) {
                        if (first + st < citems) {
                            wsum += w[st];
                            acc.x = fmaf(w[st], v[st].x, acc.x); acc.y = fmaf(w[st], v[st].y, acc.y);
                            acc.z = fmaf(w[st], v[st].z, acc.z); acc.w = fmaf(w[st], v[st].w, acc.w);
                        }
                    }
                } else {
#pragma unroll
                    for (int st = 0; st < 4; ++st) {
                        const int it = first + st;
                        if (it < citems) {
                            const float4 v = *reinterpret_cast<const float4*>(rs + st * 128);
                            if (it == 0) {
                                self = v;
                            } else if (LONG && clong >= 0) {             // chunk partial: already weighted
                                wsum += lw.pw[clong + it - 1];
                                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                            } else {
                                const int k = ce0 + it - 1;
                                const float w = (k < EMAX) ? cew[k] : __ldg(ew + celo + k);
                                wsum += w;
                                acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
                                acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                            }
                        }
                    }
                }
            }
            cslot = (cslot + 1) % NQ;
            if (++cb < cnb) continue;

            // ---- unit complete: all 32 lanes normalise, split and store their 4 columns of their group's row
            const int tl = ctl;
            const int r = (cu % UPT) * 4 + grp;
            const int s = tl % C::STAGES;
            if (tl != last_tl) {
                mbar_wait(empty_bar(s), ((uint32_t)(tl / C::STAGES) & 1u) ^ 1u);
                last_tl = tl;
            }
            if (citems > 0) {
                const float inv = 1.0f / fmaxf(wsum, 1e-12f);
                const float4 mean = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
                unsigned char* st = smem_gen + (size_t)s * C::STAGE_BYTES;
                uint2 parts[NS];
                split4<NS>(self, parts);
                uint32_t off = sw128_offset<TN>(r, 4 * sub);
#pragma unroll
                for (int p = 0; p < NS; ++p) *reinterpret_cast<uint2*>(st + p * C::PART_BYTES + off) = parts[p];
                split4<NS>(mean, parts);
                off = sw128_offset<TN>(r, F + 4 * sub);
#pragma unroll
                for (int p = 0; p < NS; ++p) *reinterpret_cast<uint2*>(st + p * C::PART_BYTES + off) = parts[p];
            }
            fence_proxy_async();
            acc = make_float4(0.f, 0.f, 0.f, 0.f); self = acc; wsum = 0.f;
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(full_bar(s));
                mbar_arrive(idxe_bar(tl % IDX_STAGES));                  // one arrival per unit (the stage has UPT of them)
            }
            cu += GATHER_WARPS;
            cready = false;
        }
        cp_async_wait<0>();
      } else {
        // =========================================================== gather warps (producers of the B operand)
        // Row stream of this warp: i = g, g+G, g+2G, ... over the CTA's tiles.  A row is the item list
        // [edge_0 .. edge_{deg-1}] (the self row is the prep kernel's), cut into sub-batches of QS items; a row without
        // items travels as one empty sub-batch and writes a zero mean.  A sub-batch is one cp.async group into a
        // slot of this warp's shared-memory ring: each warp-wide 16-byte cp.async (LDGSTS) copies G whole source rows.
        // NQ-1 sub-batches stay in flight while the oldest is consumed (LDS + FFMA), so memory-level parallelism is
        // bounded by the ring, not by registers, and no load ever stalls a scoreboard.
        static_assert(C::SELF_SPLIT, "the row-per-warp gather writes only the mean columns");
        setmaxnreg_dec<C::PRODUCER_REGS>();
        if constexpr (C::WARPS > GATHER_WARP0 + GATHER_WARPS)           // 14 gather warps: the spare warp has no ring
            if (warp >= GATHER_WARP0 + GATHER_WARPS) return;
        constexpr int G = 32 / LPR;                                     // items consumed by one warp-wide LDS.128
        constexpr int QS = C::QS;
        constexpr int SLOT_FLOATS = QS * F;
        const int g = warp - GATHER_WARP0;
        const int grp = lane / LPR, sub = lane % LPR;
        // lane (grp, sub) moves bytes [16 sub, 16 sub + 16) of item t + grp
        const uint32_t ring_u32 = ring_base + (uint32_t)(g * C::RING_BYTES) + (uint32_t)((grp * F + 4 * sub) * 4);
        const float* xs = x + 4 * sub;
        const float* ring_gen = reinterpret_cast<const float*>(smem_gen + (ring_base - smem_base) + (size_t)g * C::RING_BYTES) + grp * F + 4 * sub;
        int stream_end = 0x7fffff00;                                     // rows of this CTA's tile stream; known once the
                                                                          // end-of-stream entry (-1) shows up
        int itile = 0, ctile = 0;

        // ---- per-row state, issue side (i*) and consume side (c*)
        int ii = g, ib = 0, inb = 1, ie0 = 0, ideg = -1, itl = -1, ilong = -1, iitems = 0;
        const int32_t* icol = nullptr; int64_t ielo = 0;
        int ci = g, cb = 0, cnb = 1, ce0 = 0, cdeg = -1, ctl = -1, clong = -1, citems = 0;
        const float* cew = nullptr; int64_t celo = 0;

        auto setup_issue_row = [&]() {                                  // ii < stream_end
            const int tl = ii / TN, r = ii % TN;
            if (tl != itl) {
                const int q = tl % IDX_STAGES;
                mbar_wait(idxf_bar(q), (uint32_t)(tl / IDX_STAGES) & 1u);          // edge block staged
                itl = tl;
                itile = tile_ids[tl % TILE_RING];
                if (itile < 0) stream_end = (tl + 1) * TN;                        // a row-less closing tile: it carries the
                                                                                  // end of stream through every pipeline
            }
            const unsigned char* ibp = idx_gen + (size_t)(tl % IDX_STAGES) * IDX_STAGE_BYTES;
            const int32_t* rp_s = reinterpret_cast<const int32_t*>(ibp + EPAD * 8);
            icol = reinterpret_cast<const int32_t*>(ibp) + rp_s[96 + 2];            // + alignment offset of the col slice
            ielo = *reinterpret_cast<const int64_t*>(ibp + EPAD * 8 + 384);
            const int64_t row = row_begin + (int64_t)itile * TN + r;
            ib = 0; inb = 1; ideg = -1;
            if (itile >= 0 && row < row_end) {
                ie0 = rp_s[r];
                ideg = rp_s[r + 1] - ie0;
                iitems = ideg;
                ilong = -1;
                if (LONG && ideg > LONG_T && lw.cap > 0) {               // hub row: [chunk partials...] if pre-aggregated
                    ilong = long_lookup(lw, row);
                    if (ilong >= 0) iitems = (ideg + LONG_CH - 1) / LONG_CH;
                }
                inb = iitems > 0 ? (iitems + QS - 1) / QS : 1;
            }
        };
        auto setup_consume_row = [&]() {                                // ci < stream_end, tile already staged
            const int tl = ci / TN, r = ci % TN;
            if (tl != ctl) ctile = tile_ids[tl % TILE_RING];
            ctl = tl;
            const unsigned char* ibp = idx_gen + (size_t)(tl % IDX_STAGES) * IDX_STAGE_BYTES;
            const int32_t* rp_s = reinterpret_cast<const int32_t*>(ibp + EPAD * 8);
            cew = reinterpret_cast<const float*>(ibp + EPAD * 4) + rp_s[96 + 3];    // + alignment offset of the ew slice
            celo = *reinterpret_cast<const int64_t*>(ibp + EPAD * 8 + 384);
            const int64_t row = row_begin + (int64_t)ctile * TN + r;
            cb = 0; cnb = 1; cdeg = -1;
            if (ctile >= 0 && row < row_end) {
                ce0 = rp_s[r];
                cdeg = rp_s[r + 1] - ce0;
                citems = cdeg;
                clong = -1;
                if (LONG && cdeg > LONG_T && lw.cap > 0) {
                    clong = long_lookup(lw, row);
                    if (clong >= 0) citems = (cdeg + LONG_CH - 1) / LONG_CH;
                }
                cnb = citems > 0 ? (citems + QS - 1) / QS : 1;
            }
        };
        // one cp.async group = sub-batch `ib` of the issue row, into ring slot `slot`
        auto issue = [&](int slot) {
            if (ii < stream_end) {
                if (ideg >= 0) {
                    const int first = ib * QS;
                    const int nitems = iitems - first;                   // items left in the row (0: a row without items)
                    const uint32_t dst = ring_u32 + (uint32_t)(slot * SLOT_FLOATS * 4);
                    const int kbase = ie0 + first;                       // item `it` of this sub-batch is edge kbase + it
                    if (!(LONG && ilong >= 0) && ie0 + ideg <= EMAX) {   // whole row staged (the common case): branch free
                        uint32_t src[QS / G];
#pragma unroll
                        for (int t = 0; t < QS; t += G) src[t / G] = (uint32_t)icol[kbase + t + grp];   // slack reads stay in smem
#pragma unroll
                        for (int t = 0; t < QS; t += G)
                            cp_async16_pred_hint(dst + (uint32_t)(t * F * 4), xs + (size_t)src[t / G] * F, t + grp < nitems, pol());
                    } else if (LONG && ilong >= 0) {                     // hub row: items are pre-aggregated chunk partials
#pragma unroll
                        for (int t = 0; t < QS; t += G) {
                            const int it = t + grp;
                            if (it < nitems)
                                cp_async16(dst + (uint32_t)(t * F * 4), lw.partial + (size_t)(ilong + first + it) * 128 + 4 * sub);
                        }
                    } else {
#pragma unroll
                        for (int t = 0; t < QS; t += G) {
                            const int it = t + grp;
                            if (it < nitems) {
                                const int k = kbase + it;
                                const uint32_t src = (uint32_t)((k < EMAX) ? icol[k] : __ldg(col + ielo + k));
                                cp_async16(dst + (uint32_t)(t * F * 4), xs + (size_t)src * F);
                            }
                        }
                    }
                }
                if (++ib >= inb) {
                    ii += GATHER_WARPS;
                    if (ii < stream_end) setup_issue_row();
                }
            }
            cp_async_commit();                                            // (possibly empty) group keeps the count in step
        };

        if (ii < stream_end) { setup_issue_row(); }
        if (ci < stream_end) { setup_consume_row(); }
        int islot = 0, cslot = 0;
#pragma unroll
        for (int d = 0; d < NQ - 1; ++d) { issue(islot); islot = (islot + 1) % NQ; }   // prologue: NQ-1 groups in flight
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float wsum = 0.f;
        int last_tl = -1;
        while (ci < stream_end) {
            cp_async_wait<NQ - 2>();                                      // oldest group landed (this lane's part) ...
            __syncwarp();                                                 // ... and everyone else's; all lanes are done
                                                                          // reading the slot consumed last iteration
            issue(islot);                                                 // refill that slot
            islot = (islot + 1) % NQ;
            if (cdeg >= 0) {
                const int first = cb * QS;
                const int nitems = citems - first;
                const float* rs = ring_gen + cslot * SLOT_FLOATS;
                const int kbase = ce0 + first;
                if (!(LONG && clong >= 0) && ce0 + cdeg <= EMAX) {       // whole row staged: batched LDS, predicated math
                    float4 v[QS / G];
                    float w[QS / G];
#pragma unroll
                    for (int t = 0; t < QS; t += G) {
                        v[t / G] = *reinterpret_cast<const float4*>(rs + t * F);
                        w[t / G] = cew[kbase + t + grp];
                    }
#pragma unroll
                    for (int t = 0; t < QS; t += G) {
                        if (t + grp < nitems) {
                            const float wt = w[t / G];
                            const float4 vt = v[t / G];
                            wsum += wt;
                            acc.x = fmaf(wt, vt.x, acc.x); acc.y = fmaf(wt, vt.y, acc.y);
                            acc.z = fmaf(wt, vt.z, acc.z); acc.w = fmaf(wt, vt.w, acc.w);
                        }
                    }
                } else {
#pragma unroll
                    for (int t = 0; t < QS; t += G) {
                        const int it = t + grp;
                        if (it < nitems) {
                            const float4 v = *reinterpret_cast<const float4*>(rs + t * F);
                            if (LONG && clong >= 0) {                    // chunk partial: already weighted
                                wsum += lw.pw[clong + first + it];
                                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                            } else {
                                const int k = kbase + it;
                                const float w = (k < EMAX) ? cew[k] : __ldg(ew + celo + k);
                                wsum += w;
                                acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
                                acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                            }
                        }
                    }
                }
            }
            cslot = (cslot + 1) % NQ;
            if (++cb < cnb) continue;

            // ---- row complete: normalise, split to bf16 terms, write the wgmma B operand, signal
            const int tl = ctl;
            const int r = ci % TN;
            const int s = tl % C::STAGES;
            if (G > 1) {                                                  // combine the G lane groups
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {
                    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
                    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
                    wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
                }
            }
            if (tl != last_tl) {                                         // first write of this warp into the stage
                mbar_wait(empty_bar(s), ((uint32_t)(tl / C::STAGES) & 1u) ^ 1u);
                last_tl = tl;
            }
            if (cdeg >= 0) {                                             // (no items: acc = wsum = 0, a zero mean)
                const float inv = 1.0f / fmaxf(wsum, 1e-12f);
                const float4 mean = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
                if (lane < LPR) {
                    unsigned char* st = smem_gen + (size_t)s * C::STAGE_BYTES;
                    uint2 parts[NS];
                    split4<NS>(mean, parts);
                    const uint32_t off = sw128_offset<TN>(r, 4 * lane);
#pragma unroll
                    for (int p = 0; p < NS; ++p) *reinterpret_cast<uint2*>(st + p * C::PART_BYTES + off) = parts[p];
                }
                fence_proxy_async();                                     // generic-proxy writes -> async proxy (wgmma)
                acc = make_float4(0.f, 0.f, 0.f, 0.f); wsum = 0.f;
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(full_bar(s));
                if ((ci + GATHER_WARPS) / TN != tl) mbar_arrive(idxe_bar(tl % IDX_STAGES));   // this warp's last row in the tile
            }
            ci += GATHER_WARPS;
            if (ci < stream_end) setup_consume_row();
        }
        cp_async_wait<0>();
      }
    } else if (warp == LOADER_WARP) {
        // =========================================================== edge-block loader
        setmaxnreg_dec<C::PRODUCER_REGS>();
        constexpr int RPW = (TN + 1 + 31) / 32;
        auto load_rp = [&](int64_t tile, int64_t (&rp)[RPW]) {          // rowptr[row0 .. row0+TN], clamped to row_end
            const int64_t row0 = row_begin + tile * TN;
#pragma unroll
            for (int k = 0; k < RPW; ++k) {
                int64_t rr = row0 + lane + 32 * k;
                if (rr > row_end) rr = row_end;
                rp[k] = (lane + 32 * k <= TN) ? (int64_t)rowptr[rr] : 0;
            }
        };
        // Software pipeline, two tiles deep and free of register copies (the loop body is instantiated twice with the roles of
        // the two rowptr register sets swapped): the atomic that claims tile t+2 and the rowptr loads of tile t+1 are issued
        // in iteration t and first needed one iteration later, so neither latency sits on the per-tile path -- at F=32 a
        // tile period is short enough that a serial loader (claim -> dependent loads -> use) would set the pace.
        unsigned craw = 0;                                               // lane 0: raw result of the claim in flight
        auto claim_issue = [&]() { if (lane == 0) craw = atomicAdd(tile_ctr, 1u); };
        auto claim_take = [&]() -> int64_t { return (int64_t)__shfl_sync(0xffffffffu, craw, 0); };
        // one iteration: stage tile `tile` (its rowptr words in rp_cur) as the CTA's tl-th tile; returns true at the end of stream
        auto body = [&](int64_t tl, int64_t tile, int64_t (&rp_cur)[RPW], int64_t& tile_nx, int64_t (&rp_nx)[RPW]) -> bool {
            const bool end = tile >= n_tiles;
            tile_nx = n_tiles;
            if (!end) {
                tile_nx = claim_take();                                  // claimed one iteration ago
                claim_issue();                                           // for the iteration after the next
                if (tile_nx < n_tiles) load_rp(tile_nx, rp_nx);          // needed in the next iteration
            }
            const int q = (int)(tl % IDX_STAGES);
            mbar_wait_relaxed(idxe_bar(q), ((uint32_t)(tl / IDX_STAGES) & 1u) ^ 1u);
            if (lane == 0) {
                tile_ids[tl % TILE_RING] = end ? -1 : (int)tile;
                if (end) *end_tl = (int)tl;                              // ordered before the closing release below
            }
            if (end) {                                                   // closing entry: no rows, no edges
                __syncwarp();
                if (lane == 0) mbar_arrive_expect_tx(idxf_bar(q), 0u);
                return true;
            }
            const int64_t e_lo = __shfl_sync(0xffffffffu, rp_cur[0], 0);
            const int64_t e_hi = __shfl_sync(0xffffffffu, rp_cur[TN / 32], TN % 32);
            unsigned char* ib = idx_gen + (size_t)q * IDX_STAGE_BYTES;
            int32_t* rp_s = reinterpret_cast<int32_t*>(ib + EPAD * 8);
#pragma unroll
            for (int k = 0; k < RPW; ++k)
                if (lane + 32 * k <= TN) rp_s[lane + 32 * k] = (int32_t)(rp_cur[k] - e_lo);
            const int n = (int)((e_hi - e_lo) < EMAX ? (e_hi - e_lo) : EMAX);
            // the col / ew slices [e_lo, e_lo + n) as the 16-byte aligned supersets bulk copies need: the slice starts
            // `off` elements into its staged array (the gather warps add it); an over-read stays inside the 16-byte
            // line that holds the first / last element
            const uintptr_t ca = reinterpret_cast<uintptr_t>(col + e_lo), wa = reinterpret_cast<uintptr_t>(ew + e_lo);
            const uint32_t c_off = (uint32_t)(ca & 15u) >> 2, w_off = (uint32_t)(wa & 15u) >> 2;
            const uint32_t c_bytes = n ? (((uint32_t)n + c_off) * 4u + 15u) & ~15u : 0u;
            const uint32_t w_bytes = n ? (((uint32_t)n + w_off) * 4u + 15u) & ~15u : 0u;
            if (lane == 0) {
                *reinterpret_cast<int64_t*>(ib + EPAD * 8 + 384) = e_lo;
                rp_s[96 + 2] = (int32_t)c_off; rp_s[96 + 3] = (int32_t)w_off;
                if constexpr (C::SELF_SPLIT) {                           // the tile's self terms, read by the consumers
                    const int64_t row0 = row_begin + tile * TN;
                    const int64_t nr = row_end - row0 < TN ? row_end - row0 : TN;
                    bulk_prefetch_l2_hint(out + row0 * UM, (uint32_t)(nr * UM * 4), pol());
                }
            }
            __syncwarp();                                                // every lane's rowptr words are written ...
            if (lane == 0) {
                const uint32_t cs = idx_base + (uint32_t)(q * IDX_STAGE_BYTES), ws = cs + EPAD * 4;
                mbar_arrive_expect_tx(idxf_bar(q), c_bytes + w_bytes);   // ... and published by this release-arrive
                if (n) {
                    if constexpr (QUAD) {
                        bulk_g2s(cs, reinterpret_cast<const void*>(ca & ~(uintptr_t)15), c_bytes, idxf_bar(q));
                        bulk_g2s(ws, reinterpret_cast<const void*>(wa & ~(uintptr_t)15), w_bytes, idxf_bar(q));
                    } else {
                        bulk_g2s_hint(cs, reinterpret_cast<const void*>(ca & ~(uintptr_t)15), c_bytes, idxf_bar(q), pol());
                        bulk_g2s_hint(ws, reinterpret_cast<const void*>(wa & ~(uintptr_t)15), w_bytes, idxf_bar(q), pol());
                    }
                }
            }
            return false;
        };
        int64_t rp_a[RPW], rp_b[RPW];
        claim_issue();
        int64_t tile_a = claim_take(), tile_b = n_tiles;
        claim_issue();                                                   // in flight for the first body()
        if (tile_a < n_tiles) load_rp(tile_a, rp_a);
        for (int64_t tl = 0;; tl += 2) {
            if (body(tl, tile_a, rp_a, tile_b, rp_b)) break;
            if (body(tl + 1, tile_b, rp_b, tile_a, rp_a)) break;
        }
    } else if (warp < EPI_WARPS) {
        // =========================================================== consumer warpgroups: wgmma + epilogue
        setmaxnreg_inc<C::CONSUMER_REGS>();
        // Warpgroup h computes output features [64 h, 64 h + 64).  Its accumulator row m = 16 wq + i (warp wq of the
        // warpgroup, i < 16) is feature 64 h + 16 wq + 2 (i & 7) + (i >> 3): a thread's two rows are two CONSECUTIVE
        // features f0, f0 + 1, so its outputs are 8-byte stores and a warp writes 64 contiguous bytes of a row.  The
        // accumulator register d[4 nb + 2 b + e] of thread (wq, lane = 4 g + c) holds feature f0 + b of tile row
        // 8 nb + 2 c + e.  The A fragments (W^T terms) come pre-split from `wsplit` (the prep kernel; F = 32:
        // split_w_kernel), 16 bytes per thread, term and K step.
        const int h = warp >> 2, wq = warp & 3, et = tid & 127;
        const int g = lane >> 2, c = lane & 3;
        const int f0 = 64 * h + 16 * wq + 2 * g;
        const float2 b2 = *reinterpret_cast<const float2*>(bias + f0);
        const float2 nw2 = node_w ? *reinterpret_cast<const float2*>(node_w + f0) : make_float2(0.f, 0.f);
        const uint4* wfr = reinterpret_cast<const uint4*>(wsplit) + (size_t)h * NS * 128 + et;   // + (2 j NS + p) * 128
        auto load_a = [&](int j, uint32_t (&a)[NS][4]) {
#pragma unroll
            for (int p = 0; p < NS; ++p) {
                const uint4 v = __ldg(wfr + (size_t)(2 * j * NS + p) * 128);
                a[p][0] = v.x; a[p][1] = v.y; a[p][2] = v.z; a[p][3] = v.w;
            }
        };
        auto self_terms = [&](int64_t t, int nb, int e) -> float2 {           // (row 8 nb + 2 c + e of tile t, f0)
            const int64_t row = row_begin + t * TN + 8 * nb + 2 * c + e;
            return row < row_end ? ld_nc_na_hint(reinterpret_cast<const float2*>(out + row * UM + f0), pol()) : make_float2(0.f, 0.f);
        };
        auto wait_full = [&](int64_t t) -> int {                              // the CTA's t-th tile id, once gathered
            mbar_wait_relaxed(full_bar((int)(t % C::STAGES)), (uint32_t)(t / C::STAGES) & 1u);
            return tile_ids[t % TILE_RING];
        };
        if constexpr (QUAD) {
            // F = 32: all of the split W^T (K = 2F: KSTEPS x NS fragments, 48 registers at NS = 3) is loaded once and stays
            // in registers, so no fragment register is ever redefined while a wgmma runs and a tile is all its products in
            // ONE commit group with one wait -- the same instructions on the same registers in the same order (scale-d 0 on
            // the first only) as one K step at a time, hence the same bits.
            uint32_t a[C::KSTEPS][NS][4];
#pragma unroll
            for (int j = 0; j < C::KSTEPS; ++j) load_a(j, a[j]);
            float d[16];
            for (int64_t tl = 0;; ++tl) {
                const int tile = wait_full(tl);
                if (tile < 0) break;                                          // closing entry: end of stream
                const int s = (int)(tl % C::STAGES);
                const uint32_t st0 = smem_base + (uint32_t)(s * C::STAGE_BYTES);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < C::KSTEPS; ++j) {
                    const uint32_t boff = (uint32_t)((j >> 2) * (TN * 128) + (j & 3) * 32);
                    uint64_t xb[NS];
#pragma unroll
                    for (int p = 0; p < NS; ++p) xb[p] = make_b_desc(st0 + (uint32_t)(p * C::PART_BYTES) + boff);   // x term p
                    wgmma_split_products<NS>(d, a[j], xb, j > 0 ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait_all();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));                     // this warp's MMAs no longer read the stage

                // ---- epilogue: + bias, ReLU, one 8-byte store per (row, thread), the fused node head (as below)
                const int64_t row0 = row_begin + (int64_t)tile * TN;
                float part[8];
#pragma unroll
                for (int nb = 0; nb < 4; ++nb) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float2 o = make_float2(d[4 * nb + e] + b2.x, d[4 * nb + 2 + e] + b2.y);
                        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                        part[2 * nb + e] = o.x * nw2.x + o.y * nw2.y;
                        const int64_t row = row0 + 8 * nb + 2 * c + e;
                        if (row < row_end) {
                            const int64_t off = row * UM + f0;
                            if (peers.mc) {
                                multimem_st2(peers.mc + off, o);
                            } else {
                                *reinterpret_cast<float2*>(out + off) = o;
                                if (peers.n) {
                                    const unsigned need = peers.need ? (unsigned)__ldg(peers.need + row) : 0xFFu;
#pragma unroll
                                    for (int pr = 0; pr < MAX_PEERS; ++pr)
                                        if (pr < peers.n && ((need >> pr) & 1u)) *reinterpret_cast<float2*>(peers.out[pr] + off) = o;
                                }
                            }
                        }
                    }
                }
                if (node_w) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        part[i] += __shfl_xor_sync(0xffffffffu, part[i], 4);
                        part[i] += __shfl_xor_sync(0xffffffffu, part[i], 8);
                        part[i] += __shfl_xor_sync(0xffffffffu, part[i], 16);
                    }
                    const int half = (int)(tl & 1);
                    float* hb = head_red + (half * EPI_WARPS + warp) * 32;
                    if (g == 0) {
#pragma unroll
                        for (int nb = 0; nb < 4; ++nb) { hb[8 * nb + 2 * c] = part[2 * nb]; hb[8 * nb + 2 * c + 1] = part[2 * nb + 1]; }
                    }
                    named_bar(1, 256);                                       // the eight consumer warps
                    if (warp == 0) {
                        const float* hr = head_red + half * EPI_WARPS * 32 + lane;
                        const float dot = ((hr[0] + hr[32]) + (hr[64] + hr[96])) + ((hr[128] + hr[160]) + (hr[192] + hr[224]));
                        if (row0 + lane < row_end) score[row0 + lane] = 1.f / (1.f + expf(-(dot + node_b)));
                    }
                }
            }
        } else {
            // F = 128 without hub rows (RESIDENT): the split W^T of the mean half (K = F: KSTEPS x NS fragments, 96 registers
            // at NS = 3) is loaded once and stays in registers, as at F = 32: no fragment register is
            // redefined while a wgmma runs, so a pass is all its products in ONE commit group with one wait.
            // F = 64, and F = 128 with hub rows: the fragments are re-read from L2 for every pass, one K step ahead of the MMAs across tile
            // boundaries (an L2 round trip under the gather's load is longer than one K step of one tile, and a K step issues
            // both tiles' MMAs); a step's MMAs are waited for before the next fragments are written, because ptxas serializes
            // the MMAs when a wgmma input register is redefined while one is in flight.
            constexpr int TP = 2;                                                 // tiles per pass
            uint32_t a[C::RESIDENT ? C::KSTEPS : 1][NS][4];                       // (with hub rows: the next K step's)
#pragma unroll
            for (int j = 0; j < (C::RESIDENT ? C::KSTEPS : 1); ++j) load_a(j, a[j]);
            // The accumulators start from the prep kernel's self terms (the first F/16 K steps), stored raw in out -- the
            // local buffer: peers and the multicast address never hold this rank's self terms.
            // TILE PAIRS: a warpgroup takes the CTA's tiles two at a time (operand stages tl and tl + 1) and issues each K
            // step's products for both tiles into two independent accumulator sets: two MMA chains the tensor pipe can
            // overlap, and one wait per 64 rows.  Each tile runs the same wgmma sequence as it would alone (same fragments,
            // same product order, scale-d 1 from its self terms), so its outputs do not depend on its partner.  A closing
            // entry (-1) in the second slot ends the stream: that pass stores only the first tile (the products over the
            // closing stage are discarded).
            // The epilogue of a pass already loads the next pass's self terms into d when the loader has published those
            // tiles' ids: the ids of a CTA's tiles increase, so a ring entry greater than the pass's last tile is a later
            // tile's, not a stale one.
            static_assert(C::STAGES % TP == 0 && C::STAGES >= 2 * TP, "operand stages per pass");
            float d[TP][16];
            int s_tile[TP];                                                       // tile whose self terms d[u] holds
#pragma unroll
            for (int u = 0; u < TP; ++u) s_tile[u] = -1;
            for (int64_t tl = 0;; tl += TP) {
                const int s0 = (int)(tl % C::STAGES);                             // stages s0 .. s0 + TP - 1
                int tile[TP];
                tile[0] = wait_full(tl);
                if (tile[0] < 0) break;                                           // closing entry: end of stream
                tile[1] = wait_full(tl + 1);                                      // (-1: the closing entry)
                if constexpr (C::SELF_SPLIT) {
#pragma unroll
                    for (int u = 0; u < TP; ++u) {
                        if (tile[u] >= 0 && tile[u] != s_tile[u]) {
#pragma unroll
                            for (int nb = 0; nb < 4; ++nb)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const float2 sv = self_terms(tile[u], nb, e);
                                    d[u][4 * nb + e] = sv.x; d[u][4 * nb + 2 + e] = sv.y;
                                }
                        }
                    }
                }
                auto pair_products = [&](int j, const uint32_t (&aj)[NS][4]) {      // K step j of both tiles
                    const uint32_t boff = (uint32_t)((j >> 2) * (TN * 128) + (j & 3) * 32);
#pragma unroll
                    for (int u = 0; u < TP; ++u) {
                        const uint32_t st0 = smem_base + (uint32_t)((s0 + u) * C::STAGE_BYTES);
                        uint64_t xb[NS];
#pragma unroll
                        for (int p = 0; p < NS; ++p) xb[p] = make_b_desc(st0 + (uint32_t)(p * C::PART_BYTES) + boff);   // x term p
                        wgmma_split_products<NS>(d[u], aj, xb, 1u);                 // (the self terms start d)
                    }
                };
                if constexpr (C::RESIDENT) {
                    wgmma_fence();
#pragma unroll
                    for (int j = 0; j < C::KSTEPS; ++j) pair_products(j, a[j]);
                    wgmma_commit();
                    wgmma_wait_all();
                } else {
    #pragma unroll 1
                    for (int j = 0; j < C::KSTEPS; ++j) {
                        uint32_t a_cur[NS][4];
#pragma unroll
                        for (int p = 0; p < NS; ++p)
#pragma unroll
                            for (int r = 0; r < 4; ++r) a_cur[p][r] = a[0][p][r];
                        load_a(j + 1 < C::KSTEPS ? j + 1 : j + 1 - C::KSTEPS, a[0]);
                        wgmma_fence();
                        pair_products(j, a_cur);
                        wgmma_commit();
                        wgmma_wait_all();
                    }
                }
                __syncwarp();
                if (lane == 0) {
#pragma unroll
                    for (int u = 0; u < TP; ++u) mbar_arrive(empty_bar(s0 + u));  // this warp's MMAs no longer read the stages
                }

                // ---- epilogue, per tile: + bias, ReLU, one 8-byte store per (row, thread)
                int s_next[TP];
#pragma unroll
                for (int u = 0; u < TP; ++u) {
                    s_next[u] = -1;
                    if constexpr (C::SELF_SPLIT) {
                        const int nx = tile_ids[(tl + TP + u) % TILE_RING];
                        if (tile[TP - 1] >= 0 && nx > tile[TP - 1]) s_next[u] = nx;
                    }
                }
#pragma unroll
                for (int u = 0; u < TP; ++u) {
                    if (tile[u] < 0) break;                                       // the closing entry in the second slot
                    const int64_t row0 = row_begin + (int64_t)tile[u] * TN;
                    float part[8];
#pragma unroll
                    for (int nb = 0; nb < 4; ++nb) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float2 o = make_float2(d[u][4 * nb + e] + b2.x, d[u][4 * nb + 2 + e] + b2.y);
                            if (C::SELF_SPLIT && s_next[u] >= 0) {
                                const float2 sv = self_terms(s_next[u], nb, e);
                                d[u][4 * nb + e] = sv.x; d[u][4 * nb + 2 + e] = sv.y;
                            }
                            if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                            part[2 * nb + e] = o.x * nw2.x + o.y * nw2.y;
                            const int64_t row = row0 + 8 * nb + 2 * c + e;
                            if (row < row_end) {
                                const int64_t off = row * UM + f0;
                                if (peers.mc) {                                   // NVSwitch multicast: every rank's buffer at once
                                    multimem_st2(peers.mc + off, o);
                                } else {
                                    if constexpr (QUAD) *reinterpret_cast<float2*>(out + off) = o;
                                    else st_hint(reinterpret_cast<float2*>(out + off), o, pol());
                                    if (peers.n) {                                // fused exchange over NVLink
                                        const unsigned need = peers.need ? (unsigned)__ldg(peers.need + row) : 0xFFu;
#pragma unroll
                                        for (int pr = 0; pr < MAX_PEERS; ++pr)
                                            if (pr < peers.n && ((need >> pr) & 1u)) *reinterpret_cast<float2*>(peers.out[pr] + off) = o;
                                    }
                                }
                            }
                        }
                    }
                    s_tile[u] = s_next[u];
                    if (node_w) {
                        // fused node head: score[row] = sigmoid(h[row,:] . node_w + node_b); a warp's 16 features summed over g.
                        // The halves of head_red alternate by tile (the first and second tile of a pass); warp 0 reads a half
                        // before it reaches the next tile's barrier, which orders that read before the half is written again.
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            part[i] += __shfl_xor_sync(0xffffffffu, part[i], 4);
                            part[i] += __shfl_xor_sync(0xffffffffu, part[i], 8);
                            part[i] += __shfl_xor_sync(0xffffffffu, part[i], 16);
                        }
                        const int half = (int)((tl + u) & 1);
                        float* hb = head_red + (half * EPI_WARPS + warp) * 32;
                        if (g == 0) {
#pragma unroll
                            for (int nb = 0; nb < 4; ++nb) { hb[8 * nb + 2 * c] = part[2 * nb]; hb[8 * nb + 2 * c + 1] = part[2 * nb + 1]; }
                        }
                        named_bar(1, 256);                                       // the eight consumer warps
                        if (warp == 0) {
                            const float* hr = head_red + half * EPI_WARPS * 32 + lane;
                            const float dot = ((hr[0] + hr[32]) + (hr[64] + hr[96])) + ((hr[128] + hr[160]) + (hr[192] + hr[224]));
                            if (row0 + lane < row_end) score[row0 + lane] = 1.f / (1.f + expf(-(dot + node_b)));
                        }
                    }
                }
                if (tile[TP - 1] < 0) break;                                      // the pass held the closing entry
            }
        }
    }
}

// W [K][128] fp32 -> the A fragment of thread t of consumer warpgroup h at K step j (W rows 16 j .. 16 j + 15), split
// into NS bf16 terms
template <int NS>
__device__ __forceinline__ void w_fragment(const float* __restrict__ W, int j, int h, int t, uint32_t (&a)[NS][4]) {
    const int wq = t >> 5, g = (t & 31) >> 2, c = t & 3;
    const int f0 = 64 * h + 16 * wq + 2 * g;
#pragma unroll
    for (int r = 0; r < 4; ++r) {                                     // register r: row g + 8 (r & 1), K pair r >> 1
        const int k = 16 * j + 2 * c + 8 * (r >> 1), f = f0 + (r & 1);
        uint32_t pp[NS];
        split_pair<NS>(W[(size_t)k * UM + f], W[(size_t)(k + 1) * UM + f], pp);
#pragma unroll
        for (int p = 0; p < NS; ++p) a[p][r] = pp[p];
    }
}
// layout the consumer role reads: wsplit[((2 j + h) NS + p) 128 + t] = uint4 of term p of thread t of warpgroup h at
// the layer kernel's K step j
template <int NS>
__device__ __forceinline__ void store_w_fragment(uint4* __restrict__ wsplit, int j, int h, int t, const uint32_t (&a)[NS][4]) {
#pragma unroll
    for (int p = 0; p < NS; ++p) wsplit[(size_t)((2 * j + h) * NS + p) * 128 + t] = make_uint4(a[p][0], a[p][1], a[p][2], a[p][3]);
}

// F = 32: all 2F/16 K steps of W, one fragment per thread
template <int NS>
__global__ void __launch_bounds__(256) split_w_kernel(const float* __restrict__ W, int ksteps, uint4* __restrict__ wsplit) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;               // (j, h, t)
    if (i >= ksteps * 2 * 128) return;
    const int t = i & 127, h = (i >> 7) & 1, j = i >> 8;
    uint32_t a[NS][4];
    w_fragment<NS>(W, j, h, t, a);
    store_w_fragment<NS>(wsplit, j, h, t, a);
}

// F = 64 / 128: the prep kernel of a layer launch.  Two jobs:
//  - the split fragments of the MEAN half of W (rows F .. 2F-1, K steps F/16 .. 2F/16-1) into wsplit, as the layer
//    kernel's K steps 0 .. F/16-1;
//  - the SELF half of the GEMM, S[v] = x_v . W[0:F] for v in [row_begin, row_end), written raw (no bias, no ReLU) into
//    out[v, :] with the consumer role's accumulator -> (row, feature) mapping.  The layer kernel loads S into its
//    accumulators and continues with the mean K steps.
// The self product runs exactly the wgmma sequence the fused [x_v || m_v] tile would have run for its first F/16 K steps
// (same split_pair terms, same m64n32k16 instructions in the same product order, scale-d 0 first), and between wgmma
// instructions the accumulator is plain fp32 in registers, so the layer's outputs are the bits of the fused K = 2F GEMM.
// Two consumer-shaped warpgroups; the self half of W stays in registers for the whole launch (96 registers per thread at
// F = 128 / NS = 3), so W is read from L2 once per CTA; x arrives in 64-row tiles (two 32-row slices sharing each A
// fragment), the next tile's rows loaded into registers while the current tile's MMAs run.  (A 3- or 4-deep cp.async
// ring of fp32 tiles, a double-buffered bf16 operand, and a second accumulator set storing tile t-1 under tile t's MMAs
// all measured no faster: the kernel moves 1 GB at F = 128.)
constexpr int PREP_ROWS = 64;
template <int F, int NS>
struct PrepCfg {
    static constexpr int KS = F / 16;                         // self K steps (= the mean half's)
    static constexpr int PART_BYTES = (F / 64) * TN * 128;    // one bf16 term of one 32-row slice
    static constexpr int SLICE_BYTES = NS * PART_BYTES;
    static constexpr int SLICES = PREP_ROWS / TN;
    static constexpr int SMEM = SLICES * SLICE_BYTES + 1024 /*align*/;
};

template <int F, int NS>
__global__ void __launch_bounds__(256, 1)
sage_self_prep_kernel(const float* __restrict__ x, const float* __restrict__ W, float* __restrict__ out, int64_t row_begin,
                      int64_t row_end, uint4* __restrict__ wsplit, int l2_policy) {
    using P = PrepCfg<F, NS>;
    const uint64_t pol = l2_policy ? l2_policy_evict_first() : l2_policy_evict_normal();   // x and S: read / written once
    constexpr int KS = P::KS, SLICES = P::SLICES;
    constexpr int LPR = F / 4;                                // float4 per x row
    constexpr int RPP = 256 / LPR;                            // rows per pass of the CTA
    constexpr int NV = PREP_ROWS / RPP;                       // float4 per thread and tile
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;         // SWIZZLE_128B needs 1024-B alignment
    unsigned char* gen = smem_dyn + (base - smem_u32(smem_dyn));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h = warp >> 2, wq = warp & 3, et = tid & 127;
    const int g = lane >> 2, c = lane & 3;
    const int f0 = 64 * h + 16 * wq + 2 * g;

    for (int j = blockIdx.x; j < KS; j += gridDim.x) {
        uint32_t a[NS][4];
        w_fragment<NS>(W, KS + j, h, et, a);
        store_w_fragment<NS>(wsplit, j, h, et, a);
    }
    uint32_t a[KS][NS][4];
#pragma unroll
    for (int j = 0; j < KS; ++j) w_fragment<NS>(W, j, h, et, a[j]);

    const int q = tid % LPR, r0 = tid / LPR;
    const int64_t n_tiles = (row_end - row_begin + PREP_ROWS - 1) / PREP_ROWS;
    float4 v[NV];
    auto load = [&](int64_t tile) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int64_t row = row_begin + tile * PREP_ROWS + r0 + RPP * i;
            v[i] = (tile < n_tiles && row < row_end) ? ld_nc_na_hint(reinterpret_cast<const float4*>(x + row * F) + q, pol)
                                                      : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    load(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        __syncthreads();                                      // both warpgroups' MMAs of the last tile have retired
#pragma unroll
        for (int i = 0; i < NV; ++i) {                        // bf16 terms into the swizzled K-major slices
            const int r = r0 + RPP * i;
            uint2 parts[NS];
            split4<NS>(v[i], parts);
            const uint32_t off = (uint32_t)((r / TN) * P::SLICE_BYTES) + sw128_offset<TN>(r % TN, 4 * q);
#pragma unroll
            for (int p = 0; p < NS; ++p) *reinterpret_cast<uint2*>(gen + p * P::PART_BYTES + off) = parts[p];
        }
        fence_proxy_async();                                  // generic-proxy writes -> async proxy (wgmma)
        __syncthreads();
        load(tile + gridDim.x);                               // in flight under the MMAs and the stores

        float d[SLICES][16];
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < KS; ++j) {
            const uint32_t boff = (uint32_t)((j >> 2) * (TN * 128) + (j & 3) * 32);
#pragma unroll
            for (int sl = 0; sl < SLICES; ++sl) {
                uint64_t xb[NS];
#pragma unroll
                for (int p = 0; p < NS; ++p) xb[p] = make_b_desc(base + (uint32_t)(sl * P::SLICE_BYTES + p * P::PART_BYTES) + boff);
                wgmma_split_products<NS>(d[sl], a[j], xb, j > 0 ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait_all();

        const int64_t row0 = row_begin + tile * PREP_ROWS;
#pragma unroll
        for (int sl = 0; sl < SLICES; ++sl)
#pragma unroll
            for (int nb = 0; nb < 4; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int64_t row = row0 + TN * sl + 8 * nb + 2 * c + e;
                    if (row < row_end)
                        st_hint(reinterpret_cast<float2*>(out + row * UM + f0), make_float2(d[sl][4 * nb + e], d[sl][4 * nb + 2 + e]), pol);
                }
    }
}

// per-device ring of launch-private tile counters (1 KB, allocated on first use and kept): a launch zeroes its slot on its
// own stream, so launches on different streams do not share a counter unless 256 of them are in flight at once
inline unsigned* tile_counter_slot(cudaStream_t st) {
    static unsigned* ring[64] = {};
    static unsigned next[64] = {};
    int dev_ = 0;
    cudaGetDevice(&dev_);
    dev_ &= 63;
    if (!ring[dev_] && cudaMalloc((void**)&ring[dev_], 256 * sizeof(unsigned)) != cudaSuccess) return nullptr;
    unsigned* slot = ring[dev_] + (__atomic_fetch_add(&next[dev_], 1u, __ATOMIC_RELAXED) & 255u);
    if (cudaMemsetAsync(slot, 0, sizeof(unsigned), st) != cudaSuccess) return nullptr;
    return slot;
}

// Scratch for the split W^T of one launch (192 KB at F=128, three terms), one buffer per (device, stream), allocated on
// the stream's first launch and kept: launches on one stream run in order, so each one re-splits its weights into the
// buffer the previous one has finished with, and the layer launches themselves allocate nothing.
constexpr size_t WSPLIT_MAX_BYTES = (size_t)(2 * 128 / 16) * 2 * 3 * 128 * sizeof(uint4);
inline uint4* wsplit_buffer(cudaStream_t st) {
    static std::mutex mu;
    static std::map<std::pair<int, cudaStream_t>, uint4*> bufs;
    int dev_ = 0;
    if (cudaGetDevice(&dev_) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    uint4*& buf = bufs[std::make_pair(dev_, st)];
    if (!buf && cudaMalloc((void**)&buf, WSPLIT_MAX_BYTES) != cudaSuccess) buf = nullptr;
    return buf;
}

template <int F, int NS, typename RP>
int launch_umma(const float* x, const RP* rowptr, const int32_t* col, const float* ew, const float* W, const float* b,
                float* out, int64_t row_begin, int64_t row_end, int relu, const float* node_w, float node_b, float* score,
                void* long_ws, size_t long_ws_bytes, bool reuse_scan, const Peers& peers, int l2_policy, cudaStream_t st) {
    using C = UmmaCfg<F, NS, false>;
    using CL = UmmaCfg<F, NS, true>;                                     // with hub-row scratch
    int rc = set_max_dynamic_smem((const void*)sage_layer_umma_kernel<F, NS, RP, false>, C::SMEM);
    if (!rc) rc = set_max_dynamic_smem((const void*)sage_layer_umma_kernel<F, NS, RP, true>, CL::SMEM);
    if (rc) return rc;
    const int64_t rows = row_end - row_begin;
    const int64_t tiles = (rows + TN - 1) / TN;
    if (tiles == 0) return NERRF_OK;
    LongWs lw = long_ws_carve(long_ws, long_ws_bytes);
    if (lw.cap > 0) {
        // hub-row pre-pass: clear header + hash, mark the queue empty, find long rows, aggregate their chunks
        const int sms = sm_count();
        if (!reuse_scan) {       // the scan (hub-row list, hash, chunk queue) depends on the graph only, not on x
            const size_t hash_bytes = (size_t)(lw.hash_mask + 1) * 8;
            NERRF_CHECK_CUDA(cudaMemsetAsync(lw.hdr, 0, 256 + hash_bytes, st));
            NERRF_CHECK_CUDA(cudaMemsetAsync(lw.queue, 0xFF, (size_t)lw.cap * 8, st));
            long_scan_kernel<RP><<<sms * 4, 256, 0, st>>>(rowptr, row_begin, row_end, lw);
        }
        long_chunk_kernel<F, RP><<<sms * 4, 256, 0, st>>>(x, rowptr, col, ew, lw);
        rc = launch_status("long-row pre-pass");
        if (rc) return rc;
    }
    const int64_t grid = tiles < sm_count() ? tiles : sm_count();
    unsigned* tile_ctr = tile_counter_slot(st);
    if (!tile_ctr) { set_error("could not allocate the tile counter"); return NERRF_ERR_CUDA; }
    // W^T split into bf16 terms in fragment order, once per launch (the weights may have changed in place since the last
    // one); at F = 64 / 128 by the prep kernel, which also writes the self terms into out
    static_assert((size_t)C::KSTEPS * 2 * NS * 128 * sizeof(uint4) <= WSPLIT_MAX_BYTES, "split W scratch");
    uint4* wsplit = wsplit_buffer(st);
    if (!wsplit) { set_error("could not allocate the split-weight scratch"); return NERRF_ERR_CUDA; }
    if constexpr (C::SELF_SPLIT) {
        using P = PrepCfg<F, NS>;
        rc = set_max_dynamic_smem((const void*)sage_self_prep_kernel<F, NS>, P::SMEM);
        if (rc) return rc;
        const int64_t ptiles = (rows + PREP_ROWS - 1) / PREP_ROWS;
        sage_self_prep_kernel<F, NS><<<(unsigned)(ptiles < sm_count() ? ptiles : sm_count()), 256, P::SMEM, st>>>(x, W, out, row_begin, row_end, wsplit,
                                                                                                            l2_policy);
    } else {
        split_w_kernel<NS><<<(C::KSTEPS * 2 * 128 + 255) / 256, 256, 0, st>>>(W, C::KSTEPS, wsplit);
    }
    // the col / ew slices are staged with bulk copies, which only need 4-byte aligned slices (the aligned superset is copied)
    if (lw.cap > 0)
        sage_layer_umma_kernel<F, NS, RP, true><<<(unsigned)grid, CL::THREADS, CL::SMEM, st>>>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu, node_w, node_b, score, lw, peers, tile_ctr, wsplit, l2_policy);
    else
        sage_layer_umma_kernel<F, NS, RP, false><<<(unsigned)grid, C::THREADS, C::SMEM, st>>>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu, node_w, node_b, score, lw, peers, tile_ctr, wsplit, l2_policy);
    return launch_status("sage_layer_umma_kernel");
}

}  // namespace

int sage_layer_umma(const float* x, const void* rowptr, int is64, const int32_t* col, const float* ew, const float* W,
                    const float* b, float* out, int64_t n_nodes, int64_t row_begin, int64_t row_end, int F, int relu,
                    int nsplit, const float* node_w, float node_b, float* score, void* long_ws, size_t long_ws_bytes,
                    bool reuse_scan, float* const* peer_out, int n_peers, const uint8_t* peer_need, int l2_policy,
                    cudaStream_t st) {
    (void)n_nodes;
    Peers peers{};
    peers.need = peer_need;
    if (n_peers == -1) {                      // peer_out[0] is a multicast address covering every rank's buffer
        peers.mc = peer_out[0];
    } else {
        if (n_peers < 0 || n_peers > MAX_PEERS) { set_error("n_peers must be -1 (multicast) or 0..%d", MAX_PEERS); return NERRF_ERR_INVALID; }
        for (int i = 0; i < n_peers; ++i) peers.out[i] = peer_out[i];
        peers.n = n_peers;
    }
#define GO(FV, NSV)                                                                                                                                                                               \
    return is64 ? launch_umma<FV, NSV, int64_t>(x, (const int64_t*)rowptr, col, ew, W, b, out, row_begin, row_end, relu, node_w, node_b, score, long_ws, long_ws_bytes, reuse_scan, peers, l2_policy, st) \
                : launch_umma<FV, NSV, int32_t>(x, (const int32_t*)rowptr, col, ew, W, b, out, row_begin, row_end, relu, node_w, node_b, score, long_ws, long_ws_bytes, reuse_scan, peers, l2_policy, st)
    if (nsplit == 3) {
        switch (F) {
            case 32: GO(32, 3);
            case 64: GO(64, 3);
            case 128: GO(128, 3);
        }
    } else if (nsplit == 2) {
        switch (F) {
            case 32: GO(32, 2);
            case 64: GO(64, 2);
            case 128: GO(128, 2);
        }
    }
#undef GO
    set_error("tensor-core layer: unsupported feature width F=%d / split %d (supported: F in 32, 64, 128; split 2 or 3)", F, nsplit);
    return NERRF_ERR_INVALID;
}

}  // namespace nerrf
