// BiLSTM on Hopper tensor cores (wgmma), sm_90a -- lstm.forward (SURVEY.md 8a row a4).
//
// One LSTM layer-direction step is   gates[4H, seqs] = G_x[:, t] + W_hh[4H, H] . h_{t-1}[H, seqs]   followed by the cell
// update.  Everything that multiplies a weight matrix runs on wgmma: the weight slice is the A operand, register
// fragments read from L2 and split into three bf16 terms (six products per K step: fp32-equivalent accuracy, same
// scheme as sage_umma.cu), and the activations are the B operand, bulk-copied (cp.async.bulk, byte-counting mbarrier)
// from a global-memory OPERAND IMAGE -- the exact byte layout wgmma reads (K-major, SWIZZLE_128B, three bf16 planes):
//
//   image of a time-major activation X[t][b][K]:   tile (t, bt = b / 64, khalf):  [plane 3][kblock KB][row 64][128 B]
//
//   * lstm_image_kernel     layer-1 input seq [B,T,D] -> image (K padded to 64, one K block)
//   * lstm_proj_kernel      input projection G_x = X W_ih^T (+ b) for all (t, b): persistent CTAs, each owns ONE
//                           (direction, gate slice) of W_ih^T (one K half of 256) and streams 64-row tiles of the image
//                           through a two-stage bulk-copy pipeline into one consumer warpgroup
//   * lstm_rec_kernel       the recurrence.  W_hh (1024 x 256) is cut into 8 slices of 128 gate rows (4 gates x 32 units);
//                           8 CTAs (one per slice) form a GROUP that advances tiles of 64 sequences of one direction.
//                           Per step every CTA computes gates^T[128, 64] = G_x[:, t] + W_slice . h_{t-1}^T in the
//                           registers of a warpgroup, applies the activations, updates c / h in registers, splits the
//                           new h into its three bf16 terms and stores them INTO THE LAYER'S OUTPUT IMAGE (tile (t, bt,
//                           khalf = direction)) -- which is at once the next layer's projection operand and the h_{t}
//                           exchange between the 8 CTAs: after one release-increment of the group's counter every CTA
//                           bulk-copies the whole 96 KB tile back as its next B operand.  The step is a latency chain
//                           (MMA -> cell update -> publish -> poll -> 96 KB copy -> MMA), so every CTA works on TWO
//                           tiles at once (two operand buffers, one warpgroup each).
//
// Groups are independent (no grid barrier): group g owns direction g & 1.  The 8 CTAs of a group must be co-resident:
// cooperative launch, one CTA per SM, grid = 8 * G <= #SMs.  Every wait is bounded and ends in a trap, never a hang.
#include <cuda_bf16.h>
#include <stdlib.h>
#include "common.cuh"
#include "ptx.cuh"

namespace nerrf {

namespace {

constexpr int LH = 256;                 // hidden size
constexpr int NSEQ = 64;                // sequences per tile = wgmma N
constexpr int SLICES = 8;               // CTAs per group
constexpr int UM = 128;                 // gate rows per slice = two wgmma M=64 halves
constexpr int NS = 3;                   // bf16 terms per fp32 value
constexpr int KB_H = LH / 64;           // 128-byte K blocks of a 256-wide operand
constexpr int KSTEPS_H = LH / 16;
constexpr int PLANE_BYTES_H = KB_H * NSEQ * 128;     // 32 KB: one bf16 plane of a [64 rows, 256] tile
constexpr int TILE_BYTES_H = NS * PLANE_BYTES_H;     // 96 KB

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// activations: |abs error| ~ 2e-7 (ex2.approx + rcp), far inside the 1e-4 spec bound; tanh(x) = 2 sigmoid(2x) - 1
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return fmaf(2.0f, sigmoid_fast(2.0f * x), -1.0f); }

// Fragment layout shared by both kernels (one warpgroup, thread = (warp w, lane = 4 g + c)): accumulator row m of half h
// (m = 16 w + i) holds slice column 32 w + 4 (i & 7) + 2 h + (i >> 3), so a thread's four rows are the four CONSECUTIVE
// slice columns f0 .. f0 + 3 (f0 = 32 w + 4 g) -- with the slice packing of pack_slices_kernel, the gates i, f, g, o of
// hidden unit 8 w + g.  Its accumulator registers d[h][4 nb + 2 b + e] hold column f0 + 2 h + b, tile row 8 nb + 2 c + e.
//
// D[128, 64] (+)= W[128, K] . X[64, K]^T for one 64-row tile: W^T fragments are read from the fp32 slice [K][128] (L2)
// and split into three bf16 terms per K step (six products: fp32-equivalent), X's three planes are in shared memory.
template <int KSTEPS>
__device__ __forceinline__ void mma_tile(float (&d)[2][32], const float* __restrict__ W, uint32_t x_smem, uint32_t plane_bytes,
                                         bool accumulate_first, int warp, int lane) {
    const int g = lane >> 2, c = lane & 3;
    const float* wsrc = W + (size_t)(2 * c) * UM + warp * 32 + 4 * g;
    auto load_w = [&](int j, float4 (&q)[4]) {
        const float* p = wsrc + (size_t)(16 * j) * UM;
        q[0] = __ldg(reinterpret_cast<const float4*>(p));
        q[1] = __ldg(reinterpret_cast<const float4*>(p + UM));
        q[2] = __ldg(reinterpret_cast<const float4*>(p + 8 * UM));
        q[3] = __ldg(reinterpret_cast<const float4*>(p + 9 * UM));
    };
    auto comp = [](const float4& v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w)); };
    float4 q[4];
    load_w(0, q);
#pragma unroll 1
    for (int j = 0; j < KSTEPS; ++j) {
        uint32_t wa[2][NS][4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int r = 0; r < 4; ++r) {                 // fragment register r: row g + 8 (r & 1), k pair r >> 1
                const int kq = (r >> 1) * 2;
                uint32_t pp[NS];
                split_pair(comp(q[kq], 2 * h + (r & 1)), comp(q[kq + 1], 2 * h + (r & 1)), pp);
#pragma unroll
                for (int p = 0; p < NS; ++p) wa[h][p][r] = pp[p];
            }
        if (j + 1 < KSTEPS) load_w(j + 1, q);
        const uint32_t boff = (uint32_t)((j >> 2) * (NSEQ * 128) + (j & 3) * 32);
        uint64_t xb[NS];
#pragma unroll
        for (int p = 0; p < NS; ++p) xb[p] = make_b_desc(x_smem + (uint32_t)p * plane_bytes + boff);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            wgmma_rs(d[h], wa[h][0], xb[0], (j > 0 || accumulate_first) ? 1u : 0u);
            wgmma_rs(d[h], wa[h][0], xb[1], 1u);
            wgmma_rs(d[h], wa[h][1], xb[0], 1u);
            wgmma_rs(d[h], wa[h][1], xb[1], 1u);
            wgmma_rs(d[h], wa[h][0], xb[2], 1u);
            wgmma_rs(d[h], wa[h][2], xb[0], 1u);
        }
        wgmma_commit();
        wgmma_wait_all();                                  // the fragments are rewritten next step
    }
}

// ================================================================================================ layer-1 input image
// seq [B, T, D] fp32 -> image tiles (t, bt): [plane 3][1 K block][64 rows][128 B], K padded to 64, rows past B zero
__global__ void lstm_image_kernel(const float* __restrict__ seq, int D, int64_t B, int T, int64_t n_bt, unsigned char* __restrict__ img) {
    constexpr int TILE = NS * NSEQ * 128;                            // 24 KB
    const int64_t total = (int64_t)T * n_bt * NSEQ * 32;             // one thread per (t, bt, row, k pair)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int kp = (int)(i & 31);
        const int r = (int)((i >> 5) % NSEQ);
        const int64_t tile = i / (32 * NSEQ);
        const int64_t t = tile / n_bt, bt = tile % n_bt;
        const int64_t b = bt * NSEQ + r;
        float a = 0.f, c = 0.f;
        if (b < B) {
            const float* s = seq + ((size_t)b * T + t) * D;
            if (2 * kp < D) a = s[2 * kp];
            if (2 * kp + 1 < D) c = s[2 * kp + 1];
        }
        uint32_t pp[NS];
        split_pair(a, c, pp);
        unsigned char* dst = img + (size_t)tile * TILE + (r * 128 + ((((kp >> 2) ^ (r & 7)) << 4) | ((kp & 3) << 2)));
#pragma unroll
        for (int p = 0; p < NS; ++p) *reinterpret_cast<uint32_t*>(dst + p * (NSEQ * 128)) = pp[p];
    }
}

// ================================================================================================ input projection
// G[dir][slice][row = t*Bp + b][128] = X_tile . W_ih^T slice (+ bias), for one K range of KB 64-wide blocks.
//   img       activation image; tile (t, bt) = the K range starts at img + tile * tile_stride + k_off
//   wih       [16 combos = dir*8 + slice][K = 64*KB][128] fp32 (packed by pack_slices_kernel), bias [16][128] or nullptr
struct ProjArgs {
    const unsigned char* img;
    size_t tile_stride;        // bytes between consecutive (t, bt) tiles
    size_t k_off;              // byte offset of this K range inside a tile
    const float* wih;
    const float* bias;
    float* gx;                 // [16][T*Bp][128]
    int64_t n_tiles;           // T * n_bt
    int64_t rows_total;        // T * Bp
    int ctas_per_combo;
};

constexpr int PROJ_THREADS = 160;                   // warps 0-3: wgmma + epilogue, warp 4: loader

template <int KB>
__global__ void __launch_bounds__(PROJ_THREADS, 1) lstm_proj_kernel(ProjArgs P) {
    constexpr int K = 64 * KB, KSTEPS = K / 16;
    constexpr int PLANE = KB * NSEQ * 128, TILE = NS * PLANE;       // bytes of one (tile, K range)
    constexpr int STAGES = 2;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + STAGES * TILE;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int combo = blockIdx.x / P.ctas_per_combo, j0 = blockIdx.x % P.ctas_per_combo;
    if (warp == 4) {
        if (lane == 0) {
            for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4); }
            fence_barrier_init();
        }
        __syncwarp();
    }
    __syncthreads();

    const int64_t n_mine = j0 < P.n_tiles ? (P.n_tiles - j0 + P.ctas_per_combo - 1) / P.ctas_per_combo : 0;
    if (warp == 4) {
        if (lane == 0) {
            for (int64_t i = 0; i < n_mine; ++i) {
                const int s = (int)(i % STAGES);
                mbar_wait_bounded(empty_bar(s), ((uint32_t)(i / STAGES) & 1u) ^ 1u);
                const unsigned char* src = P.img + (size_t)(j0 + i * P.ctas_per_combo) * P.tile_stride + P.k_off;
                mbar_arrive_expect_tx(full_bar(s), (uint32_t)TILE);
                constexpr int CH = 8192;                                 // divides both tile sizes (24 KB, 96 KB)
                static_assert(TILE % CH == 0, "tile must be a whole number of bulk copies");
#pragma unroll 1
                for (int c = 0; c < TILE / CH; ++c)
                    bulk_g2s(smem_base + (uint32_t)(s * TILE + c * CH), src + (size_t)c * CH, (uint32_t)CH, full_bar(s));
            }
        }
    } else {
        const int g = lane >> 2, c = lane & 3;
        const int f0 = warp * 32 + 4 * g;
        const float4 b4 = P.bias ? *reinterpret_cast<const float4*>(P.bias + (size_t)combo * UM + f0) : make_float4(0.f, 0.f, 0.f, 0.f);
        float* gout = P.gx + (size_t)combo * P.rows_total * UM + f0;
        const float* W = P.wih + (size_t)combo * K * UM;
        for (int64_t i = 0; i < n_mine; ++i) {
            const int s = (int)(i % STAGES);
            mbar_wait_bounded(full_bar(s), (uint32_t)(i / STAGES) & 1u);
            float d[2][32];
            mma_tile<KSTEPS>(d, W, smem_base + (uint32_t)(s * TILE), (uint32_t)PLANE, false, warp, lane);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));                    // this warp's MMAs no longer read the stage
            const int64_t row0 = (j0 + i * P.ctas_per_combo) * NSEQ;      // rows of the padded time-major matrix
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float4 o = make_float4(d[0][4 * nb + e] + b4.x, d[0][4 * nb + 2 + e] + b4.y,
                                                 d[1][4 * nb + e] + b4.z, d[1][4 * nb + 2 + e] + b4.w);
                    *reinterpret_cast<float4*>(gout + (size_t)(row0 + 8 * nb + 2 * c + e) * UM) = o;
                }
        }
    }
}

// ================================================================================================ recurrence
// One warpgroup per tile slot (two slots per CTA, so that one tile's MMAs run while the other waits for its exchange).
// Per step the warpgroup loads G_x[:, t] into its accumulators, adds W_slice . h_{t-1} (wgmma, h_{t-1} bulk-copied into
// its operand buffer), applies the cell update in registers -- a thread holds the four gates of one hidden unit for 16
// sequences -- and stores h_t's three bf16 terms into the layer's output image, then publishes the step.
constexpr int REC_THREADS = 256;
constexpr size_t REC_SMEM = (size_t)2 * TILE_BYTES_H + 2 * NSEQ * 4 + 1024 /*align*/ + 128 /*barriers*/;
static_assert(REC_SMEM <= 227 * 1024, "shared memory budget");

struct RecArgs {
    const float* gx_a;        // [2 dirs * 8 slices][Rp = T*Bp rows][128]: first K range of the input projection + bias
    const float* gx_b;        // second K half, or nullptr
    const float* whh;         // [2 dirs * 8 slices][256 (k)][128 (gate row in slice)]
    const int32_t* len;       // [B]
    unsigned char* out_img;   // output image: tile (t, bt) at (t*n_bt + bt) * 2*TILE_BYTES_H, K half = direction
    float* hfin;              // [B][512]
    unsigned* counter;        // [groups][2 slots], zero at launch
    int64_t B, Bp, n_bt;
    int T;
    int groups;
};

__global__ void __launch_bounds__(REC_THREADS, 1) lstm_rec_kernel(RecArgs P) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    unsigned char* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    int* len_s = reinterpret_cast<int*>(smem_gen + 2 * TILE_BYTES_H);                              // [2 slots][64]
    const uint32_t bar_base = smem_base + 2 * TILE_BYTES_H + 2 * NSEQ * 4;
    auto opfull_bar = [&](int s) { return bar_base + 8u * s; };

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int group = blockIdx.x / SLICES, slice = blockIdx.x % SLICES;
    const int dir = group & 1;
    const int groups_dir = P.groups >> 1;                          // groups per direction
    const int gd = group >> 1;                                     // this group's index inside its direction
    if (tid == 0) {
        for (int s = 0; s < 2; ++s) mbar_init(opfull_bar(s), 1);  // one arrive (+ the bulk copies' transaction bytes)
        fence_barrier_init();
    }
    __syncthreads();

    const int slot = warp >> 2, wq = warp & 3;
    const int et = wq * 32 + lane;                                 // thread index inside the slot's warpgroup
    const int g = lane >> 2, c = lane & 3;
    const int unit = wq * 8 + g;                                   // hidden unit (inside the slice) of this thread
    const int ucol = slice * 32 + unit;
    const int f0 = wq * 32 + 4 * g;                                // its gate columns i, f, g, o in the packed slice
    const int bar_id = 1 + slot;
    const int64_t Rp = (int64_t)P.T * P.Bp;
    const float* gxa = P.gx_a + (size_t)(dir * SLICES + slice) * Rp * UM + f0;
    const float* gxb = P.gx_b ? P.gx_b + (size_t)(dir * SLICES + slice) * Rp * UM + f0 : nullptr;
    const float* whh = P.whh + (size_t)(dir * SLICES + slice) * LH * UM;
    int* ls = len_s + slot * NSEQ;
    unsigned* counter = P.counter + (size_t)group * 2 + slot;
    const uint32_t op_u32 = smem_base + (uint32_t)(slot * TILE_BYTES_H);
    // tile sequence of (group, slot): bt = gd + (2 * i + slot) * groups_dir, i = 0, 1, ...
    const int64_t first = gd + (int64_t)slot * groups_dir;
    const int64_t items = first < P.n_bt ? (P.n_bt - first + 2 * groups_dir - 1) / (2 * groups_dir) : 0;
    uint32_t q = 0, fetched = 0;                                   // steps published / operand fetches waited for
    for (int64_t it = 0; it < items; ++it) {
        const int64_t bt = gd + (2 * it + slot) * groups_dir;
        const int64_t b0 = bt * NSEQ;
        named_bar(bar_id, 128);                                    // the previous tile's last reads of ls are done
        if (et < NSEQ) { const int64_t b = b0 + et; ls[et] = b < P.B ? P.len[b] : 0; }
        named_bar(bar_id, 128);
        float c_reg[16], h_reg[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) { c_reg[j] = 0.f; h_reg[j] = 0.f; }
        for (int step = 0; step < P.T; ++step, ++q) {
            const int t = dir ? (P.T - 1 - step) : step;
            // ---- accumulator <- G_x[:, t] (rows of the padded time-major matrix: always in range)
            float d[2][32];
            const size_t rbase = (size_t)((int64_t)t * P.Bp + b0) * UM;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const size_t off = rbase + (size_t)(8 * nb + 2 * c + e) * UM;
                    float4 v = __ldg(reinterpret_cast<const float4*>(gxa + off));
                    if (gxb) {
                        const float4 w = __ldg(reinterpret_cast<const float4*>(gxb + off));
                        v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
                    }
                    d[0][4 * nb + e] = v.x; d[0][4 * nb + 2 + e] = v.y; d[1][4 * nb + e] = v.z; d[1][4 * nb + 2 + e] = v.w;
                }
            // ---- + W_slice . h_{t-1} (h_{-1} = 0: the first step is G_x alone)
            if (step > 0) {
                mbar_wait_bounded(opfull_bar(slot), fetched & 1u);
                ++fetched;
                mma_tile<KSTEPS_H>(d, whh, op_u32, (uint32_t)PLANE_BYTES_H, true, wq, lane);
            }
            // ---- cell update in registers; h (state, kept when masked) -> three bf16 terms -> output image = exchange.
            // Masked positions of the layer output are never read by the next layer (its own steps are masked there).
            unsigned char* tile = P.out_img + ((size_t)t * P.n_bt + bt) * (2 * TILE_BYTES_H) + (size_t)dir * TILE_BYTES_H;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = 8 * nb + 2 * c + e;                  // sequence inside the tile
                    const int j = 2 * nb + e;
                    if (t < ls[n]) {
                        const float ig = sigmoid_fast(d[0][4 * nb + e]), fg = sigmoid_fast(d[0][4 * nb + 2 + e]);
                        const float gg = tanh_fast(d[1][4 * nb + e]), og = sigmoid_fast(d[1][4 * nb + 2 + e]);
                        c_reg[j] = fmaf(fg, c_reg[j], ig * gg);
                        h_reg[j] = og * tanh_fast(c_reg[j]);
                    }
                    float r = h_reg[j];
                    uint32_t term[NS];
#pragma unroll
                    for (int p = 0; p < NS; ++p) {
                        const __nv_bfloat16 hb = __float2bfloat16_rn(r);
                        term[p] = (uint32_t)__bfloat16_as_ushort(hb);
                        r -= __bfloat162float(hb);
                    }
                    unsigned char* dstp = tile + sw128_offset<NSEQ>(n, ucol);
#pragma unroll
                    for (int p = 0; p < NS; ++p) {                      // units (even, odd) = lanes (l, l + 4): one 4-byte store
                        const uint32_t nbv = __shfl_down_sync(0xffffffffu, term[p], 4);
                        if (!(g & 1)) *reinterpret_cast<uint32_t*>(dstp + p * PLANE_BYTES_H) = term[p] | (nbv << 16);
                    }
                }
            fence_proxy_async_all();                                  // generic stores above are read by bulk (async-proxy) copies
            named_bar(bar_id, 128);                                   // the whole slice of h_t is written, every MMA has retired
            if (et == 0) {
                __threadfence();
                atomicAdd(counter, 1u);                               // release: this CTA's h_t slice is published
                if (step + 1 < P.T) {
                    // every CTA of the group has published this step: fetch the whole h_t tile as the next B operand
                    const unsigned want = (unsigned)SLICES * (q + 1);
                    for (uint32_t spin = 0; ld_acquire(counter) < want; ++spin) {
                        if (spin > 64) __nanosleep(32);
                        if (spin > (1u << 25)) __trap();
                    }
                    fence_proxy_async_all();                          // acquired generic writes -> async-proxy reads
                    mbar_arrive_expect_tx(opfull_bar(slot), (uint32_t)TILE_BYTES_H);
#pragma unroll 1
                    for (int i = 0; i < TILE_BYTES_H / 16384; ++i)
                        bulk_g2s(op_u32 + (uint32_t)(i * 16384), tile + (size_t)i * 16384, 16384u, opfull_bar(slot));
                }
            }
        }
        // final state of the tile
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int64_t b = b0 + 8 * (j >> 1) + 2 * c + (j & 1);
            if (b < P.B) P.hfin[b * (2 * LH) + dir * LH + ucol] = h_reg[j];
        }
    }
}

// ---------------------------------------------------------------- packing kernels
// Wt [K_src, 1024] (k-major, gate row = w*256 + unit) -> [8 slices][K_dst][128], slice column = 4 u + w (the four gates
// of one unit side by side):  dst[s][k][4u+w] = (k < k_real) ? Wt[(k_lo + k) * 1024 + w*256 + s*32 + u] : 0
__global__ void pack_slices_kernel(const float* __restrict__ Wt, int k_lo, int k_real, int K_dst, float* __restrict__ dst) {
    const int total = SLICES * K_dst * UM;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int j = i % UM, k = (i / UM) % K_dst, s = i / (UM * K_dst);
        const int g = (j & 3) * LH + s * 32 + (j >> 2);
        dst[i] = k < k_real ? Wt[(size_t)(k_lo + k) * (4 * LH) + g] : 0.f;
    }
}
__global__ void pack_bias_kernel(const float* __restrict__ bias, float* __restrict__ dst) {      // [8][128]
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < SLICES * UM) {
        const int j = i % UM, s = i / UM;
        dst[i] = bias[(j & 3) * LH + s * 32 + (j >> 2)];
    }
}

struct Ws {
    size_t gxa, gxb, img0, img_a, img_b, wih, whh, bias, counter, total;
};
inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }
Ws carve(int64_t B, int T, int num_layers) {
    const int64_t n_bt = (B + NSEQ - 1) / NSEQ;
    const size_t Rp = (size_t)T * n_bt * NSEQ;
    const size_t tiles = (size_t)T * n_bt;
    Ws w{};
    size_t o = 0;
    w.gxa = o; o += up256(2 * SLICES * Rp * UM * 4);
    w.gxb = o; o += up256(num_layers > 1 ? 2 * SLICES * Rp * UM * 4 : 0);
    w.img0 = o; o += up256(tiles * NS * NSEQ * 128);                 // layer-1 input image (K = 64)
    w.img_a = o; o += up256(tiles * 2 * TILE_BYTES_H);               // layer outputs, ping-pong
    w.img_b = o; o += up256(num_layers > 1 ? tiles * 2 * TILE_BYTES_H : 0);
    w.wih = o; o += up256((size_t)2 * SLICES * LH * UM * 4);         // one K range of both directions
    w.whh = o; o += up256((size_t)2 * SLICES * LH * UM * 4);
    w.bias = o; o += up256((size_t)2 * SLICES * UM * 4);
    w.counter = o; o += 1024;
    w.total = o;
    return w;
}
int groups_for_device() {
    int g = sm_count() / SLICES;
    g &= ~1;                                         // groups alternate directions
    return g < 2 ? 0 : g;
}

template <int KB>
int launch_proj(const ProjArgs& a, cudaStream_t st) {
    constexpr size_t smem = (size_t)2 * NS * KB * NSEQ * 128 + 1024 + 128;
    const int rc = set_max_dynamic_smem((const void*)lstm_proj_kernel<KB>, smem);
    if (rc) return rc;
    lstm_proj_kernel<KB><<<16 * a.ctas_per_combo, PROJ_THREADS, smem, st>>>(a);
    return launch_status("lstm_proj_kernel");
}

}  // namespace

// NERRF_LSTM_ALGO=ffma selects the fp32 CUDA-core kernel of lstm.cu (kept as an independent cross-check of this path)
bool lstm_umma_enabled() {
    const char* e = getenv("NERRF_LSTM_ALGO");
    return !(e && (e[0] == 'f' || e[0] == 'F'));
}

size_t lstm_umma_workspace_bytes(int64_t B, int T, int num_layers) { return carve(B, T, num_layers).total + 256; }

// Runs every layer; fills hfin [B, 2H] with the top layer's final states.  Weights in the layout of nerrf_lstm_forward.
int lstm_layers_umma(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int num_layers, const float* const* Wih_t,
                     const float* const* Whh_t, const float* const* bias, float* hfin, void* workspace, size_t workspace_bytes,
                     cudaStream_t st) {
    const int groups = groups_for_device();
    NERRF_REQUIRE(groups >= 2, "tensor-core LSTM needs at least 16 SMs");
    NERRF_REQUIRE(D_in <= 64, "tensor-core LSTM: D_in <= 64 (got %d)", D_in);
    const Ws w = carve(B, T, num_layers);
    NERRF_REQUIRE(workspace_bytes >= w.total, "lstm workspace too small for the tensor-core path");
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    const int64_t n_bt = (B + NSEQ - 1) / NSEQ, Bp = n_bt * NSEQ;
    const int64_t n_tiles = (int64_t)T * n_bt;
    float* gxa = (float*)(ws + w.gxa); float* gxb = (float*)(ws + w.gxb);
    unsigned char* img0 = (unsigned char*)(ws + w.img0);
    unsigned char* img[2] = {(unsigned char*)(ws + w.img_a), (unsigned char*)(ws + w.img_b)};
    float* wih = (float*)(ws + w.wih); float* whh = (float*)(ws + w.whh); float* bp = (float*)(ws + w.bias);
    unsigned* counter = (unsigned*)(ws + w.counter);
    const int blk = sm_count() * 4;
    const int ctas_per_combo = sm_count() / 16 > 0 ? sm_count() / 16 : 1;
    lstm_image_kernel<<<blk, 256, 0, st>>>(seq, D_in, B, T, n_bt, img0);
    int rc = set_max_dynamic_smem((const void*)lstm_rec_kernel, REC_SMEM);
    if (rc) return rc;
    for (int l = 0; l < num_layers; ++l) {
        // ---- input projection: one launch per K range, 16 (direction, slice) combos each
        const unsigned char* in_img = l == 0 ? img0 : img[(l - 1) & 1];
        for (int d = 0; d < 2; ++d) pack_bias_kernel<<<(SLICES * UM + 255) / 256, 256, 0, st>>>(bias[2 * l + d], bp + (size_t)d * SLICES * UM);
        const int ranges = l == 0 ? 1 : 2;
        for (int kr = 0; kr < ranges; ++kr) {
            const int Kdst = l == 0 ? 64 : LH;
            for (int d = 0; d < 2; ++d) {
                if (l == 0) pack_slices_kernel<<<blk, 256, 0, st>>>(Wih_t[2 * l + d], 0, D_in, 64, wih + (size_t)d * SLICES * Kdst * UM);
                else pack_slices_kernel<<<blk, 256, 0, st>>>(Wih_t[2 * l + d], kr * LH, LH, LH, wih + (size_t)d * SLICES * Kdst * UM);
            }
            ProjArgs a{};
            a.img = in_img;
            a.tile_stride = l == 0 ? (size_t)NS * NSEQ * 128 : (size_t)2 * TILE_BYTES_H;
            a.k_off = l == 0 ? 0 : (size_t)kr * TILE_BYTES_H;
            a.wih = wih; a.bias = kr == 0 ? bp : nullptr; a.gx = kr == 0 ? gxa : gxb;
            a.n_tiles = n_tiles; a.rows_total = (int64_t)T * Bp; a.ctas_per_combo = ctas_per_combo;
            rc = l == 0 ? launch_proj<1>(a, st) : launch_proj<KB_H>(a, st);
            if (rc) return rc;
        }
        for (int d = 0; d < 2; ++d)
            pack_slices_kernel<<<blk, 256, 0, st>>>(Whh_t[2 * l + d], 0, LH, LH, whh + (size_t)d * SLICES * LH * UM);
        // ---- recurrence
        NERRF_CHECK_CUDA(cudaMemsetAsync(counter, 0, 1024, st));
        RecArgs r{};
        r.gx_a = gxa; r.gx_b = l == 0 ? nullptr : gxb; r.whh = whh; r.len = len;
        r.out_img = img[l & 1]; r.hfin = hfin; r.counter = counter;
        r.B = B; r.Bp = Bp; r.n_bt = n_bt; r.T = T; r.groups = groups;
        void* args[] = {&r};
        NERRF_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)lstm_rec_kernel, dim3(groups * SLICES), dim3(REC_THREADS), args,
                                                     REC_SMEM, st));
    }
    return launch_status("lstm_rec_kernel");
}

}  // namespace nerrf
