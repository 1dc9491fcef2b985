// GraphSAGE-T layer BACKWARD (SURVEY.md 8f rank 3: "backward for K1/K2"; reference surface: ai/train.py, README.md:75,
// ROADMAP.md:62-69 -- named, never written).  fp32, deterministic (no atomics: every reduction has a fixed order, and the
// row chunking of the weight gradient depends on n only, so every card gives the same bits).
//
//   forward   Z = [h || m],  m = A h (A = row-normalised weighted adjacency, CSR by destination),  Y = act(Z W + b)
//   backward  dP = dY * [Y > 0]                      (ReLU mask from the saved output)
//             db = sum_v dP[v, :]                    dW = Z^T dP                        (K2 backward, weight side)
//             dZ = dP W^T                                                                (K2 backward, input side)
//             dh = dZ[:, :F] + A^T dZ[:, F:]                                             (K1 backward)
//
// A^T is applied as a GATHER over the transposed graph (CSR by SOURCE, edge weights pre-normalised by the destination's
// weight sum), which the caller builds once per graph: the same warp-per-row gather loop as the forward K1
// (sage_gather.cuh), so the backward of the aggregate costs what the forward aggregate costs and is bit-reproducible.
//
// Kernels (CUDA cores; training is not the north-star hot path -- DESIGN.md 2.7 -- but it no longer leaves the GPU):
//   sage_bwd_dz_kernel   64-row tiles: dP tile in shared memory, W^T streamed in 64-column chunks, 4x4 register blocks
//   sage_bwd_dw_kernel   grid (row chunks, 2F/64): each CTA accumulates a [64 x 128] slab of dW over its rows in registers
//                        (4 x 8 per thread) and writes a partial; slab 0 also accumulates db
//   sage_bwd_reduce_kernel  partials -> dW / db, chunk order fixed
//   sage_bwd_dh_kernel   one warp per source row: dZ[u, :F] + gather of dZ[dst, F:] over the transposed row
//   sage_bwd_dew_kernel  one warp per destination row: the edge-weight gradient d_ew (nerrf_sage_layer_bwd_ex; node
//                        explanations, nerrf_b200.explain)
//   sage_norm_weights_kernel  one warp per destination row: a_e = w_e / max(row weight sum, 1e-12), the weight sum taken in
//                        gather_row's lane order and warp_sum, so A^T holds the forward aggregate's A entries to the bit
#include "common.cuh"
#include "sage_gather.cuh"

namespace nerrf {
namespace {

constexpr int HB = 128;              // hidden width (layer output)
constexpr int DZ_BM = 64;            // rows per dZ tile
constexpr int DZ_LDP = HB + 4;       // padded dP row (floats)
constexpr int DZ_KC = 64;            // dZ columns per W^T chunk
constexpr int DZ_LDW = DZ_KC + 4;
constexpr size_t DZ_SMEM = (size_t)(DZ_BM * DZ_LDP + HB * DZ_LDW) * sizeof(float);

constexpr int DW_BR = 32;            // rows per dW tile
constexpr int DW_KS = 64;            // k rows of dW per CTA slab
constexpr int DW_LDZ = DW_KS + 4;
constexpr int DW_LDP = HB + 4;
constexpr int MAX_CHUNKS = 264;      // dW row chunks at most (2 per SM of a 132-SM H100, fixed so the bits do not depend on the card)

// dZ[r, k] = sum_j dP[r, j] W[k, j],  dP = dY * [Y > 0] (relu) or dY
template <int F>
__global__ void __launch_bounds__(256) sage_bwd_dz_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                                          const float* __restrict__ W, float* __restrict__ dz, int64_t n,
                                                          int relu) {
    constexpr int K2 = 2 * F;
    extern __shared__ __align__(16) float smem[];
    float* Ps = smem;                         // [DZ_BM][DZ_LDP]
    float* Wt = smem + DZ_BM * DZ_LDP;        // [HB][DZ_LDW]:  Wt[j][kk] = W[k0 + kk][j]
    const int tid = threadIdx.x;
    const int64_t row0 = (int64_t)blockIdx.x * DZ_BM;
    for (int i = tid; i < DZ_BM * (HB / 4); i += 256) {
        const int r = i / (HB / 4), c4 = i % (HB / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row0 + r < n) {
            v = ldg4(dy + (row0 + r) * HB + 4 * c4);
            if (relu) {
                const float4 o = ldg4(y + (row0 + r) * HB + 4 * c4);
                v.x = o.x > 0.f ? v.x : 0.f; v.y = o.y > 0.f ? v.y : 0.f; v.z = o.z > 0.f ? v.z : 0.f; v.w = o.w > 0.f ? v.w : 0.f;
            }
        }
        *reinterpret_cast<float4*>(Ps + r * DZ_LDP + 4 * c4) = v;
    }
    const int tx = tid & 15, ty = tid >> 4;       // thread = rows 4 ty .. +3, chunk columns 4 tx .. +3
    for (int k0 = 0; k0 < K2; k0 += DZ_KC) {
        __syncthreads();                          // Ps complete (first pass) / previous chunk consumed
        for (int i = tid; i < DZ_KC * HB; i += 256) {
            const int kk = i / HB, j = i % HB;    // coalesced along j
            Wt[j * DZ_LDW + kk] = __ldg(W + (size_t)(k0 + kk) * HB + j);
        }
        __syncthreads();
        float acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
#pragma unroll 4
        for (int j = 0; j < HB; j += 4) {
            float4 p[4], w[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) p[a] = *reinterpret_cast<const float4*>(Ps + (ty * 4 + a) * DZ_LDP + j);
#pragma unroll
            for (int q = 0; q < 4; ++q) w[q] = *reinterpret_cast<const float4*>(Wt + (j + q) * DZ_LDW + 4 * tx);
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                acc[a][0] = fmaf(p[a].x, w[0].x, acc[a][0]); acc[a][1] = fmaf(p[a].x, w[0].y, acc[a][1]);
                acc[a][2] = fmaf(p[a].x, w[0].z, acc[a][2]); acc[a][3] = fmaf(p[a].x, w[0].w, acc[a][3]);
                acc[a][0] = fmaf(p[a].y, w[1].x, acc[a][0]); acc[a][1] = fmaf(p[a].y, w[1].y, acc[a][1]);
                acc[a][2] = fmaf(p[a].y, w[1].z, acc[a][2]); acc[a][3] = fmaf(p[a].y, w[1].w, acc[a][3]);
                acc[a][0] = fmaf(p[a].z, w[2].x, acc[a][0]); acc[a][1] = fmaf(p[a].z, w[2].y, acc[a][1]);
                acc[a][2] = fmaf(p[a].z, w[2].z, acc[a][2]); acc[a][3] = fmaf(p[a].z, w[2].w, acc[a][3]);
                acc[a][0] = fmaf(p[a].w, w[3].x, acc[a][0]); acc[a][1] = fmaf(p[a].w, w[3].y, acc[a][1]);
                acc[a][2] = fmaf(p[a].w, w[3].z, acc[a][2]); acc[a][3] = fmaf(p[a].w, w[3].w, acc[a][3]);
            }
        }
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int64_t r = row0 + ty * 4 + a;
            if (r < n) *reinterpret_cast<float4*>(dz + r * K2 + k0 + 4 * tx) = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
        }
    }
}

// partial dW slab: part[chunk][k][j] = sum over the chunk's rows of Z[r, k] dP[r, j]; slab 0 also dbpart[chunk][j]
template <int F>
__global__ void __launch_bounds__(256) sage_bwd_dw_kernel(const float* __restrict__ h, const float* __restrict__ m,
                                                          const float* __restrict__ dy, const float* __restrict__ y,
                                                          float* __restrict__ part, float* __restrict__ dbpart, int64_t n,
                                                          int64_t rows_per_chunk, int relu) {
    constexpr int K2 = 2 * F;
    __shared__ __align__(16) float Zs[DW_BR * DW_LDZ];
    __shared__ __align__(16) float Ps[DW_BR * DW_LDP];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;   // thread = k rows 4 ty .. +3 of the slab, j columns 8 tx .. +7
    const int chunk = blockIdx.x, k0 = blockIdx.y * DW_KS;
    const int64_t r_begin = (int64_t)chunk * rows_per_chunk;
    int64_t r_end = r_begin + rows_per_chunk;
    if (r_end > n) r_end = n;
    float acc[4][8], dbacc[8];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
#pragma unroll
    for (int b = 0; b < 8; ++b) dbacc[b] = 0.f;
    for (int64_t t0 = r_begin; t0 < r_end; t0 += DW_BR) {
        __syncthreads();
        for (int i = tid; i < DW_BR * (DW_KS / 4); i += 256) {
            const int r = i / (DW_KS / 4), c4 = i % (DW_KS / 4);
            const int k = k0 + 4 * c4;                                  // F is a multiple of 4: a float4 never straddles h | m
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t0 + r < r_end) v = (k < F) ? ldg4(h + (t0 + r) * F + k) : ldg4(m + (t0 + r) * F + (k - F));
            *reinterpret_cast<float4*>(Zs + r * DW_LDZ + 4 * c4) = v;
        }
        for (int i = tid; i < DW_BR * (HB / 4); i += 256) {
            const int r = i / (HB / 4), c4 = i % (HB / 4);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t0 + r < r_end) {
                v = ldg4(dy + (t0 + r) * HB + 4 * c4);
                if (relu) {
                    const float4 o = ldg4(y + (t0 + r) * HB + 4 * c4);
                    v.x = o.x > 0.f ? v.x : 0.f; v.y = o.y > 0.f ? v.y : 0.f; v.z = o.z > 0.f ? v.z : 0.f; v.w = o.w > 0.f ? v.w : 0.f;
                }
            }
            *reinterpret_cast<float4*>(Ps + r * DW_LDP + 4 * c4) = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int r = 0; r < DW_BR; ++r) {
            const float4 z = *reinterpret_cast<const float4*>(Zs + r * DW_LDZ + 4 * ty);
            const float4 p0 = *reinterpret_cast<const float4*>(Ps + r * DW_LDP + 8 * tx);
            const float4 p1 = *reinterpret_cast<const float4*>(Ps + r * DW_LDP + 8 * tx + 4);
            const float zz[4] = {z.x, z.y, z.z, z.w};
            const float pp[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(zz[a], pp[b], acc[a][b]);
            if (ty == 0) {
#pragma unroll
                for (int b = 0; b < 8; ++b) dbacc[b] += pp[b];
            }
        }
    }
    float* out = part + ((size_t)chunk * K2 + k0) * HB;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        *reinterpret_cast<float4*>(out + (size_t)(4 * ty + a) * HB + 8 * tx) = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
        *reinterpret_cast<float4*>(out + (size_t)(4 * ty + a) * HB + 8 * tx + 4) = make_float4(acc[a][4], acc[a][5], acc[a][6], acc[a][7]);
    }
    if (blockIdx.y == 0 && ty == 0) {
#pragma unroll
        for (int b = 0; b < 8; ++b) dbpart[(size_t)chunk * HB + 8 * tx + b] = dbacc[b];
    }
}

// out[i] = sum_c part[c][i], c ascending (deterministic)
__global__ void __launch_bounds__(256) sage_bwd_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int elems,
                                                              int chunks) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= elems) return;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[(size_t)c * elems + i];
    out[i] = s;
}

// dh[u, :] = dZ[u, :F] + sum_{e in t_row(u)} t_w[e] dZ[t_col[e], F:]
template <int F, typename RP>
__global__ void __launch_bounds__(256) sage_bwd_dh_kernel(const float* __restrict__ dz, const RP* __restrict__ t_rowptr,
                                                          const int32_t* __restrict__ t_col, const float* __restrict__ t_w,
                                                          float* __restrict__ dh, int64_t n) {
    constexpr int LPR = F / 4;
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    const int64_t e0 = t_rowptr[row], e1 = t_rowptr[row + 1];
    float wsum;
    float4 acc = gather_row<F, 0, 2 * F>(dz + F, t_col, t_w, e0, e1, lane, &wsum);      // unnormalised weighted sum
    if (lane < LPR) {
        const float4 s = ldg4(dz + row * (2 * F) + 4 * lane);
        *reinterpret_cast<float4*>(dh + row * F + 4 * lane) = make_float4(s.x + acc.x, s.y + acc.y, s.z + acc.z, s.w + acc.w);
    }
}

// d_ew[e] += dZ[u, F:] . (h[src(e)] - [S_u >= 1e-12] m_u) / max(S_u, 1e-12) for every edge e of destination row u: the
// derivative of this layer's output w.r.t. the edge weight (the derivative of m_u = sum_e w_e h_src / max(S_u, 1e-12)).
// One warp per row, no atomics (each edge belongs to one row).  S_u is summed in gather_row's lane order and warp_sum, so
// it is the forward's S_u to the bit.  The differences are taken against r = h[src(first edge)]:
//     h_src - m = (h_src - r) - (m - r),   m - r = sum_e w_e (h_src(e) - r) / max(S, 1e-12)
// so a row whose sources are one node (a file written by one process, event after event) gets exactly 0 instead of the
// fp32 rounding of h - m / S amplified by 1 / S.  dZ[u, F:] is read once; G = 32 / LPR edges per step get one LPR-lane
// dot product each.
template <int F, typename RP>
__global__ void __launch_bounds__(256) sage_bwd_dew_kernel(const float* __restrict__ dz, const float* __restrict__ h,
                                                           const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                           const float* __restrict__ ew, float* __restrict__ d_ew, int64_t n) {
    constexpr int LPR = F / 4;
    constexpr int G = 32 / LPR;
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
    if (e1 <= e0) return;
    float wpart = 0.f;
    for (int64_t e = e0 + lane; e < e1; e += 32) wpart += __ldg(ew + e);
    const float wsum = warp_sum(wpart);
    const float inv = 1.0f / fmaxf(wsum, 1e-12f);
    const int g = lane / LPR, sub = lane % LPR;
    const float4 r = ldg4(h + (int64_t)__ldg(col + e0) * F + 4 * sub);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);                       // sum_e w_e (h_src(e) - r), this lane's group's edges
    for (int64_t e = e0 + g; e < e1; e += G) {
        const float w = __ldg(ew + e);
        const float4 v = ldg4(h + (int64_t)__ldg(col + e) * F + 4 * sub);
        acc.x = fmaf(w, v.x - r.x, acc.x); acc.y = fmaf(w, v.y - r.y, acc.y);
        acc.z = fmaf(w, v.z - r.z, acc.z); acc.w = fmaf(w, v.w - r.w, acc.w);
    }
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    const float4 d = ldg4(dz + row * (2 * F) + F + 4 * sub);
    // c = dZ . (m - r) when the gradient of max(S, 1e-12) passes ([S >= 1e-12], torch clamp_min); else -dZ . r, so that
    // p - c below is dZ . h_src either way
    float c = (wsum >= 1e-12f) ? (d.x * (acc.x * inv) + d.y * (acc.y * inv) + d.z * (acc.z * inv) + d.w * (acc.w * inv))
                               : -(d.x * r.x + d.y * r.y + d.z * r.z + d.w * r.w);
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    for (int64_t base = e0; base < e1; base += G) {
        const int64_t e = base + g;
        float p = 0.f;
        if (e < e1) {
            const float4 v = ldg4(h + (int64_t)__ldg(col + e) * F + 4 * sub);
            p = d.x * (v.x - r.x) + d.y * (v.y - r.y) + d.z * (v.z - r.z) + d.w * (v.w - r.w);
        }
#pragma unroll
        for (int o = 1; o < LPR; o <<= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        if (sub == 0 && e < e1) d_ew[e] += (p - c) * inv;
    }
}

// a[e] = ew[e] * (1 / max(sum of the row's weights, 1e-12)) over the CSR-by-destination rows: lane l sums edges e0 + l,
// e0 + l + 32, ... then warp_sum, exactly as gather_row sums the weights it normalises by
template <typename RP>
__global__ void __launch_bounds__(256) sage_norm_weights_kernel(const RP* __restrict__ rowptr, const float* __restrict__ ew,
                                                                float* __restrict__ a, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
    float wpart = 0.f;
    for (int64_t e = e0 + lane; e < e1; e += 32) wpart += __ldg(ew + e);
    const float inv = 1.0f / fmaxf(warp_sum(wpart), 1e-12f);
    for (int64_t e = e0 + lane; e < e1; e += 32) a[e] = __ldg(ew + e) * inv;
}

struct BwdPlan {
    int chunks;
    int64_t rows_per_chunk;
    size_t dz_bytes, part_bytes, dbpart_bytes;
};
BwdPlan bwd_plan(int64_t n, int F) {
    BwdPlan p;
    int64_t tiles = (n + DW_BR - 1) / DW_BR;
    if (tiles < 1) tiles = 1;                               // n = 0: one empty chunk
    const int64_t c = tiles < MAX_CHUNKS ? tiles : MAX_CHUNKS;
    p.rows_per_chunk = ((tiles + c - 1) / c) * DW_BR;
    p.chunks = (int)((n + p.rows_per_chunk - 1) / p.rows_per_chunk);
    if (p.chunks < 1) p.chunks = 1;
    p.dz_bytes = (((size_t)n * 2 * F * 4) + 255) & ~(size_t)255;
    p.part_bytes = (size_t)p.chunks * 2 * F * HB * 4;
    p.dbpart_bytes = (size_t)p.chunks * HB * 4;
    return p;
}

template <int F>
int launch_bwd(const float* h, const float* m, const float* y, const float* dy, const float* W, const void* t_rowptr, int is64,
               const int32_t* t_col, const float* t_w, float* dh, float* dW, float* db, float* ws, int64_t n, int relu,
               const void* rowptr, int rp64, const int32_t* col, const float* ew, float* d_ew, cudaStream_t st) {
    const BwdPlan p = bwd_plan(n, F);
    float* dz = ws;
    float* part = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(ws) + p.dz_bytes);
    float* dbpart = part + (size_t)p.chunks * 2 * F * HB;
    const int rc = set_max_dynamic_smem((const void*)sage_bwd_dz_kernel<F>, DZ_SMEM);
    if (rc) return rc;
    if (dW) {
        sage_bwd_dw_kernel<F><<<dim3((unsigned)p.chunks, 2 * F / DW_KS), 256, 0, st>>>(h, m, dy, y, part, dbpart, n, p.rows_per_chunk, relu);
        sage_bwd_reduce_kernel<<<(2 * F * HB + 255) / 256, 256, 0, st>>>(part, dW, 2 * F * HB, p.chunks);
        sage_bwd_reduce_kernel<<<1, 256, 0, st>>>(dbpart, db, HB, p.chunks);
    }
    if (dh || d_ew) sage_bwd_dz_kernel<F><<<(unsigned)((n + DZ_BM - 1) / DZ_BM), 256, DZ_SMEM, st>>>(dy, y, W, dz, n, relu);
    if (dh) {
        if (is64)
            sage_bwd_dh_kernel<F, int64_t><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(dz, (const int64_t*)t_rowptr, t_col, t_w, dh, n);
        else
            sage_bwd_dh_kernel<F, int32_t><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(dz, (const int32_t*)t_rowptr, t_col, t_w, dh, n);
    }
    if (d_ew) {
        if (rp64)
            sage_bwd_dew_kernel<F, int64_t><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(dz, h, (const int64_t*)rowptr, col, ew, d_ew, n);
        else
            sage_bwd_dew_kernel<F, int32_t><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(dz, h, (const int32_t*)rowptr, col, ew, d_ew, n);
    }
    return launch_status("sage layer backward");
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_sage_layer_bwd_workspace_bytes(int64_t n_nodes, int F, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_nodes >= 0, "bad argument");
    NERRF_REQUIRE(F == 32 || F == 64 || F == 128, "F must be 32, 64 or 128 (got %d)", F);
    const BwdPlan p = bwd_plan(n_nodes, F);
    *bytes = p.dz_bytes + p.part_bytes + p.dbpart_bytes + 256;
    return NERRF_OK;
}

extern "C" int nerrf_sage_layer_bwd_ex(const float* h_in, const float* m, const float* y, const float* dy, const float* W,
                                       const void* t_rowptr, int t_rowptr_is64, const int32_t* t_col, const float* t_w,
                                       float* dh, float* dW, float* db, float* workspace, size_t workspace_bytes,
                                       int64_t n_nodes, int F, int H, int relu, const void* rowptr, int rowptr_is64,
                                       const int32_t* col, const float* ew, float* d_ew, nerrf_stream_t stream) {
    NERRF_REQUIRE(H == HB, "hidden width must be 128 (got %d)", H);
    NERRF_REQUIRE(F == 32 || F == 64 || F == 128, "F must be 32, 64 or 128 (got %d)", F);
    NERRF_REQUIRE(n_nodes >= 0, "negative node count");
    NERRF_REQUIRE(dy && W && workspace, "null pointer");
    NERRF_REQUIRE(!relu || y, "the ReLU mask needs the layer output y");
    NERRF_REQUIRE(!dW || (h_in && m && db), "dW needs h_in, m and db");
    NERRF_REQUIRE(!dh || t_rowptr, "dh needs the transposed graph");     // t_col / t_w may be null when the graph has no edges
    NERRF_REQUIRE(!d_ew || (h_in && rowptr), "d_ew needs h_in and the graph");   // col / ew / d_ew null: no edges
    NERRF_REQUIRE(n_nodes / 8 < (1ll << 31), "too many nodes");
    size_t need = 0;
    nerrf_sage_layer_bwd_workspace_bytes(n_nodes, F, &need);
    if (workspace_bytes < need) {
        set_error("backward workspace too small: need %zu bytes", need);
        return NERRF_ERR_WORKSPACE;
    }
    for (const void* p : {(const void*)h_in, (const void*)m, (const void*)y, (const void*)dy, (const void*)W, (const void*)dh,
                          (const void*)dW, (const void*)db, (const void*)workspace})
        NERRF_REQUIRE(((uintptr_t)p & 15) == 0, "backward buffers must be 16-byte aligned");
    if (n_nodes == 0) {
        if (dW) {
            NERRF_CHECK_CUDA(cudaMemsetAsync(dW, 0, (size_t)2 * F * HB * 4, (cudaStream_t)stream));
            NERRF_CHECK_CUDA(cudaMemsetAsync(db, 0, (size_t)HB * 4, (cudaStream_t)stream));
        }
        return NERRF_OK;
    }
    cudaStream_t st = (cudaStream_t)stream;
    switch (F) {
        case 32: return launch_bwd<32>(h_in, m, y, dy, W, t_rowptr, t_rowptr_is64, t_col, t_w, dh, dW, db, workspace, n_nodes, relu,
                                       rowptr, rowptr_is64, col, ew, d_ew, st);
        case 64: return launch_bwd<64>(h_in, m, y, dy, W, t_rowptr, t_rowptr_is64, t_col, t_w, dh, dW, db, workspace, n_nodes, relu,
                                       rowptr, rowptr_is64, col, ew, d_ew, st);
        default: return launch_bwd<128>(h_in, m, y, dy, W, t_rowptr, t_rowptr_is64, t_col, t_w, dh, dW, db, workspace, n_nodes, relu,
                                        rowptr, rowptr_is64, col, ew, d_ew, st);
    }
}

extern "C" int nerrf_sage_layer_bwd(const float* h_in, const float* m, const float* y, const float* dy, const float* W,
                                    const void* t_rowptr, int t_rowptr_is64, const int32_t* t_col, const float* t_w,
                                    float* dh, float* dW, float* db, float* workspace, size_t workspace_bytes,
                                    int64_t n_nodes, int F, int H, int relu, nerrf_stream_t stream) {
    return nerrf_sage_layer_bwd_ex(h_in, m, y, dy, W, t_rowptr, t_rowptr_is64, t_col, t_w, dh, dW, db, workspace, workspace_bytes,
                                   n_nodes, F, H, relu, nullptr, 0, nullptr, nullptr, nullptr, stream);
}

extern "C" int nerrf_sage_norm_weights(const void* rowptr, int rowptr_is64, const float* ew, float* a, int64_t n_nodes,
                                       nerrf_stream_t stream) {
    NERRF_REQUIRE(n_nodes >= 0, "negative node count");
    NERRF_REQUIRE(rowptr, "null rowptr");                     // ew / a may be null when the graph has no edges
    if (n_nodes == 0) return NERRF_OK;
    NERRF_REQUIRE(n_nodes / 8 < (1ll << 31), "too many nodes");
    const unsigned blocks = (unsigned)((n_nodes + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (rowptr_is64)
        sage_norm_weights_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)rowptr, ew, a, n_nodes);
    else
        sage_norm_weights_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)rowptr, ew, a, n_nodes);
    return launch_status("sage edge weight normalisation");
}
