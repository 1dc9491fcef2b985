// GraphSAGE-T edge head BACKWARD (training the attack / normal edge classifier).  fp32, deterministic (no atomics: every
// reduction has a fixed order, and the row chunking of the weight gradient depends on n_nodes only).
//
//   forward   proj[v]  = (h_v . We[0:H, 0], h_v . We[0:H, 1], h_v . We[H:2H, 0], h_v . We[H:2H, 1])
//             logit[e] = proj[src_e][0:2] + proj[dst_e][2:4] + be            (edges in CSR-by-destination order)
//   backward  g_src[v] = sum_{e: src(e)=v} dL[e]      (gather over the transposed graph: t_eid = CSR position of an out-edge)
//             g_dst[v] = sum_{e: dst(e)=v} dL[e]      (the contiguous CSR row v)
//             dh[v]    = g_src[v] We[0:H]^T + g_dst[v] We[H:2H]^T
//             dWe      = [h^T g_src ; h^T g_dst],   dbe = sum_v g_dst[v]
//
// Kernels:
//   sage_edge_bwd_g_kernel   one warp per node: both row sums (each lane walks edges lane, lane+32, ... into four
//                            interleaved accumulators, combined (a0+a1)+(a2+a3), then a butterfly warp sum), g[v] -> the
//                            workspace, and the node's dh row from the butterfly result (every lane holds g)
//   sage_edge_bwd_dw_kernel  one CTA per row chunk: warp w takes rows w, w+8, ...; lane owns k = 4 lane .. +3 (16 sums);
//                            the eight warps are combined in warp order into a partial [2H*2 + 2] slab
//   sage_edge_bwd_reduce_kernel  partials -> dWe / dbe, chunk order fixed
#include "common.cuh"

namespace nerrf {
namespace {

constexpr int EH = 128;                   // hidden width
constexpr int EW_SLAB = 2 * EH * 2 + 4;   // partial slab: dWe [2H][2] then dbe [2] (padded to 16 bytes)
constexpr int EW_MAX_CHUNKS = 1024;

template <typename RP, typename TP>
__global__ void __launch_bounds__(256) sage_edge_bwd_g_kernel(const float* __restrict__ dL, const RP* __restrict__ rowptr,
                                                              const TP* __restrict__ t_rowptr, const TP* __restrict__ t_eid,
                                                              const float* __restrict__ We, float4* __restrict__ g,
                                                              float* __restrict__ dh, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    const float2* d2 = reinterpret_cast<const float2*>(dL);
    float2 a[4];
    // g_dst: the row's own edges, contiguous
    {
        const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
#pragma unroll
        for (int u = 0; u < 4; ++u) a[u] = make_float2(0.f, 0.f);
        int64_t e = e0 + lane;
        for (; e + 96 < e1; e += 128) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float2 v = __ldg(d2 + e + 32 * u);
                a[u].x += v.x; a[u].y += v.y;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (e + 32 * u < e1) {
                const float2 v = __ldg(d2 + e + 32 * u);
                a[u].x += v.x; a[u].y += v.y;
            }
        }
    }
    float gd0 = warp_sum((a[0].x + a[1].x) + (a[2].x + a[3].x));
    float gd1 = warp_sum((a[0].y + a[1].y) + (a[2].y + a[3].y));
    // g_src: the out-edges, gathered through t_eid
    {
        const int64_t j0 = (int64_t)t_rowptr[row], j1 = (int64_t)t_rowptr[row + 1];
#pragma unroll
        for (int u = 0; u < 4; ++u) a[u] = make_float2(0.f, 0.f);
        int64_t j = j0 + lane;
        for (; j + 96 < j1; j += 128) {
            int64_t id[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) id[u] = (int64_t)__ldg(t_eid + j + 32 * u);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float2 v = __ldg(d2 + id[u]);
                a[u].x += v.x; a[u].y += v.y;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (j + 32 * u < j1) {
                const float2 v = __ldg(d2 + (int64_t)__ldg(t_eid + j + 32 * u));
                a[u].x += v.x; a[u].y += v.y;
            }
        }
    }
    const float gs0 = warp_sum((a[0].x + a[1].x) + (a[2].x + a[3].x));
    const float gs1 = warp_sum((a[0].y + a[1].y) + (a[2].y + a[3].y));
    if (g && lane == 0) g[row] = make_float4(gs0, gs1, gd0, gd1);
    if (dh) {
        // lane owns k = 4 lane .. +3: We[k][0..1] (source half) and We[H + k][0..1] (destination half)
        const float4 s0 = ldg4(We + 8 * lane), s1 = ldg4(We + 8 * lane + 4);
        const float4 t0 = ldg4(We + 2 * EH + 8 * lane), t1 = ldg4(We + 2 * EH + 8 * lane + 4);
        const float ws[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        const float wd[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
        float o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            o[q] = fmaf(gd1, wd[2 * q + 1], fmaf(gd0, wd[2 * q], fmaf(gs1, ws[2 * q + 1], gs0 * ws[2 * q])));
        *reinterpret_cast<float4*>(dh + row * EH + 4 * lane) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// part[chunk] = [ sum_r h[r, k] g_src[r, c]  (k < H) ; sum_r h[r, k] g_dst[r, c] ; sum_r g_dst[r, c] ] over the chunk's rows
__global__ void __launch_bounds__(256) sage_edge_bwd_dw_kernel(const float* __restrict__ h, const float4* __restrict__ g,
                                                               float* __restrict__ part, int64_t n, int64_t rows_per_chunk) {
    __shared__ __align__(16) float red[8][EW_SLAB];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r_begin = (int64_t)blockIdx.x * rows_per_chunk;
    int64_t r_end = r_begin + rows_per_chunk;
    if (r_end > n) r_end = n;
    float acc[4][4];                       // [k q][ gs0, gs1, gd0, gd1 ]
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[q][c] = 0.f;
    float db0 = 0.f, db1 = 0.f;
    for (int64_t r = r_begin + warp; r < r_end; r += 8) {
        const float4 gv = __ldg(g + r);
        const float4 hv = ldg4(h + r * EH + 4 * lane);
        const float hh[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            acc[q][0] = fmaf(hh[q], gv.x, acc[q][0]); acc[q][1] = fmaf(hh[q], gv.y, acc[q][1]);
            acc[q][2] = fmaf(hh[q], gv.z, acc[q][2]); acc[q][3] = fmaf(hh[q], gv.w, acc[q][3]);
        }
        db0 += gv.z; db1 += gv.w;
    }
    // slab layout = dWe row-major [2H][2]: source half rows k, destination half rows H + k
    float* mine = red[warp];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int k = 4 * lane + q;
        mine[2 * k] = acc[q][0]; mine[2 * k + 1] = acc[q][1];
        mine[2 * (EH + k)] = acc[q][2]; mine[2 * (EH + k) + 1] = acc[q][3];
    }
    if (lane == 0) { mine[4 * EH] = db0; mine[4 * EH + 1] = db1; mine[4 * EH + 2] = 0.f; mine[4 * EH + 3] = 0.f; }
    __syncthreads();
    float* out = part + (size_t)blockIdx.x * EW_SLAB;
    for (int i = threadIdx.x; i < EW_SLAB; i += 256) {
        float s = red[0][i];
#pragma unroll
        for (int w = 1; w < 8; ++w) s += red[w][i];
        out[i] = s;
    }
}

__global__ void __launch_bounds__(256) sage_edge_bwd_reduce_kernel(const float* __restrict__ part, float* __restrict__ dW,
                                                                   float* __restrict__ db, int chunks) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= 4 * EH + 2) return;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[(size_t)c * EW_SLAB + i];
    if (i < 4 * EH) dW[i] = s;
    else db[i - 4 * EH] = s;
}

struct EdgeBwdPlan {
    int chunks;
    int64_t rows_per_chunk;
    size_t g_bytes, part_bytes;
};
EdgeBwdPlan edge_bwd_plan(int64_t n) {
    EdgeBwdPlan p;
    int64_t rpc = (n + EW_MAX_CHUNKS - 1) / EW_MAX_CHUNKS;
    if (rpc < 64) rpc = 64;
    p.rows_per_chunk = (rpc + 7) & ~(int64_t)7;
    p.chunks = (int)((n + p.rows_per_chunk - 1) / p.rows_per_chunk);
    if (p.chunks < 1) p.chunks = 1;
    p.g_bytes = (((size_t)n * 16) + 255) & ~(size_t)255;
    p.part_bytes = (size_t)p.chunks * EW_SLAB * 4;
    return p;
}

template <typename RP, typename TP>
void launch_g(const float* dL, const void* rowptr, const void* t_rowptr, const void* t_eid, const float* We, float4* g,
              float* dh, int64_t n, cudaStream_t st) {
    sage_edge_bwd_g_kernel<RP, TP><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(dL, (const RP*)rowptr, (const TP*)t_rowptr,
                                                                            (const TP*)t_eid, We, g, dh, n);
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_sage_edge_head_bwd_workspace_bytes(int64_t n_nodes, int H, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_nodes >= 0, "bad argument");
    NERRF_REQUIRE(H == EH, "hidden width must be 128 (got %d)", H);
    const EdgeBwdPlan p = edge_bwd_plan(n_nodes);
    *bytes = p.g_bytes + p.part_bytes + 256;
    return NERRF_OK;
}

extern "C" int nerrf_sage_edge_head_bwd(const float* h, const float* edge_W, const float* d_logit, const void* rowptr,
                                        int rowptr_is64, const void* t_rowptr, const void* t_eid, int t_is64, float* dh,
                                        float* d_edge_W, float* d_edge_b, void* workspace, size_t workspace_bytes,
                                        int64_t n_nodes, int H, nerrf_stream_t stream) {
    NERRF_REQUIRE(H == EH, "hidden width must be 128 (got %d)", H);
    NERRF_REQUIRE(n_nodes >= 0, "negative node count");
    NERRF_REQUIRE(rowptr && t_rowptr, "null graph pointer");     // d_logit / t_eid may be null when the graph has no edges
    NERRF_REQUIRE(!dh || edge_W, "dh needs edge_W");
    NERRF_REQUIRE(!d_edge_W || (h && d_edge_b && workspace), "d_edge_W needs h, d_edge_b and the workspace");
    size_t need = 0;
    nerrf_sage_edge_head_bwd_workspace_bytes(n_nodes, H, &need);
    if (d_edge_W && workspace_bytes < need) {
        set_error("edge head backward workspace too small: need %zu bytes", need);
        return NERRF_ERR_WORKSPACE;
    }
    for (const void* p : {(const void*)h, (const void*)edge_W, (const void*)d_logit, (const void*)dh, (const void*)d_edge_W,
                          (const void*)workspace})
        NERRF_REQUIRE(((uintptr_t)p & 15) == 0, "edge head backward buffers must be 16-byte aligned");
    NERRF_REQUIRE(((uintptr_t)d_edge_b & 3) == 0, "d_edge_b must be 4-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_nodes == 0) {
        if (d_edge_W) {
            NERRF_CHECK_CUDA(cudaMemsetAsync(d_edge_W, 0, (size_t)2 * EH * 2 * 4, st));
            NERRF_CHECK_CUDA(cudaMemsetAsync(d_edge_b, 0, 2 * 4, st));
        }
        return NERRF_OK;
    }
    if (!dh && !d_edge_W) return NERRF_OK;
    NERRF_REQUIRE(n_nodes / 8 < (1ll << 31), "too many nodes");
    const EdgeBwdPlan p = edge_bwd_plan(n_nodes);
    float4* g = d_edge_W ? reinterpret_cast<float4*>(workspace) : nullptr;
    float* part = d_edge_W ? reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + p.g_bytes) : nullptr;
    if (rowptr_is64) {
        if (t_is64) launch_g<int64_t, int64_t>(d_logit, rowptr, t_rowptr, t_eid, edge_W, g, dh, n_nodes, st);
        else launch_g<int64_t, int32_t>(d_logit, rowptr, t_rowptr, t_eid, edge_W, g, dh, n_nodes, st);
    } else {
        if (t_is64) launch_g<int32_t, int64_t>(d_logit, rowptr, t_rowptr, t_eid, edge_W, g, dh, n_nodes, st);
        else launch_g<int32_t, int32_t>(d_logit, rowptr, t_rowptr, t_eid, edge_W, g, dh, n_nodes, st);
    }
    if (d_edge_W) {
        sage_edge_bwd_dw_kernel<<<(unsigned)p.chunks, 256, 0, st>>>(h, g, part, n_nodes, p.rows_per_chunk);
        sage_edge_bwd_reduce_kernel<<<(4 * EH + 2 + 255) / 256, 256, 0, st>>>(part, d_edge_W, d_edge_b, p.chunks);
    }
    return launch_status("sage edge head backward");
}
