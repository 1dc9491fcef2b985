// GraphSAGE-T forward kernels (SURVEY.md 8a rows a1-a3; DESIGN.md "GraphSAGE-T kernels").
//
//   K1  gather + weighted-mean aggregate over the CSR-by-destination temporal graph
//   K2  [x_v || m_v] @ W + b, ReLU            -- fused with K1: the aggregate tile is written
//       straight into the shared-memory A operand and never round-trips HBM.
// This file holds the fp32 CUDA-core (FFMA) fused kernel, the standalone K1, the heads, the
// whole-forward driver and the host-buffer session.  The tensor-core (wgmma) fused kernel is sage_umma.cu.
#include "common.cuh"
#include "ptx.cuh"
#include "sage_gather.cuh"

namespace nerrf {

int sage_layer_umma(const float* x, const void* rowptr, int is64, const int32_t* col, const float* ew,
                    const float* W, const float* b, float* out, int64_t n_nodes, int64_t row_begin,
                    int64_t row_end, int F, int relu, int nsplit, const float* node_w, float node_b, float* score,
                    void* long_ws, size_t long_ws_bytes, bool reuse_scan, float* const* peer_out, int n_peers,
                    const uint8_t* peer_need, int l2_policy, cudaStream_t st);   // sage_umma.cu (node_w != NULL: node head fused into the epilogue)

// `algo` of one layer call of a multi-layer driver: the caller's selector and L2 flag, REUSE_LONG_SCAN set by the driver
static int layer_algo(int algo, bool reuse_scan) {
    return (algo & ~NERRF_SAGE_FLAG_REUSE_LONG_SCAN) | (reuse_scan ? NERRF_SAGE_FLAG_REUSE_LONG_SCAN : 0);
}

// ------------------------------------------------------------------------------------------
// K1 standalone: one warp per destination row.
template <int F, typename RP>
__global__ void __launch_bounds__(256) sage_aggregate_kernel(const float* __restrict__ x, const RP* __restrict__ rowptr,
                                                             const int32_t* __restrict__ col, const float* __restrict__ ew,
                                                             float* __restrict__ m, int64_t row_begin, int64_t row_end) {
    constexpr int LPR = F / 4;
    const int lane = threadIdx.x & 31;
    const int64_t row = row_begin + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= row_end) return;
    const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
    float4 acc = gather_row<F>(x, col, ew, e0, e1, lane);
    if (lane < LPR) *reinterpret_cast<float4*>(m + (row - row_begin) * F + 4 * lane) = acc;
}

// ------------------------------------------------------------------------------------------
// Fused layer, fp32 CUDA cores.  CTA = 256 threads, tile = 64 destination rows x H=128.
//   phase 1: 8 warps gather/aggregate 64 rows -> smem A tile [64][2F] (self || mean)
//   phase 2: A[64 x 2F] @ W[2F x 128]; W streamed from L2 in 32-row chunks (cp.async, 2 stages)
//   thread (ty, tx) owns a 4 x 8 output block.
constexpr int BM = 64;
constexpr int KC = 32;
constexpr int HH = 128;

template <int F>
struct FfmaCfg {
    static constexpr int K = 2 * F;
    static constexpr int LDA = K + 4;                       // padded row stride (floats)
    static constexpr size_t smem = (size_t)(BM * LDA + 2 * KC * HH) * sizeof(float);
};

template <int F, typename RP>
__global__ void __launch_bounds__(256, 2)
sage_layer_ffma_kernel(const float* __restrict__ x, const RP* __restrict__ rowptr, const int32_t* __restrict__ col,
                       const float* __restrict__ ew, const float* __restrict__ W, const float* __restrict__ bias,
                       float* __restrict__ out, int64_t row_begin, int64_t row_end, int relu) {
    using C = FfmaCfg<F>;
    constexpr int K = C::K, LDA = C::LDA, LPR = F / 4;
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                      // [BM][LDA]
    float* Ws = smem + BM * LDA;           // [2][KC][HH]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tile_row0 = row_begin + (int64_t)blockIdx.x * BM;

    // prefetch W chunk 0 while gathering
    auto load_w_chunk = [&](int chunk, int stage) {
        const float* src = W + (size_t)chunk * KC * HH;
        float* dst = Ws + stage * KC * HH;
#pragma unroll
        for (int i = 0; i < (KC * HH / 4) / 256; ++i) {
            int idx = tid + i * 256;
            cp_async16(smem_u32(dst + idx * 4), src + idx * 4);
        }
        cp_async_commit();
    };
    load_w_chunk(0, 0);

    // ---- phase 1: gather + aggregate
    for (int r = warp; r < BM; r += 8) {
        const int64_t row = tile_row0 + r;
        float4 self = make_float4(0.f, 0.f, 0.f, 0.f), acc = self;
        if (row < row_end) {
            const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
            if (lane < LPR) self = ldg4(x + row * F + 4 * lane);
            acc = gather_row<F>(x, col, ew, e0, e1, lane);
        }
        if (lane < LPR) {
            *reinterpret_cast<float4*>(As + r * LDA + 4 * lane) = self;
            *reinterpret_cast<float4*>(As + r * LDA + F + 4 * lane) = acc;
        }
    }

    // ---- phase 2: GEMM
    const int tx = tid & 15, ty = tid >> 4;
    float c[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) c[i][j] = 0.f;

    constexpr int NCHUNK = K / KC;
    for (int ch = 0; ch < NCHUNK; ++ch) {
        if (ch + 1 < NCHUNK) {
            load_w_chunk(ch + 1, (ch + 1) & 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();   // W chunk ch landed for everyone (and, for ch==0, the A tile is complete)
        const float* Wc = Ws + (ch & 1) * KC * HH;
        const float* Ab = As + (ty * 4) * LDA + ch * KC;
#pragma unroll
        for (int kk = 0; kk < KC; kk += 4) {
            float4 a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(Ab + i * LDA + kk);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 w0 = *reinterpret_cast<const float4*>(Wc + (kk + q) * HH + tx * 8);
                const float4 w1 = *reinterpret_cast<const float4*>(Wc + (kk + q) * HH + tx * 8 + 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float av = q == 0 ? a[i].x : (q == 1 ? a[i].y : (q == 2 ? a[i].z : a[i].w));
                    c[i][0] = fmaf(av, w0.x, c[i][0]); c[i][1] = fmaf(av, w0.y, c[i][1]);
                    c[i][2] = fmaf(av, w0.z, c[i][2]); c[i][3] = fmaf(av, w0.w, c[i][3]);
                    c[i][4] = fmaf(av, w1.x, c[i][4]); c[i][5] = fmaf(av, w1.y, c[i][5]);
                    c[i][6] = fmaf(av, w1.z, c[i][6]); c[i][7] = fmaf(av, w1.w, c[i][7]);
                }
            }
        }
        __syncthreads();   // everyone done with stage (ch&1) before it is refilled at ch+2
    }

    // ---- epilogue: bias + ReLU, 2 x float4 per row
    const float4 b0 = ldg4(bias + tx * 8), b1 = ldg4(bias + tx * 8 + 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t row = tile_row0 + ty * 4 + i;
        if (row >= row_end) continue;
        float4 o0 = make_float4(c[i][0] + b0.x, c[i][1] + b0.y, c[i][2] + b0.z, c[i][3] + b0.w);
        float4 o1 = make_float4(c[i][4] + b1.x, c[i][5] + b1.y, c[i][6] + b1.z, c[i][7] + b1.w);
        if (relu) {
            o0.x = fmaxf(o0.x, 0.f); o0.y = fmaxf(o0.y, 0.f); o0.z = fmaxf(o0.z, 0.f); o0.w = fmaxf(o0.w, 0.f);
            o1.x = fmaxf(o1.x, 0.f); o1.y = fmaxf(o1.y, 0.f); o1.z = fmaxf(o1.z, 0.f); o1.w = fmaxf(o1.w, 0.f);
        }
        float* dst = out + row * HH + tx * 8;
        *reinterpret_cast<float4*>(dst) = o0;
        *reinterpret_cast<float4*>(dst + 4) = o1;
    }
}

// ------------------------------------------------------------------------------------------
// Heads.  One warp per node.
__global__ void __launch_bounds__(256) sage_node_head_kernel(const float* __restrict__ h, const float* __restrict__ node_w,
                                                             float node_b, float* __restrict__ score,
                                                             const float* __restrict__ edge_W, float* __restrict__ proj,
                                                             int64_t row_begin, int64_t row_end, int H) {
    const int lane = threadIdx.x & 31;
    const int64_t row = row_begin + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= row_end) return;
    float s = 0.f, p0 = 0.f, p1 = 0.f, p2 = 0.f, p3 = 0.f;
    for (int k = lane * 4; k < H; k += 128) {
        const float4 hv = ldg4(h + row * H + k);
        const float4 wv = ldg4(node_w + k);
        s += hv.x * wv.x + hv.y * wv.y + hv.z * wv.z + hv.w * wv.w;
        if (edge_W) {
            const float hh[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                p0 += hh[j] * __ldg(edge_W + (k + j) * 2 + 0);
                p1 += hh[j] * __ldg(edge_W + (k + j) * 2 + 1);
                p2 += hh[j] * __ldg(edge_W + (H + k + j) * 2 + 0);
                p3 += hh[j] * __ldg(edge_W + (H + k + j) * 2 + 1);
            }
        }
    }
    s = warp_sum(s);
    if (edge_W) { p0 = warp_sum(p0); p1 = warp_sum(p1); p2 = warp_sum(p2); p3 = warp_sum(p3); }
    if (lane == 0) {
        score[row] = 1.f / (1.f + expf(-(s + node_b)));
        if (edge_W) *reinterpret_cast<float4*>(proj + row * 4) = make_float4(p0, p1, p2, p3);
    }
}

template <typename RP>
__global__ void __launch_bounds__(256) sage_edge_head_kernel(const float* __restrict__ proj, const RP* __restrict__ rowptr,
                                                             const int32_t* __restrict__ col, const float* __restrict__ edge_b,
                                                             float* __restrict__ logit, int64_t row_begin, int64_t row_end) {
    // one warp per destination row; lanes stride over the row's edges
    const int lane = threadIdx.x & 31;
    const int64_t row = row_begin + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= row_end) return;
    const float4 pd = ldg4(proj + row * 4);
    const float b0 = __ldg(edge_b), b1 = __ldg(edge_b + 1);
    const int64_t e0 = rowptr[row], e1 = rowptr[row + 1];
    for (int64_t e = e0 + lane; e < e1; e += 32) {
        const float4 ps = ldg4(proj + (int64_t)col[e] * 4);
        *reinterpret_cast<float2*>(logit + e * 2) = make_float2(ps.x + pd.z + b0, ps.y + pd.w + b1);
    }
}

// ------------------------------------------------------------------------------------------
template <int F, typename RP>
static int launch_ffma(const float* x, const RP* rowptr, const int32_t* col, const float* ew, const float* W,
                       const float* b, float* out, int64_t row_begin, int64_t row_end, int relu, cudaStream_t st) {
    using C = FfmaCfg<F>;
    const int rc = set_max_dynamic_smem((const void*)sage_layer_ffma_kernel<F, RP>, C::smem);
    if (rc) return rc;
    const int64_t rows = row_end - row_begin;
    const int64_t tiles = (rows + BM - 1) / BM;
    if (tiles == 0) return NERRF_OK;
    NERRF_REQUIRE(tiles < (1ll << 31), "too many row tiles");
    sage_layer_ffma_kernel<F, RP><<<(unsigned)tiles, 256, C::smem, st>>>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu);
    return launch_status("sage_layer_ffma_kernel");
}

template <typename RP>
static int layer_dispatch(const float* x, const RP* rowptr, const int32_t* col, const float* ew, const float* W,
                          const float* b, float* out, int64_t row_begin, int64_t row_end, int F, int relu,
                          cudaStream_t st) {
    switch (F) {
        case 32: return launch_ffma<32, RP>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu, st);
        case 64: return launch_ffma<64, RP>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu, st);
        case 128: return launch_ffma<128, RP>(x, rowptr, col, ew, W, b, out, row_begin, row_end, relu, st);
    }
    set_error("unsupported feature width F=%d (supported: 32, 64, 128)", F);
    return NERRF_ERR_INVALID;
}

static int check_graph_args(const void* x, const void* rowptr, const void* col, const void* ew, int64_t n_nodes,
                            int64_t row_begin, int64_t row_end) {
    NERRF_REQUIRE(x && rowptr, "null graph pointer");   // col / ew may be null when the graph has no edges
    (void)col; (void)ew;
    NERRF_REQUIRE(n_nodes >= 0 && row_begin >= 0 && row_begin <= row_end && row_end <= n_nodes,
                  "bad row range [%lld,%lld) for %lld nodes", (long long)row_begin, (long long)row_end, (long long)n_nodes);
    NERRF_REQUIRE(((uintptr_t)x & 15) == 0, "x must be 16-byte aligned");
    return NERRF_OK;
}

}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_sage_aggregate(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                                    const float* ew, float* m, int64_t n_nodes, int64_t row_begin, int64_t row_end,
                                    int F, nerrf_stream_t stream) {
    int rc = check_graph_args(x, rowptr, col, ew, n_nodes, row_begin, row_end);
    if (rc) return rc;
    NERRF_REQUIRE(m, "null output");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t rows = row_end - row_begin;
    if (rows == 0) return NERRF_OK;
    const unsigned grid = (unsigned)((rows + 7) / 8);
#define AGG(FV)                                                                                                         \
    if (rowptr_is64)                                                                                                    \
        sage_aggregate_kernel<FV, int64_t><<<grid, 256, 0, st>>>(x, (const int64_t*)rowptr, col, ew, m, row_begin, row_end); \
    else                                                                                                                \
        sage_aggregate_kernel<FV, int32_t><<<grid, 256, 0, st>>>(x, (const int32_t*)rowptr, col, ew, m, row_begin, row_end);
    switch (F) {
        case 32: AGG(32); break;
        case 64: AGG(64); break;
        case 128: AGG(128); break;
        default: set_error("unsupported feature width F=%d (supported: 32, 64, 128)", F); return NERRF_ERR_INVALID;
    }
#undef AGG
    return launch_status("sage_aggregate_kernel");
}

static int layer_fwd_impl(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col, const float* ew,
                          const float* W, const float* b, float* out, int64_t n_nodes, int64_t row_begin, int64_t row_end,
                          int F, int H, int relu, int algo, const float* node_w, float node_b, float* score,
                          void* long_ws, size_t long_ws_bytes, float* const* peer_out, int n_peers,
                          const uint8_t* peer_need, nerrf_stream_t stream) {
    int rc = check_graph_args(x, rowptr, col, ew, n_nodes, row_begin, row_end);
    if (rc) return rc;
    NERRF_REQUIRE(W && b && out, "null weight/output pointer");
    NERRF_REQUIRE(H == HH, "hidden width must be 128 (got %d)", H);
    NERRF_REQUIRE(((uintptr_t)out & 15) == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)b & 15) == 0 &&
                  ((uintptr_t)node_w & 15) == 0, "out/W/b/node_w must be 16-byte aligned");
    NERRF_REQUIRE(x != out, "in-place layer is not supported");
    NERRF_REQUIRE(!node_w || score, "score output required with node_w");
    cudaStream_t st = (cudaStream_t)stream;
    const bool reuse_scan = (algo & NERRF_SAGE_FLAG_REUSE_LONG_SCAN) != 0;
    const int l2_policy = (algo & NERRF_SAGE_FLAG_NO_L2_POLICY) ? 0 : 1;
    algo &= 0xFF;
    if (algo == NERRF_SAGE_ALGO_AUTO) algo = NERRF_SAGE_ALGO_UMMA;
    if (algo == NERRF_SAGE_ALGO_UMMA || algo == NERRF_SAGE_ALGO_UMMA2)
        return sage_layer_umma(x, rowptr, rowptr_is64, col, ew, W, b, out, n_nodes, row_begin, row_end, F, relu,
                               algo == NERRF_SAGE_ALGO_UMMA ? 3 : 2, node_w, node_b, score, long_ws, long_ws_bytes,
                               reuse_scan, peer_out, n_peers, peer_need, l2_policy, st);
    NERRF_REQUIRE(n_peers == 0, "the fused peer exchange needs the tensor-core layer (algo umma)");
    NERRF_REQUIRE(algo == NERRF_SAGE_ALGO_FFMA, "unknown algo %d", algo);
    rc = rowptr_is64
             ? layer_dispatch<int64_t>(x, (const int64_t*)rowptr, col, ew, W, b, out, row_begin, row_end, F, relu, st)
             : layer_dispatch<int32_t>(x, (const int32_t*)rowptr, col, ew, W, b, out, row_begin, row_end, F, relu, st);
    if (rc || !node_w) return rc;
    return nerrf_sage_node_head(out, node_w, node_b, score, nullptr, nullptr, row_begin, row_end, H, stream);
}

extern "C" int nerrf_sage_layer_fwd(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                                    const float* ew, const float* W, const float* b, float* out, int64_t n_nodes,
                                    int64_t row_begin, int64_t row_end, int F, int H, int relu, int algo,
                                    nerrf_stream_t stream) {
    return layer_fwd_impl(x, rowptr, rowptr_is64, col, ew, W, b, out, n_nodes, row_begin, row_end, F, H, relu, algo,
                          nullptr, 0.f, nullptr, nullptr, 0, nullptr, 0, nullptr, stream);
}

extern "C" int nerrf_sage_layer_head_fwd(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                                         const float* ew, const float* W, const float* b, float* out, int64_t n_nodes,
                                         int64_t row_begin, int64_t row_end, int F, int H, int relu, int algo,
                                         const float* node_w, float node_b, float* score, nerrf_stream_t stream) {
    NERRF_REQUIRE(node_w && score, "null head pointer");
    return layer_fwd_impl(x, rowptr, rowptr_is64, col, ew, W, b, out, n_nodes, row_begin, row_end, F, H, relu, algo, node_w,
                          node_b, score, nullptr, 0, nullptr, 0, nullptr, stream);
}

extern "C" int nerrf_sage_long_rows_workspace_bytes(int64_t n_edges, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_edges >= 0, "bad argument");
    // rows with more than 128 in-edges are cut into 256-edge chunks: <= n_edges/256 full chunks + one partial chunk per
    // such row (<= n_edges/128 rows); 560 B per chunk item.  Capacity driven: what does not fit is processed inline.
    const int64_t items = 3 * (n_edges / 256) + 64;
    *bytes = (size_t)items * 560 + 8192;
    return NERRF_OK;
}

extern "C" int nerrf_sage_layer_fwd_ex(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                                       const float* ew, const float* W, const float* b, float* out, int64_t n_nodes,
                                       int64_t row_begin, int64_t row_end, int F, int H, int relu, int algo,
                                       const float* node_w, float node_b, float* score, void* long_ws,
                                       size_t long_ws_bytes, float* const* peer_out, int n_peers,
                                       const uint8_t* peer_need, nerrf_stream_t stream) {
    NERRF_REQUIRE(n_peers == 0 || peer_out, "peer_out required with n_peers != 0");
    return layer_fwd_impl(x, rowptr, rowptr_is64, col, ew, W, b, out, n_nodes, row_begin, row_end, F, H, relu, algo, node_w,
                          node_b, score, long_ws, long_ws_bytes, peer_out, n_peers, peer_need, stream);
}

extern "C" int nerrf_sage_node_head(const float* h, const float* node_w, float node_b, float* score,
                                    const float* edge_W, float* proj, int64_t row_begin, int64_t row_end, int H,
                                    nerrf_stream_t stream) {
    NERRF_REQUIRE(h && node_w && score, "null pointer");
    NERRF_REQUIRE(H % 4 == 0 && H > 0, "H must be a positive multiple of 4");
    NERRF_REQUIRE(!edge_W || proj, "proj output required with edge_W");
    NERRF_REQUIRE(row_begin >= 0 && row_begin <= row_end, "bad row range");
    const int64_t rows = row_end - row_begin;
    if (rows == 0) return NERRF_OK;
    sage_node_head_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(h, node_w, node_b, score, edge_W,
                                                                                         proj, row_begin, row_end, H);
    return launch_status("sage_node_head_kernel");
}

extern "C" int nerrf_sage_edge_head(const float* proj, const void* rowptr, int rowptr_is64, const int32_t* col,
                                    const float* edge_b, float* edge_logit, int64_t row_begin, int64_t row_end,
                                    nerrf_stream_t stream) {
    NERRF_REQUIRE(proj && rowptr && edge_b, "null pointer");     // col / edge_logit may be null when the graph has no edges
    NERRF_REQUIRE(row_begin >= 0 && row_begin <= row_end, "bad row range");
    const int64_t rows = row_end - row_begin;
    if (rows == 0) return NERRF_OK;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (rowptr_is64)
        sage_edge_head_kernel<int64_t><<<grid, 256, 0, st>>>(proj, (const int64_t*)rowptr, col, edge_b, edge_logit, row_begin, row_end);
    else
        sage_edge_head_kernel<int32_t><<<grid, 256, 0, st>>>(proj, (const int32_t*)rowptr, col, edge_b, edge_logit, row_begin, row_end);
    return launch_status("sage_edge_head_kernel");
}

extern "C" int nerrf_sage_forward(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                                  const float* ew, int64_t n_nodes, int f_in, int hidden, int num_layers,
                                  const float* const* W, const float* const* b, const float* node_w, float node_b,
                                  float* h_out, float* score_out, float* workspace, size_t workspace_bytes, int algo,
                                  nerrf_stream_t stream) {
    NERRF_REQUIRE(num_layers >= 1 && num_layers <= 64, "num_layers out of range");
    NERRF_REQUIRE(W && b && h_out, "null pointer");
    if (num_layers > 1) {
        NERRF_REQUIRE(workspace, "workspace required for num_layers > 1");
        if (workspace_bytes < (size_t)n_nodes * hidden * sizeof(float)) {
            set_error("workspace too small: need %zu bytes", (size_t)n_nodes * hidden * sizeof(float));
            return NERRF_ERR_WORKSPACE;
        }
    }
    if (score_out) NERRF_REQUIRE(node_w, "node_w required for score_out");
    // workspace beyond the [n_nodes, hidden] ping-pong buffer (if any) is the hub-row pre-aggregation scratch
    const size_t pp = num_layers > 1 ? (((size_t)n_nodes * hidden * sizeof(float) + 255) & ~(size_t)255) : 0;
    void* long_ws = (workspace && workspace_bytes > pp + 8192) ? (void*)((unsigned char*)workspace + pp) : nullptr;
    const size_t long_ws_bytes = long_ws ? workspace_bytes - pp : 0;
    const float* in = x;
    int F = f_in;
    for (int l = 0; l < num_layers; ++l) {
        float* o = ((num_layers - 1 - l) % 2 == 0) ? h_out : workspace;
        const bool last = l == num_layers - 1;
        int rc = layer_fwd_impl(in, rowptr, rowptr_is64, col, ew, W[l], b[l], o, n_nodes, 0, n_nodes, F, hidden, 1,
                                layer_algo(algo, l > 0),
                                (last && score_out) ? node_w : nullptr, node_b, (last && score_out) ? score_out : nullptr,
                                long_ws, long_ws_bytes, nullptr, 0, nullptr, stream);
        if (rc) return rc;
        in = o;
        F = hidden;
    }
    return NERRF_OK;
}

// ------------------------------------------------------------------------------------------ session
static size_t session_ws_bytes(int64_t max_nodes, int64_t max_edges, int hidden) {
    size_t lb = 0;
    nerrf_sage_long_rows_workspace_bytes(max_edges, &lb);
    return (((size_t)max_nodes * hidden * 4 + 255) & ~(size_t)255) + lb;
}

constexpr int SESSION_CHUNKS = 4;
constexpr int SESSION_SLOTS = 2;      // input / score buffer sets: the upload of step i+1 runs under the compute of step i

struct nerrf_sage_session {
    int64_t max_nodes, max_edges;
    int f_in, hidden, L;
    float *x[SESSION_SLOTS], *ew[SESSION_SLOTS], *score[SESSION_SLOTS];
    int32_t *rowptr[SESSION_SLOTS], *col[SESSION_SLOTS];
    float *h, *ws, *node_w;         // activations: one set (the compute of consecutive steps is serial on `st`)
    float* Wd[64];
    float* bd[64];
    float node_b;
    cudaStream_t st;                // compute
    cudaStream_t cst;               // H2D: the edge arrays arrive in row-aligned chunks while layer 1 already runs
    cudaStream_t dst;               // D2H of the scores (PCIe is full duplex: it runs under the next step's upload)
    cudaEvent_t ev[SESSION_SLOTS][SESSION_CHUNKS];
    cudaEvent_t compute_done[SESSION_SLOTS], out_done[SESSION_SLOTS];
    uint64_t next_ticket;           // tickets are 1, 2, ...; ticket t uses slot t % SESSION_SLOTS
    uint64_t slot_ticket[SESSION_SLOTS];   // ticket whose work is (or was last) queued on the slot, 0 = none
    bool has_weights;
};

extern "C" int nerrf_sage_session_create(int64_t max_nodes, int64_t max_edges, int f_in, int hidden, int num_layers,
                                         nerrf_sage_session** out) {
    NERRF_REQUIRE(out, "null out");
    NERRF_REQUIRE(max_nodes > 0 && max_edges >= 0 && num_layers >= 1 && num_layers <= 64, "bad session sizes");
    NERRF_REQUIRE(max_edges < (1ll << 31), "host session uses int32 rowptr: max_edges must be < 2^31");
    nerrf_sage_session* s = new nerrf_sage_session();
    memset(s, 0, sizeof(*s));
    s->max_nodes = max_nodes; s->max_edges = max_edges; s->f_in = f_in; s->hidden = hidden; s->L = num_layers;
    cudaError_t e = cudaSuccess;
    auto A = [&](void** p, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(p, bytes ? bytes : 16); };
    for (int k = 0; k < SESSION_SLOTS; ++k) {
        A((void**)&s->x[k], (size_t)max_nodes * f_in * 4);
        A((void**)&s->rowptr[k], (size_t)(max_nodes + 1) * 4);
        A((void**)&s->col[k], (size_t)max_edges * 4);
        A((void**)&s->ew[k], (size_t)max_edges * 4);
        A((void**)&s->score[k], (size_t)max_nodes * 4);
    }
    A((void**)&s->h, (size_t)max_nodes * hidden * 4);
    A((void**)&s->ws, session_ws_bytes(max_nodes, max_edges, hidden));
    A((void**)&s->node_w, (size_t)hidden * 4);
    int F = f_in;
    for (int l = 0; l < num_layers; ++l) {
        A((void**)&s->Wd[l], (size_t)2 * F * hidden * 4);
        A((void**)&s->bd[l], (size_t)hidden * 4);
        F = hidden;
    }
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->cst, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->dst, cudaStreamNonBlocking);
    for (int k = 0; k < SESSION_SLOTS; ++k) {
        for (int i = 0; i < SESSION_CHUNKS && e == cudaSuccess; ++i) e = cudaEventCreateWithFlags(&s->ev[k][i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->compute_done[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->out_done[k], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) {
        set_error("session allocation failed: %s", cudaGetErrorString(e));
        nerrf_sage_session_destroy(s);
        return NERRF_ERR_CUDA;
    }
    *out = s;
    return NERRF_OK;
}

extern "C" int nerrf_sage_session_set_weights(nerrf_sage_session* s, const float* const* W, const float* const* b,
                                              const float* node_w, float node_b) {
    NERRF_REQUIRE(s && W && b && node_w, "null pointer");
    NERRF_CHECK_CUDA(cudaStreamSynchronize(s->st));                  // steps in flight read the old weights
    int F = s->f_in;
    for (int l = 0; l < s->L; ++l) {
        NERRF_CHECK_CUDA(cudaMemcpyAsync(s->Wd[l], W[l], (size_t)2 * F * s->hidden * 4, cudaMemcpyHostToDevice, s->st));
        NERRF_CHECK_CUDA(cudaMemcpyAsync(s->bd[l], b[l], (size_t)s->hidden * 4, cudaMemcpyHostToDevice, s->st));
        F = s->hidden;
    }
    NERRF_CHECK_CUDA(cudaMemcpyAsync(s->node_w, node_w, (size_t)s->hidden * 4, cudaMemcpyHostToDevice, s->st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(s->st));
    s->node_b = node_b;
    s->has_weights = true;
    return NERRF_OK;
}

// Queue one step: H2D of the graph (copy stream) -> forward (compute stream) -> D2H of the scores (third stream), all
// asynchronous.  Two buffer sets: the upload of ticket t+1 overlaps the layers of ticket t, whose score read-back
// overlaps both -- the steady state of a stream of graphs (one per sliding-window tick) is bounded by PCIe H2D time
// alone.  The host buffers of a ticket must stay valid and unmodified until nerrf_sage_session_wait(ticket) returns.
extern "C" int nerrf_sage_session_submit_host(nerrf_sage_session* s, const float* x_host, const int32_t* rowptr_host,
                                              const int32_t* col_host, const float* ew_host, int64_t n_nodes,
                                              int64_t n_edges, float* score_out_host, float* h_out_host, int algo,
                                              uint64_t* ticket) {
    NERRF_REQUIRE(s && x_host && rowptr_host && col_host && ew_host && ticket, "null pointer");
    NERRF_REQUIRE(s->has_weights, "session has no weights (call nerrf_sage_session_set_weights)");
    NERRF_REQUIRE(n_nodes >= 0 && n_nodes <= s->max_nodes && n_edges >= 0 && n_edges <= s->max_edges,
                  "graph (%lld nodes, %lld edges) exceeds the session capacity", (long long)n_nodes, (long long)n_edges);
    const uint64_t t = ++s->next_ticket;
    const int k = (int)(t % SESSION_SLOTS);
    *ticket = t;
    if (s->slot_ticket[k]) NERRF_CHECK_CUDA(cudaEventSynchronize(s->out_done[k]));   // at most SESSION_SLOTS steps in flight
    s->slot_ticket[k] = t;
    cudaStream_t st = s->st, cst = s->cst, dst = s->dst;
    if (n_nodes == 0) {
        NERRF_CHECK_CUDA(cudaEventRecord(s->compute_done[k], st));
        NERRF_CHECK_CUDA(cudaEventRecord(s->out_done[k], st));
        return NERRF_OK;
    }
    float *dx = s->x[k], *dew = s->ew[k], *dscore = s->score[k];
    int32_t *drp = s->rowptr[k], *dcol = s->col[k];
    const size_t ws_bytes = session_ws_bytes(s->max_nodes, s->max_edges, s->hidden);
    int rc;
    // the slot's inputs were last read by the compute of ticket t - SESSION_SLOTS (complete: out_done was waited above)
    if (s->L >= 2 && n_edges >= (1 << 20)) {
        // Overlap inside a step (VERDICT r1 #8): x and rowptr first, then col / ew in SESSION_CHUNKS edge-balanced,
        // row-aligned chunks; layer 1 of a row range starts as soon as its edge chunk has landed.  Layers 2.. need the
        // whole h_1 and therefore the whole upload.
        int64_t cut[SESSION_CHUNKS + 1];
        cut[0] = 0; cut[SESSION_CHUNKS] = n_nodes;
        for (int c = 1; c < SESSION_CHUNKS; ++c) {                   // first row whose edge offset reaches c/C of the edges
            const int64_t target = n_edges * c / SESSION_CHUNKS;
            int64_t lo = cut[c - 1], hi = n_nodes;
            while (lo < hi) { const int64_t mid = (lo + hi) / 2; if ((int64_t)rowptr_host[mid] < target) lo = mid + 1; else hi = mid; }
            cut[c] = lo;
        }
        NERRF_CHECK_CUDA(cudaMemcpyAsync(drp, rowptr_host, (size_t)(n_nodes + 1) * 4, cudaMemcpyHostToDevice, cst));
        NERRF_CHECK_CUDA(cudaMemcpyAsync(dx, x_host, (size_t)n_nodes * s->f_in * 4, cudaMemcpyHostToDevice, cst));
        for (int c = 0; c < SESSION_CHUNKS; ++c) {
            const int64_t e0 = rowptr_host[cut[c]], e1 = rowptr_host[cut[c + 1]];
            if (e1 > e0) {
                NERRF_CHECK_CUDA(cudaMemcpyAsync(dcol + e0, col_host + e0, (size_t)(e1 - e0) * 4, cudaMemcpyHostToDevice, cst));
                NERRF_CHECK_CUDA(cudaMemcpyAsync(dew + e0, ew_host + e0, (size_t)(e1 - e0) * 4, cudaMemcpyHostToDevice, cst));
            }
            NERRF_CHECK_CUDA(cudaEventRecord(s->ev[k][c], cst));
        }
        const size_t pp = (((size_t)n_nodes * s->hidden * sizeof(float) + 255) & ~(size_t)255);
        void* long_ws = ws_bytes > pp + 8192 ? (void*)((unsigned char*)s->ws + pp) : nullptr;
        const size_t long_ws_bytes = long_ws ? ws_bytes - pp : 0;
        const float* in = dx;
        int F = s->f_in;
        for (int l = 0; l < s->L; ++l) {
            float* o = ((s->L - 1 - l) % 2 == 0) ? s->h : s->ws;
            const bool last = l == s->L - 1;
            if (l == 0) {
                for (int c = 0; c < SESSION_CHUNKS; ++c) {
                    NERRF_CHECK_CUDA(cudaStreamWaitEvent(st, s->ev[k][c], 0));
                    if (cut[c + 1] > cut[c]) {
                        rc = layer_fwd_impl(in, drp, 0, dcol, dew, s->Wd[l], s->bd[l], o, n_nodes, cut[c], cut[c + 1], F, s->hidden, 1,
                                            layer_algo(algo, false), nullptr, 0.f, nullptr, long_ws, long_ws_bytes, nullptr, 0, nullptr, st);
                        if (rc) return rc;
                    }
                }
            } else {
                rc = layer_fwd_impl(in, drp, 0, dcol, dew, s->Wd[l], s->bd[l], o, n_nodes, 0, n_nodes, F, s->hidden, 1,
                                    layer_algo(algo, l > 1), last ? s->node_w : nullptr, s->node_b,
                                    last ? dscore : nullptr, long_ws, long_ws_bytes, nullptr, 0, nullptr, st);
                if (rc) return rc;
            }
            in = o;
            F = s->hidden;
        }
    } else {
        NERRF_CHECK_CUDA(cudaMemcpyAsync(drp, rowptr_host, (size_t)(n_nodes + 1) * 4, cudaMemcpyHostToDevice, cst));
        NERRF_CHECK_CUDA(cudaMemcpyAsync(dcol, col_host, (size_t)n_edges * 4, cudaMemcpyHostToDevice, cst));
        NERRF_CHECK_CUDA(cudaMemcpyAsync(dew, ew_host, (size_t)n_edges * 4, cudaMemcpyHostToDevice, cst));
        NERRF_CHECK_CUDA(cudaMemcpyAsync(dx, x_host, (size_t)n_nodes * s->f_in * 4, cudaMemcpyHostToDevice, cst));
        NERRF_CHECK_CUDA(cudaEventRecord(s->ev[k][0], cst));
        NERRF_CHECK_CUDA(cudaStreamWaitEvent(st, s->ev[k][0], 0));
        rc = nerrf_sage_forward(dx, drp, 0, dcol, dew, n_nodes, s->f_in, s->hidden, s->L, s->Wd, s->bd,
                                s->node_w, s->node_b, s->h, dscore, s->ws, ws_bytes, algo, st);
        if (rc) return rc;
    }
    if (h_out_host)     // the activations are shared by consecutive steps: their read-back stays on the compute stream
        NERRF_CHECK_CUDA(cudaMemcpyAsync(h_out_host, s->h, (size_t)n_nodes * s->hidden * 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaEventRecord(s->compute_done[k], st));
    NERRF_CHECK_CUDA(cudaStreamWaitEvent(dst, s->compute_done[k], 0));
    if (score_out_host)
        NERRF_CHECK_CUDA(cudaMemcpyAsync(score_out_host, dscore, (size_t)n_nodes * 4, cudaMemcpyDeviceToHost, dst));
    NERRF_CHECK_CUDA(cudaEventRecord(s->out_done[k], dst));
    return NERRF_OK;
}

extern "C" int nerrf_sage_session_wait(nerrf_sage_session* s, uint64_t ticket) {
    NERRF_REQUIRE(s, "null session");
    NERRF_REQUIRE(ticket >= 1 && ticket <= s->next_ticket, "unknown ticket %llu", (unsigned long long)ticket);
    const int k = (int)(ticket % SESSION_SLOTS);
    if (s->slot_ticket[k] != ticket) return NERRF_OK;                // an older ticket: its slot was reused, i.e. it completed
    NERRF_CHECK_CUDA(cudaEventSynchronize(s->out_done[k]));
    return NERRF_OK;
}

extern "C" int nerrf_sage_session_forward_host(nerrf_sage_session* s, const float* x_host, const int32_t* rowptr_host,
                                               const int32_t* col_host, const float* ew_host, int64_t n_nodes,
                                               int64_t n_edges, float* score_out_host, float* h_out_host, int algo) {
    uint64_t t = 0;
    int rc = nerrf_sage_session_submit_host(s, x_host, rowptr_host, col_host, ew_host, n_nodes, n_edges, score_out_host,
                                            h_out_host, algo, &t);
    if (rc) return rc;
    return nerrf_sage_session_wait(s, t);
}

extern "C" int nerrf_sage_session_destroy(nerrf_sage_session* s) {
    if (!s) return NERRF_OK;
    if (s->st) cudaStreamSynchronize(s->st);
    if (s->cst) cudaStreamSynchronize(s->cst);
    if (s->dst) cudaStreamSynchronize(s->dst);
    for (int k = 0; k < SESSION_SLOTS; ++k) {
        cudaFree(s->x[k]); cudaFree(s->rowptr[k]); cudaFree(s->col[k]); cudaFree(s->ew[k]); cudaFree(s->score[k]);
        for (int i = 0; i < SESSION_CHUNKS; ++i) if (s->ev[k][i]) cudaEventDestroy(s->ev[k][i]);
        if (s->compute_done[k]) cudaEventDestroy(s->compute_done[k]);
        if (s->out_done[k]) cudaEventDestroy(s->out_done[k]);
    }
    cudaFree(s->h); cudaFree(s->ws); cudaFree(s->node_w);
    for (int l = 0; l < 64; ++l) { if (s->Wd[l]) cudaFree(s->Wd[l]); if (s->bd[l]) cudaFree(s->bd[l]); }
    if (s->st) cudaStreamDestroy(s->st);
    if (s->cst) cudaStreamDestroy(s->cst);
    if (s->dst) cudaStreamDestroy(s->dst);
    delete s;
    return NERRF_OK;
}
