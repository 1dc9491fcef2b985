// BiLSTM BACKWARD-THROUGH-TIME (training; the BiLSTM half of ai/train.py "joint GNN+LSTM training script", README.md:75).
// fp32 on CUDA cores, deterministic (no atomics: every reduction has a fixed order).  Spec = oracle/lstm_ref.py (torch gate
// order i, f, g, o; packed-sequence masking; bidirectional stack); the fp64 statement of this backward is
// oracle/lstm_bwd_ref.py.  Reads the tape nerrf_lstm_forward_train writes (lstm_tape.cuh).
//
// Per layer, top layer first:
//   lstm_bwd_rec_kernel    the recurrence, mirroring lstm_layer_kernel: one CTA = 8 sequences x one direction, 256 threads,
//                          thread j owns hidden unit j, dh / dc in registers.  Steps run in reverse direction order; the
//                          pre-activation gate gradients dg are staged in shared memory [4H][8] and overwrite the saved
//                          gates in the tape (zero at padded steps); dh_{t-1} = sum_r dg[r] W_hh[r, j] reads W_hh in
//                          torch's [4H, H] layout, coalesced across j.
//   lstm_bwd_dw_kernel     dW_ih = dg^T in_l, dW_hh = dg^T h_prev, db = sum dg over all B*T rows: each CTA accumulates a
//                          64 x 64 slab over the rows of one chunk of sequences and writes a partial (both directions in
//                          one launch); the chunking depends on B only, so the bits do not depend on the device
//   lstm_bwd_reduce_kernel partials -> gradients, chunk order fixed
//   lstm_bwd_din_kernel    d in_l = [dg_fwd || dg_bwd] [W_ih_fwd ; W_ih_bwd], K = 8H (the directions add in a fixed order);
//                          the injected gradient of layer l-1's output, or dseq at l = 0
// nerrf_lstm_input_grad is the same backward without the weight gradients (explanations, DESIGN.md 1.2.1): the recurrence
// and din launches only, so its dseq equals nerrf_lstm_backward's bit for bit, and its workspace is the dout buffer.
#include "common.cuh"
#include "lstm_tape.cuh"

namespace nerrf {
namespace {

constexpr int H = LstmTape::H;
constexpr int BS = 8;                 // sequences per recurrence CTA
constexpr int REC_SMEM = 2 * 4 * H * BS * (int)sizeof(float);   // double-buffered dg staging

constexpr int GT = 64;                // GEMM tile (both output dimensions)
constexpr int GK = 32;                // reduction depth per shared-memory stage
constexpr int GLD = GT + 4;
constexpr int MAX_CHUNKS = 32;        // row chunks of the weight-gradient reduction (a function of the shape only)

__device__ __forceinline__ int clamp_len(int v, int T) { return v < 0 ? 0 : (v > T ? T : v); }

__global__ void __launch_bounds__(H, 1)
lstm_bwd_rec_kernel(const int32_t* __restrict__ len, int64_t B, int T,
                    const float* __restrict__ Whh_f, const float* __restrict__ Whh_b,   // torch layout [4H, H]
                    float* __restrict__ gates,          // [2][B, T, 4H]: saved gates in, dg out
                    const float* __restrict__ cell,     // [2][B, T, H]
                    const float* __restrict__ dout,     // [B, T, 2H] gradient of this layer's output, or nullptr (top)
                    const float* __restrict__ dhfin)    // [B, 2H] (top layer)
{
    extern __shared__ __align__(16) float dg_s[];       // [2][4H][BS]
    __shared__ int len_s[BS];
    const int j = threadIdx.x;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * BS;
    const float* Whh = dir ? Whh_b : Whh_f;
    float* G = gates + (int64_t)dir * B * T * (4 * H);
    const float* C = cell + (int64_t)dir * B * T * H;

    if (j < BS) len_s[j] = (b0 + j < B) ? clamp_len(len[b0 + j], T) : 0;
    float dh[BS], dc[BS];
#pragma unroll
    for (int b = 0; b < BS; ++b) { dh[b] = 0.f; dc[b] = 0.f; }
    __syncthreads();

    int buf = 0;
    for (int step = 0; step < T; ++step) {
        const int t = dir ? step : (T - 1 - step);
        float* dg = dg_s + buf * (4 * H * BS);
#pragma unroll
        for (int b = 0; b < BS; ++b) {
            const int L = len_s[b];
            float gi = 0.f, gf = 0.f, gg = 0.f, go = 0.f;
            const int64_t row = (b0 + b) * (int64_t)T + t;
            if (t < L) {
                float* gp = G + row * (4 * H) + j;
                const float i_ = gp[0], f_ = gp[H], g_ = gp[2 * H], o_ = gp[3 * H];
                const float c_ = C[row * H + j];
                float cp = 0.f;                                     // c_{t-1} in this direction's order
                if (dir == 0) { if (t > 0) cp = C[(row - 1) * H + j]; }
                else if (t + 1 < L) cp = C[(row + 1) * H + j];
                float inj;
                if (dout) inj = dout[row * (2 * H) + dir * H + j];
                else inj = (t == (dir ? 0 : L - 1)) ? dhfin[(b0 + b) * (2 * H) + dir * H + j] : 0.f;
                const float h = dh[b] + inj;
                const float tc = tanhf(c_);
                const float d_c = fmaf(h * o_, 1.f - tc * tc, dc[b]);
                gi = d_c * g_ * (i_ * (1.f - i_));
                gf = d_c * cp * (f_ * (1.f - f_));
                gg = d_c * i_ * (1.f - g_ * g_);
                go = h * tc * (o_ * (1.f - o_));
                dc[b] = d_c * f_;
                gp[0] = gi; gp[H] = gf; gp[2 * H] = gg; gp[3 * H] = go;
            } else if (b0 + b < B) {
                float* gp = G + row * (4 * H) + j;
                gp[0] = 0.f; gp[H] = 0.f; gp[2 * H] = 0.f; gp[3 * H] = 0.f;
            }
            dg[(0 * H + j) * BS + b] = gi; dg[(1 * H + j) * BS + b] = gf;
            dg[(2 * H + j) * BS + b] = gg; dg[(3 * H + j) * BS + b] = go;
        }
        __syncthreads();
        float acc[BS];
#pragma unroll
        for (int b = 0; b < BS; ++b) acc[b] = 0.f;
#pragma unroll 8
        for (int r = 0; r < 4 * H; ++r) {
            const float w = __ldg(Whh + (size_t)r * H + j);
            const float4 v0 = *reinterpret_cast<const float4*>(dg + r * BS);
            const float4 v1 = *reinterpret_cast<const float4*>(dg + r * BS + 4);
            acc[0] = fmaf(w, v0.x, acc[0]); acc[1] = fmaf(w, v0.y, acc[1]);
            acc[2] = fmaf(w, v0.z, acc[2]); acc[3] = fmaf(w, v0.w, acc[3]);
            acc[4] = fmaf(w, v1.x, acc[4]); acc[5] = fmaf(w, v1.y, acc[5]);
            acc[6] = fmaf(w, v1.z, acc[6]); acc[7] = fmaf(w, v1.w, acc[7]);
        }
#pragma unroll
        for (int b = 0; b < BS; ++b)
            if (t < len_s[b]) dh[b] = acc[b];
        buf ^= 1;            // double buffer: the next step writes the other half, so one barrier per step suffices
    }
}

// acc[a][c] += sum_k As[k][4 ty + a] * Bs[k][4 tx + c]
__device__ __forceinline__ void tile_acc(const float* As, const float* Bs, int tx, int ty, float (&acc)[4][4]) {
#pragma unroll 8
    for (int k = 0; k < GK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(As + k * GLD + 4 * ty);
        const float4 b = *reinterpret_cast<const float4*>(Bs + k * GLD + 4 * tx);
        const float aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[i][c] = fmaf(aa[i], bb[c], acc[i][c]);
    }
}

// part[dir][chunk][m][n] = sum over the chunk's rows r = b*T + t of dg_dir[r][m] * X_dir[r][n], where
// X_dir[r][n] = x[(b*T + t + shift[dir]) * ldx + xoff[dir] + n] if 0 <= t + shift < len[b], else 0.
// (dW_ih: x = in_l, shift 0;  dW_hh: x = out_l, shift -1 / +1 = the previous step in each direction's order.)
// With dbpart, CTAs of n-tile 0 also write dbpart[dir][chunk][m] = sum dg_dir[r][m].
__global__ void __launch_bounds__(256)
lstm_bwd_dw_kernel(const float* __restrict__ gates, const float* __restrict__ x, int ldx, int xoff_b, int N,
                   const int32_t* __restrict__ len, int64_t B, int T, int64_t seqs_per_chunk, int chunks,
                   float* __restrict__ part, float* __restrict__ dbpart, int shift) {
    __shared__ __align__(16) float As[GK * GLD];
    __shared__ __align__(16) float Bs[GK * GLD];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int dir = blockIdx.z, chunk = blockIdx.x;
    const int ntiles = (N + GT - 1) / GT;
    const int m0 = (blockIdx.y / ntiles) * GT, n0 = (blockIdx.y % ntiles) * GT;
    const int64_t BT = B * (int64_t)T;
    const float* G = gates + (int64_t)dir * BT * (4 * H);
    const int xoff = dir ? xoff_b : 0;
    const int sh = dir ? shift : -shift;
    // a chunk is whole sequences, so (b, t) of a row is tracked incrementally (no 64-bit division)
    int64_t b_base = (int64_t)chunk * seqs_per_chunk;
    int t_base = 0;
    const int64_t r_begin = b_base * T;
    const int64_t r_end = r_begin + seqs_per_chunk * T < BT ? r_begin + seqs_per_chunk * T : BT;
    const bool want_db = dbpart && n0 == 0;
    float acc[4][4] = {}, dbacc[4] = {};
    for (int64_t r0 = r_begin; r0 < r_end; r0 += GK) {
        __syncthreads();
        for (int i = tid; i < GK * (GT / 4); i += 256) {
            const int k = i / (GT / 4), c4 = i % (GT / 4);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r0 + k < r_end) v = ldg4(G + (r0 + k) * (4 * H) + m0 + 4 * c4);
            *reinterpret_cast<float4*>(As + k * GLD + 4 * c4) = v;
        }
        for (int i = tid; i < GK * GT; i += 256) {
            const int k = i / GT, n = i % GT;
            float v = 0.f;
            const int64_t r = r0 + k;
            if (r < r_end && n0 + n < N) {
                const int q = (t_base + k) / T;
                const int64_t b = b_base + q;
                const int ts = t_base + k - q * T + sh;
                if (ts >= 0 && ts < clamp_len(__ldg(len + b), T)) v = __ldg(x + (b * T + ts) * ldx + xoff + n0 + n);
            }
            Bs[k * GLD + n] = v;
        }
        t_base += GK;
        const int q = t_base / T;
        b_base += q; t_base -= q * T;
        __syncthreads();
        tile_acc(As, Bs, tx, ty, acc);
        if (want_db && tx == 0) {
#pragma unroll 4
            for (int k = 0; k < GK; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(As + k * GLD + 4 * ty);
                dbacc[0] += a.x; dbacc[1] += a.y; dbacc[2] += a.z; dbacc[3] += a.w;
            }
        }
    }
    float* out = part + ((size_t)dir * chunks + chunk) * (size_t)(4 * H) * N;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (n0 + 4 * tx + c < N) out[(size_t)(m0 + 4 * ty + a) * N + n0 + 4 * tx + c] = acc[a][c];
    if (want_db && tx == 0) {
#pragma unroll
        for (int a = 0; a < 4; ++a) dbpart[((size_t)dir * chunks + chunk) * (4 * H) + m0 + 4 * ty + a] = dbacc[a];
    }
}

// out_dir[i] = sum_c part[dir][c][i], c ascending (deterministic)
__global__ void __launch_bounds__(256) lstm_bwd_reduce_kernel(const float* __restrict__ part, float* __restrict__ out_f,
                                                              float* __restrict__ out_b, int elems, int chunks) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    const int dir = blockIdx.y;
    if (i >= elems) return;
    const float* p = part + (size_t)dir * chunks * elems;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += p[(size_t)c * elems + i];
    (dir ? out_b : out_f)[i] = s;
}

// din[r][n] = sum_{k < 4H} dg_f[r][k] W_f[k][n] + sum_{k < 4H} dg_b[r][k] W_b[k][n]   (W torch layout [4H, N])
__global__ void __launch_bounds__(256)
lstm_bwd_din_kernel(const float* __restrict__ gates, const float* __restrict__ W_f, const float* __restrict__ W_b,
                    float* __restrict__ din, int ldo, int N, int64_t BT) {
    __shared__ __align__(16) float As[GK * GLD];       // As[k][r] = dg[r0 + r][k0 + k]
    __shared__ __align__(16) float Bs[GK * GLD];       // Bs[k][n] = W[k0 + k][n0 + n]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t r0 = (int64_t)blockIdx.x * GT;
    const int n0 = blockIdx.y * GT;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < 8 * H; k0 += GK) {
        const int dir = k0 >= 4 * H;
        const int kk0 = k0 - dir * 4 * H;
        const float* G = gates + (int64_t)dir * BT * (4 * H);
        const float* W = dir ? W_b : W_f;
        __syncthreads();
        for (int i = tid; i < GT * GK; i += 256) {
            const int r = i / GK, k = i % GK;                  // coalesced along k
            As[k * GLD + r] = (r0 + r < BT) ? __ldg(G + (r0 + r) * (4 * H) + kk0 + k) : 0.f;
        }
        for (int i = tid; i < GK * GT; i += 256) {
            const int k = i / GT, n = i % GT;
            Bs[k * GLD + n] = (n0 + n < N) ? __ldg(W + (size_t)(kk0 + k) * N + n0 + n) : 0.f;
        }
        __syncthreads();
        tile_acc(As, Bs, tx, ty, acc);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int64_t r = r0 + 4 * ty + a;
        if (r >= BT) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (n0 + 4 * tx + c < N) din[r * ldo + n0 + 4 * tx + c] = acc[a][c];
    }
}

struct BwdPlan {
    int64_t seqs_per_chunk;
    int chunks;
    int nmax;                    // widest weight-gradient slab: max(D_in, H, 2H if a second layer exists)
    size_t dout_bytes, part_bytes, dbpart_bytes;
};
BwdPlan bwd_plan(int64_t B, int T, int D_in, int num_layers) {
    BwdPlan p;
    const int64_t bt = B * (int64_t)T;
    const int64_t c = B < MAX_CHUNKS ? (B > 0 ? B : 1) : MAX_CHUNKS;
    p.seqs_per_chunk = (B + c - 1) / c;
    if (p.seqs_per_chunk < 1) p.seqs_per_chunk = 1;
    p.chunks = (int)((B + p.seqs_per_chunk - 1) / p.seqs_per_chunk);
    if (p.chunks < 1) p.chunks = 1;
    p.nmax = D_in > H ? D_in : H;
    if (num_layers > 1 && p.nmax < 2 * H) p.nmax = 2 * H;
    p.dout_bytes = (((size_t)bt * 2 * H * 4) + 255) & ~(size_t)255;
    p.part_bytes = (((size_t)2 * p.chunks * 4 * H * p.nmax * 4) + 255) & ~(size_t)255;
    p.dbpart_bytes = (size_t)2 * p.chunks * 4 * H * 4;
    return p;
}

// one weight gradient (both directions): dW[dir] [4H, N] (+ db[dir] [4H])
int weight_grad(const float* gates, const float* x, int ldx, int xoff_b, int N, int shift, const int32_t* len, int64_t B,
                int T, const BwdPlan& p, float* part, float* dbpart, float* dW_f, float* dW_b, float* db_f, float* db_b,
                cudaStream_t st) {
    const int tiles = (4 * H / GT) * ((N + GT - 1) / GT);
    lstm_bwd_dw_kernel<<<dim3((unsigned)p.chunks, tiles, 2), 256, 0, st>>>(gates, x, ldx, xoff_b, N, len, B, T, p.seqs_per_chunk,
                                                                           p.chunks, part, db_f ? dbpart : nullptr, shift);
    const int elems = 4 * H * N;
    lstm_bwd_reduce_kernel<<<dim3((elems + 255) / 256, 2), 256, 0, st>>>(part, dW_f, dW_b, elems, p.chunks);
    if (db_f) lstm_bwd_reduce_kernel<<<dim3(4 * H / 256, 2), 256, 0, st>>>(dbpart, db_f, db_b, 4 * H, p.chunks);
    return launch_status("lstm weight gradient");
}

// The backward proper, layer by layer, top layer first.  weights = false is the input-gradient mode (explanations): the
// same recurrence and din launches in the same order, without the weight-gradient calls, so dseq is the same bits; the
// workspace is then the dout buffer alone.  Arguments are checked by the callers.
int backward(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int num_layers, const float* const* W_ih,
             const float* const* W_hh, void* tape, const float* dhfin, float* dseq, float* const* dW_ih, float* const* dW_hh,
             float* const* db, void* workspace, bool weights, cudaStream_t st) {
    const LstmTape tp(B, T);
    const BwdPlan p = bwd_plan(B, T, D_in, num_layers);
    float* dout = (float*)workspace;
    float* part = weights ? (float*)((char*)workspace + p.dout_bytes) : nullptr;
    float* dbpart = weights ? (float*)((char*)part + p.part_bytes) : nullptr;
    float* tf = (float*)tape;
    const int64_t BT = B * (int64_t)T;
    int rc = set_max_dynamic_smem((const void*)lstm_bwd_rec_kernel, REC_SMEM);
    if (rc) return rc;
    for (int l = num_layers - 1; l >= 0; --l) {
        float* gates = tp.gates(tf, l);
        const float* out_l = tp.out(tf, l);
        const float* in_l = l ? tp.out(tf, l - 1) : seq;
        const int D = l ? 2 * H : D_in;
        const bool top = l == num_layers - 1;
        lstm_bwd_rec_kernel<<<dim3((unsigned)((B + BS - 1) / BS), 2), H, REC_SMEM, st>>>(
            len, B, T, W_hh[2 * l], W_hh[2 * l + 1], gates, tp.cell(tf, l), top ? nullptr : dout, top ? dhfin : nullptr);
        rc = launch_status("lstm_bwd_rec_kernel");
        if (rc) return rc;
        if (weights) {
            rc = weight_grad(gates, in_l, D, 0, D, 0, len, B, T, p, part, dbpart, dW_ih[2 * l], dW_ih[2 * l + 1], db[2 * l],
                             db[2 * l + 1], st);
            if (rc) return rc;
            // h_prev: out_l one step earlier in each direction's order (forward half t-1, backward half t+1), zero at the start
            rc = weight_grad(gates, out_l, 2 * H, H, H, 1, len, B, T, p, part, dbpart, dW_hh[2 * l], dW_hh[2 * l + 1], nullptr,
                             nullptr, st);
            if (rc) return rc;
        }
        if (l > 0 || dseq) {
            float* din = l ? dout : dseq;          // the recurrence of layer l has consumed dout: overwrite it
            lstm_bwd_din_kernel<<<dim3((unsigned)((BT + GT - 1) / GT), (D + GT - 1) / GT), 256, 0, st>>>(
                gates, W_ih[2 * l], W_ih[2 * l + 1], din, D, D, BT);
            rc = launch_status("lstm_bwd_din_kernel");
            if (rc) return rc;
        }
    }
    return NERRF_OK;
}

}  // namespace
}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_lstm_train_workspace_bytes(int64_t B, int T, int D_in, int H_, int num_layers, size_t* tape_bytes,
                                                size_t* workspace_bytes) {
    NERRF_REQUIRE(tape_bytes && workspace_bytes, "null out");
    NERRF_REQUIRE(B >= 0 && T >= 1 && H_ == H, "LSTM training: need B >= 0, T >= 1, H == 256 (got H = %d)", H_);
    NERRF_REQUIRE(num_layers >= 1 && num_layers <= 8, "num_layers out of range");
    NERRF_REQUIRE(D_in >= 1 && D_in <= 1024, "D_in out of range");
    const BwdPlan p = bwd_plan(B, T, D_in, num_layers);
    *tape_bytes = LstmTape(B, T).bytes(num_layers);
    *workspace_bytes = p.dout_bytes + p.part_bytes + p.dbpart_bytes;
    return NERRF_OK;
}

extern "C" int nerrf_lstm_backward(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H_, int num_layers,
                                   const float* const* W_ih, const float* const* W_hh, void* tape, size_t tape_bytes,
                                   const float* dhfin, float* dseq, float* const* dW_ih, float* const* dW_hh,
                                   float* const* db, void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    size_t need_tape = 0, need_ws = 0;
    int rc = nerrf_lstm_train_workspace_bytes(B, T, D_in, H_, num_layers, &need_tape, &need_ws);
    if (rc) return rc;
    NERRF_REQUIRE(seq && len && W_ih && W_hh && tape && dhfin && dW_ih && dW_hh && db && workspace, "null pointer");
    NERRF_REQUIRE(((uintptr_t)tape & 15) == 0 && ((uintptr_t)workspace & 15) == 0, "tape and workspace must be 16-byte aligned");
    if (tape_bytes < need_tape) {
        set_error("lstm tape too small: need %zu bytes, got %zu", need_tape, tape_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    if (workspace_bytes < need_ws) {
        set_error("lstm backward workspace too small: need %zu bytes, got %zu", need_ws, workspace_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    for (int i = 0; i < 2 * num_layers; ++i)
        NERRF_REQUIRE(W_ih[i] && W_hh[i] && dW_ih[i] && dW_hh[i] && db[i], "null weight or gradient pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (B == 0) {
        for (int l = 0; l < num_layers; ++l) {
            const int D = l ? 2 * H : D_in;
            for (int d = 0; d < 2; ++d) {
                NERRF_CHECK_CUDA(cudaMemsetAsync(dW_ih[2 * l + d], 0, (size_t)4 * H * D * 4, st));
                NERRF_CHECK_CUDA(cudaMemsetAsync(dW_hh[2 * l + d], 0, (size_t)4 * H * H * 4, st));
                NERRF_CHECK_CUDA(cudaMemsetAsync(db[2 * l + d], 0, (size_t)4 * H * 4, st));
            }
        }
        return NERRF_OK;
    }
    return backward(seq, len, B, T, D_in, num_layers, W_ih, W_hh, tape, dhfin, dseq, dW_ih, dW_hh, db, workspace, true, st);
}

extern "C" int nerrf_lstm_input_grad_workspace_bytes(int64_t B, int T, int D_in, int H_, int num_layers, size_t* bytes) {
    size_t need_tape = 0, need_ws = 0;
    NERRF_REQUIRE(bytes, "null out");
    const int rc = nerrf_lstm_train_workspace_bytes(B, T, D_in, H_, num_layers, &need_tape, &need_ws);
    if (rc) return rc;
    *bytes = bwd_plan(B, T, D_in, num_layers).dout_bytes;
    return NERRF_OK;
}

extern "C" int nerrf_lstm_input_grad(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H_, int num_layers,
                                     const float* const* W_ih, const float* const* W_hh, void* tape, size_t tape_bytes,
                                     const float* dhfin, float* dseq, void* workspace, size_t workspace_bytes,
                                     nerrf_stream_t stream) {
    size_t need_tape = 0, need_ws = 0, need = 0;
    int rc = nerrf_lstm_train_workspace_bytes(B, T, D_in, H_, num_layers, &need_tape, &need_ws);
    if (rc) return rc;
    rc = nerrf_lstm_input_grad_workspace_bytes(B, T, D_in, H_, num_layers, &need);
    if (rc) return rc;
    if (B == 0) return NERRF_OK;
    NERRF_REQUIRE(seq && len && W_ih && W_hh && tape && dhfin && dseq && workspace, "null pointer");
    NERRF_REQUIRE(((uintptr_t)tape & 15) == 0 && ((uintptr_t)workspace & 15) == 0, "tape and workspace must be 16-byte aligned");
    if (tape_bytes < need_tape) {
        set_error("lstm tape too small: need %zu bytes, got %zu", need_tape, tape_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    if (workspace_bytes < need) {
        set_error("lstm input-gradient workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    for (int i = 0; i < 2 * num_layers; ++i) NERRF_REQUIRE(W_ih[i] && W_hh[i], "null weight pointer");
    return backward(seq, len, B, T, D_in, num_layers, W_ih, W_hh, tape, dhfin, dseq, nullptr, nullptr, nullptr, workspace, false,
                    (cudaStream_t)stream);
}
