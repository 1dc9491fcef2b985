// lstm.forward (SURVEY.md 8a row a4): BiLSTM(H=256, 2 layers) over per-file event sequences.
//
// v0 kernel: one CTA = BS sequences x one direction of one layer, resident for all T steps.
// Thread j owns hidden unit j: it accumulates the four gate pre-activations (i,f,g,o rows j,
// H+j, 2H+j, 3H+j) for all BS sequences, then applies the cell update in registers (the whole
// cell -- 4 GEMV rows, sigmoid/tanh, c/h update -- is one fused pass; c never leaves
// registers, h lives in shared memory).  Weights are pre-transposed ([K, 4H]) so the 256
// threads read 1 KB contiguous per (k, gate); they stream from L2 every step (8.2 MB of
// weights is L2-resident, too big for one SM's shared memory).
//
// SAVE = true is the training forward (nerrf_lstm_forward_train): the same arithmetic, and at every valid step it also
// stores the post-activation gates and the cell state into the tape that csrc/lstm_bwd.cu differentiates.  `out` is then
// a layer of that tape (lstm_tape.cuh), whose gates and cells follow the output at fixed offsets, so the kernel keeps
// one signature and the inference instantiation (SAVE = false) compiles exactly as it did before the flag existed.
#include "common.cuh"
#include "lstm_tape.cuh"

namespace nerrf {

// tensor-core path (lstm_umma.cu), selected with NERRF_LSTM_ALGO=umma
bool lstm_umma_enabled();
size_t lstm_umma_workspace_bytes(int64_t B, int T, int num_layers);
int lstm_layers_umma(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int num_layers, const float* const* Wih_t,
                     const float* const* Whh_t, const float* const* bias, float* hfin, void* workspace, size_t workspace_bytes,
                     cudaStream_t st);

constexpr int LH = 256;       // hidden size (threads per CTA)

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

template <int BS, bool SAVE>
__global__ void __launch_bounds__(LH, 1)
lstm_layer_kernel(const float* __restrict__ in, int in_stride_b, int in_stride_t, int D,   // in[b*in_stride_b + t*in_stride_t + k]
                  const int32_t* __restrict__ len, int64_t B, int T,
                  const float* __restrict__ Wih_f, const float* __restrict__ Whh_f, const float* __restrict__ bias_f,
                  const float* __restrict__ Wih_b, const float* __restrict__ Whh_b, const float* __restrict__ bias_b,
                  float* __restrict__ out,       // [B, T, 2H] or nullptr
                  float* __restrict__ hfin)      // [B, 2H]
{
    extern __shared__ __align__(16) float sm[];
    float* h_s = sm;                       // [2][LH][BS]
    float* x_s = sm + 2 * LH * BS;         // [D][BS]
    __shared__ int len_s[BS];

    const int j = threadIdx.x;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * BS;
    const float* Wih = dir ? Wih_b : Wih_f;
    const float* Whh = dir ? Whh_b : Whh_f;
    const float* bias = dir ? bias_b : bias_f;

    if (j < BS) len_s[j] = (b0 + j < B) ? len[b0 + j] : 0;
    for (int i = j; i < 2 * LH * BS; i += LH) h_s[i] = 0.f;
    float c[BS];
#pragma unroll
    for (int b = 0; b < BS; ++b) c[b] = 0.f;
    const float bi = bias[j], bf = bias[LH + j], bg = bias[2 * LH + j], bo = bias[3 * LH + j];
    __syncthreads();

    int cur = 0;
    for (int step = 0; step < T; ++step) {
        const int t = dir ? (T - 1 - step) : step;
        // stage x_t for the BS sequences: x_s[k][b]
        for (int i = j; i < D * BS; i += LH) {
            const int b = i / D, k = i % D;
            float v = 0.f;
            if (b0 + b < B && t < len_s[b]) v = in[(b0 + b) * (int64_t)in_stride_b + (int64_t)t * in_stride_t + k];
            x_s[k * BS + b] = v;
        }
        __syncthreads();
        float ai[BS], af[BS], ag[BS], ao[BS];
#pragma unroll
        for (int b = 0; b < BS; ++b) { ai[b] = bi; af[b] = bf; ag[b] = bg; ao[b] = bo; }
        // input projection
#pragma unroll 8
        for (int k = 0; k < D; ++k) {
            const float* wr = Wih + (size_t)k * 4 * LH + j;
            const float w0 = __ldg(wr), w1 = __ldg(wr + LH), w2 = __ldg(wr + 2 * LH), w3 = __ldg(wr + 3 * LH);
            const float4* xv = reinterpret_cast<const float4*>(x_s + k * BS);
#pragma unroll
            for (int q = 0; q < BS / 4; ++q) {
                const float4 v = xv[q];
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    ai[q * 4 + e] = fmaf(w0, vv[e], ai[q * 4 + e]); af[q * 4 + e] = fmaf(w1, vv[e], af[q * 4 + e]);
                    ag[q * 4 + e] = fmaf(w2, vv[e], ag[q * 4 + e]); ao[q * 4 + e] = fmaf(w3, vv[e], ao[q * 4 + e]);
                }
            }
        }
        // recurrent projection
        const float* hc = h_s + cur * LH * BS;
#pragma unroll 8
        for (int k = 0; k < LH; ++k) {
            const float* wr = Whh + (size_t)k * 4 * LH + j;
            const float w0 = __ldg(wr), w1 = __ldg(wr + LH), w2 = __ldg(wr + 2 * LH), w3 = __ldg(wr + 3 * LH);
            const float4* hv = reinterpret_cast<const float4*>(hc + k * BS);
#pragma unroll
            for (int q = 0; q < BS / 4; ++q) {
                const float4 v = hv[q];
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    ai[q * 4 + e] = fmaf(w0, vv[e], ai[q * 4 + e]); af[q * 4 + e] = fmaf(w1, vv[e], af[q * 4 + e]);
                    ag[q * 4 + e] = fmaf(w2, vv[e], ag[q * 4 + e]); ao[q * 4 + e] = fmaf(w3, vv[e], ao[q * 4 + e]);
                }
            }
        }
        // cell update (registers) -> next h buffer
        float* hn = h_s + (cur ^ 1) * LH * BS;
#pragma unroll
        for (int b = 0; b < BS; ++b) {
            const bool valid = t < len_s[b];
            float hval = hc[j * BS + b];
            float oval = 0.f;
            if (valid) {
                const float ig = sigmoidf_(ai[b]), fg = sigmoidf_(af[b]), gg = tanhf(ag[b]), og = sigmoidf_(ao[b]);
                c[b] = fg * c[b] + ig * gg;
                hval = og * tanhf(c[b]);
                oval = hval;
                if constexpr (SAVE) {       // out is a layer of the training tape: its gates and cells follow it
                    const int64_t bt = B * (int64_t)T, row = dir * bt + (b0 + b) * (int64_t)T + t;
                    float* gs = out + bt * (2 * LH) + row * (4 * LH) + j;
                    gs[0] = ig; gs[LH] = fg; gs[2 * LH] = gg; gs[3 * LH] = og;
                    out[bt * (2 * LH + 2 * 4 * LH) + row * LH + j] = c[b];
                }
            }
            hn[j * BS + b] = hval;
            if (out && b0 + b < B) out[((b0 + b) * (int64_t)T + t) * (2 * LH) + dir * LH + j] = oval;
        }
        cur ^= 1;
        __syncthreads();
    }
    const float* hl = h_s + cur * LH * BS;
#pragma unroll
    for (int b = 0; b < BS; ++b)
        if (b0 + b < B) hfin[(b0 + b) * (2 * LH) + dir * LH + j] = hl[j * BS + b];
}

__global__ void __launch_bounds__(256) lstm_head_kernel(const float* __restrict__ hfin, const float* __restrict__ head_W,
                                                        const float* __restrict__ head_b, float* __restrict__ out, int64_t B,
                                                        int K) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= B) return;
    float s0 = 0.f, s1 = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float h = hfin[b * K + k];
        s0 = fmaf(h, __ldg(head_W + k), s0);
        s1 = fmaf(h, __ldg(head_W + K + k), s1);
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1);
    if (lane == 0) {
        out[b * 2 + 0] = sigmoidf_(s0 + __ldg(head_b));
        out[b * 2 + 1] = sigmoidf_(s1 + __ldg(head_b + 1));
    }
}

template <int BS, bool SAVE>
static int launch_lstm_layer(const float* in, int sb, int stt, int D, const int32_t* len, int64_t B, int T,
                             const float* Wih_f, const float* Whh_f, const float* bias_f, const float* Wih_b,
                             const float* Whh_b, const float* bias_b, float* out, float* hfin, cudaStream_t st) {
    const size_t smem = (size_t)(2 * LH * BS + (size_t)D * BS) * sizeof(float);
    NERRF_REQUIRE(smem <= 200 * 1024, "LSTM input width %d too large for shared memory", D);
    const int rc = set_max_dynamic_smem((const void*)lstm_layer_kernel<BS, SAVE>, smem);
    if (rc) return rc;
    dim3 grid((unsigned)((B + BS - 1) / BS), 2);
    lstm_layer_kernel<BS, SAVE><<<grid, LH, smem, st>>>(in, sb, stt, D, len, B, T, Wih_f, Whh_f, bias_f, Wih_b, Whh_b, bias_b,
                                                        out, hfin);
    return launch_status("lstm_layer_kernel");
}

}  // namespace nerrf

using namespace nerrf;

extern "C" int nerrf_lstm_workspace_bytes(int64_t B, int T, int H, size_t* bytes) {
    NERRF_REQUIRE(bytes, "null out");
    NERRF_REQUIRE(B >= 0 && T >= 1 && H == LH, "LSTM: need B >= 0, T >= 1, H == 256");
    *bytes = ((size_t)2 * B * T * 2 * H + (size_t)B * 2 * H) * sizeof(float) + 256;
    if (lstm_umma_enabled() && B > 0) *bytes = lstm_umma_workspace_bytes(B, T, 2) + (size_t)B * 2 * H * sizeof(float) + 512;
    return NERRF_OK;
}

extern "C" int nerrf_lstm_forward(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H, int num_layers,
                                  const float* const* Wih_t, const float* const* Whh_t, const float* const* bias,
                                  const float* head_W, const float* head_b, float* out, void* workspace,
                                  size_t workspace_bytes, nerrf_stream_t stream) {
    size_t need = 0;
    int rc = nerrf_lstm_workspace_bytes(B, T, H, &need);
    if (rc) return rc;
    NERRF_REQUIRE(seq && len && Wih_t && Whh_t && bias && head_W && head_b && out && workspace, "null pointer");
    NERRF_REQUIRE(num_layers >= 1 && num_layers <= 8, "num_layers out of range");
    NERRF_REQUIRE(D_in >= 1 && D_in <= 1024, "D_in out of range");
    if (workspace_bytes < need) {
        set_error("lstm workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    if (B == 0) return NERRF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (lstm_umma_enabled()) {
        // workspace = [hfin | tensor-core scratch]
        float* hf = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
        char* scratch = (char*)hf + (((size_t)B * 2 * H * sizeof(float) + 255) & ~(size_t)255);
        const size_t left = workspace_bytes - (size_t)(scratch - (char*)workspace);
        rc = lstm_layers_umma(seq, len, B, T, D_in, num_layers, Wih_t, Whh_t, bias, hf, scratch, left, st);
        if (rc) return rc;
        lstm_head_kernel<<<(unsigned)((B + 7) / 8), 256, 0, st>>>(hf, head_W, head_b, out, B, 2 * H);
        return launch_status("lstm_head_kernel");
    }
    float* buf0 = (float*)workspace;
    float* buf1 = buf0 + (size_t)B * T * 2 * H;
    float* hfin = buf1 + (size_t)B * T * 2 * H;
    const float* in = seq;
    int sb = T * D_in, stt = D_in, D = D_in;
    for (int l = 0; l < num_layers; ++l) {
        float* o = (l == num_layers - 1) ? nullptr : ((l & 1) ? buf1 : buf0);
        rc = launch_lstm_layer<8, false>(in, sb, stt, D, len, B, T, Wih_t[2 * l], Whh_t[2 * l], bias[2 * l], Wih_t[2 * l + 1],
                                         Whh_t[2 * l + 1], bias[2 * l + 1], o, hfin, st);
        if (rc) return rc;
        in = o; sb = T * 2 * H; stt = 2 * H; D = 2 * H;
    }
    lstm_head_kernel<<<(unsigned)((B + 7) / 8), 256, 0, st>>>(hfin, head_W, head_b, out, B, 2 * H);
    return launch_status("lstm_head_kernel");
}

extern "C" int nerrf_lstm_forward_train(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H,
                                        int num_layers, const float* const* Wih_t, const float* const* Whh_t,
                                        const float* const* bias, float* hfin_out, void* tape, size_t tape_bytes,
                                        nerrf_stream_t stream) {
    size_t need = 0, ws = 0;
    int rc = nerrf_lstm_train_workspace_bytes(B, T, D_in, H, num_layers, &need, &ws);
    if (rc) return rc;
    NERRF_REQUIRE(seq && len && Wih_t && Whh_t && bias && hfin_out && tape, "null pointer");
    NERRF_REQUIRE(((uintptr_t)tape & 15) == 0, "tape must be 16-byte aligned");
    if (tape_bytes < need) {
        set_error("lstm tape too small: need %zu bytes, got %zu", need, tape_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    for (int i = 0; i < 2 * num_layers; ++i) NERRF_REQUIRE(Wih_t[i] && Whh_t[i] && bias[i], "null weight pointer");
    if (B == 0) return NERRF_OK;
    const LstmTape tp(B, T);
    const float* in = seq;
    int sb = T * D_in, stt = D_in, D = D_in;
    for (int l = 0; l < num_layers; ++l) {
        float* o = tp.out((float*)tape, l);
        rc = launch_lstm_layer<8, true>(in, sb, stt, D, len, B, T, Wih_t[2 * l], Whh_t[2 * l], bias[2 * l], Wih_t[2 * l + 1],
                                        Whh_t[2 * l + 1], bias[2 * l + 1], o, hfin_out, (cudaStream_t)stream);
        if (rc) return rc;
        in = o; sb = T * 2 * H; stt = 2 * H; D = 2 * H;
    }
    return NERRF_OK;
}
