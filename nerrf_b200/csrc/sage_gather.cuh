// K1 inner loop: weighted-mean gather of one CSR row by one warp (SURVEY.md 8a row a2).  Used by the fp32
// cross-check layer, the standalone aggregate and the hub-row chunk pre-pass; the tensor-core (wgmma) layer has its own
// cp.async ring pipeline (sage_umma.cu).
//
// A source row is F floats = F/4 float4.  LPR = F/4 lanes cover one source row with one 16-byte
// load each, so a warp fetches G = 32/LPR source rows per load instruction (F=128: 1 row of
// 512 B; F=32: 4 rows of 128 B) and keeps U load instructions in flight before it consumes
// them (memory-level parallelism: U*G rows, U*512 B per warp).  col/ew are read 32 at a time
// (coalesced) and broadcast by shuffle.  The G partial sums are combined by xor-shuffles, so
// every lane < LPR ends with the complete mean for its 4 columns.
#pragma once
#include "common.cuh"

namespace nerrf {

// 2*UH load instructions (2*UH*G source rows) are issued BEFORE anything is consumed.  Weights are
// re-broadcast at consume time instead of being held in registers.
// wsum_out != nullptr: return the UNNORMALISED weighted sum and store the weight sum (used for chunk partials).
// STRIDE: floats between consecutive source rows (F for a dense [n, F] matrix; the backward pass gathers the right half of
// dZ [n, 2F] with STRIDE = 2F).
template <int F, int UH = 0, int STRIDE = F>
__device__ __forceinline__ float4 gather_row(const float* __restrict__ x, const int32_t* __restrict__ col,
                                              const float* __restrict__ ew, int64_t e0, int64_t e1, int lane,
                                              float* wsum_out = nullptr) {
    constexpr int LPR = F / 4;        // lanes per source row
    constexpr int G = 32 / LPR;       // source rows per load instruction
    constexpr int U = UH > 0 ? UH : ((G == 1) ? 4 : 2);   // load instructions per half batch
    static_assert(F == 32 || F == 64 || F == 128, "F must be 32, 64 or 128");
    const int g = lane / LPR, sub = lane % LPR;
    const float* xs = x + 4 * sub;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float wpart = 0.f;
    for (int64_t base = e0; base < e1; base += 32) {
        const int n = (int)((e1 - base) < 32 ? (e1 - base) : 32);
        int my_c = 0;
        float my_w = 0.f;
        if (lane < n) {
            my_c = __ldg(col + base + lane);
            my_w = __ldg(ew + base + lane);
        }
        wpart += my_w;
        for (int j = 0; j < n; j += 2 * G * U) {
            float4 v[2 * U];
#pragma unroll
            for (int u = 0; u < 2 * U; ++u) {
                const int idx = j + u * G + g;
                const int c = __shfl_sync(0xffffffffu, my_c, idx & 31);
                v[u] = (idx < n) ? ldg4(xs + (int64_t)c * STRIDE) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 2 * U; ++u) {
                const int idx = j + u * G + g;
                float w = __shfl_sync(0xffffffffu, my_w, idx & 31);
                w = (idx < n) ? w : 0.f;
                acc.x = fmaf(w, v[u].x, acc.x); acc.y = fmaf(w, v[u].y, acc.y);
                acc.z = fmaf(w, v[u].z, acc.z); acc.w = fmaf(w, v[u].w, acc.w);
            }
        }
    }
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    const float wsum = warp_sum(wpart);
    if (wsum_out) { *wsum_out = wsum; return acc; }          // unnormalised partial (hub-row chunks)
    const float inv = 1.0f / fmaxf(wsum, 1e-12f);
    acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    return acc;
}


}  // namespace nerrf
