// The ranking rule of the explanation top-k kernels (DESIGN.md 1.1.1 edges, 1.2.1 sequence steps): larger |a| first,
// then the lower index; NaN ranks below every number.  Shared by nerrf_explain_topk and nerrf_lstm_explain_steps, so
// the rule exists once.
#pragma once

#include <cstdint>

namespace nerrf {

// key of an attribution: |a|, with NaN mapped below every number (-0.5) and above "no pick" (-1)
__device__ __forceinline__ float rank_key(float a) {
    const float v = fabsf(a);
    return v != v ? -0.5f : v;
}

// (key, index) ordering: does (a, i) rank before (b, j)?
__device__ __forceinline__ bool better(float a, int64_t i, float b, int64_t j) {
    return a > b || (a == b && i < j);
}

}  // namespace nerrf
