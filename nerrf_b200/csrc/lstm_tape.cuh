// Layout of the BiLSTM training tape: what nerrf_lstm_forward_train saves and nerrf_lstm_backward reads (H = 256).
// Per layer l, one after another:
//     out   [B, T, 2H]      the layer's output, zero at padded steps (the top layer's too)
//     gates [2][B, T, 4H]   per direction, i, f, g, o after activation at valid steps; the backward overwrites them
//                           with the gate pre-activation gradients (zero at padded steps)
//     cell  [2][B, T, H]    per direction, the cell state c_t at valid steps
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace nerrf {

struct LstmTape {
    static constexpr int H = 256;
    int64_t bt;
    LstmTape(int64_t B, int T) : bt(B * (int64_t)T) {}
    size_t out_floats() const { return (size_t)bt * 2 * H; }
    size_t gate_floats() const { return (size_t)2 * bt * 4 * H; }
    size_t cell_floats() const { return (size_t)2 * bt * H; }
    size_t layer_floats() const { return out_floats() + gate_floats() + cell_floats(); }
    size_t bytes(int num_layers) const { return (size_t)num_layers * layer_floats() * sizeof(float); }
    float* out(float* tape, int l) const { return tape + (size_t)l * layer_floats(); }
    float* gates(float* tape, int l) const { return out(tape, l) + out_floats(); }
    float* cell(float* tape, int l) const { return gates(tape, l) + gate_floats(); }
};

}  // namespace nerrf
