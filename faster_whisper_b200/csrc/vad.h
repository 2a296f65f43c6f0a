// Silero VAD kernels (vad.cu) as the engine's C ABI drives them.
#pragma once
#include "common.cuh"

namespace b2w {

// Device copies of the network's weights, laid out for coalesced reads across output channels.
struct VadWeights {
  const float* basis_t = nullptr;  // [256][258]: STFT basis transposed (columns 0..128 real, 129..257 imaginary)
  const float* conv_t[4] = {};     // [cin * 3 + k][cout]
  const float* conv_b[4] = {};     // [cout]
  const float* w_ih_t = nullptr;   // [128][512]: LSTM input weights transposed, gate blocks i, o, f, c
  const float* b_gates = nullptr;  // [512]: b_ih + b_hh
};

void vad_configure();  // per-device kernel attributes
// Gx[n][512] = W_ih x_n + b for the nb windows of a block.  pcm: 64 + 512 nb samples, the 64 before the block's first window
// (zeros at the start of the audio) followed by the block; last_is_tail: the block's last window is the audio's last window.
void vad_windows(const VadWeights& w, const float* pcm, int nb, bool last_is_tail, float* gx, cudaStream_t s);
// The LSTM over nb steps in one launch, from and back to state_h / state_c [128]; H[n][128] receives every step's h.
void vad_recurrence(const float* w_hh, const float* gx, int nb, float* state_h, float* state_c, float* H, cudaStream_t s);
// probs[n] = sigmoid(w . relu(H[n]) + b[0])
void vad_decoder(const float* H, const float* w, const float* b, int nb, float* probs, cudaStream_t s);

}  // namespace b2w
