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

// One stream's share of a launch: windows w0 .. w0 + nb - 1 of the launch's concatenated windows (nb >= 1, slices in window
// order).  Its PCM sits at pcm + pcm0: the 64 samples before its first window, then its nb windows.
struct VadSlice {
  int64_t pcm0;
  int32_t w0, nb;
  int32_t stream;  // row of the per-stream LSTM state (h [128] then c [128]) carried between launches
  int32_t first;   // the slice starts the stream: zero context, zero h and c
  int32_t last;    // the slice ends the stream: the last window's final 64 samples count as zero
  int32_t pad_;
};

void vad_configure();  // per-device kernel attributes
// Gx[n][512] = W_ih x_n + b for the nb windows of a launch (device table `slices`, n_slices entries).
void vad_windows(const VadWeights& w, const float* pcm, const VadSlice* slices, int n_slices, int nb, float* gx, cudaStream_t s);
// The LSTM over every slice in one launch, one 4-CTA cluster per slice, from and back to its stream's state
// states[stream][256]; H[n][128] receives every window's h.
void vad_recurrence(const float* w_hh, const VadSlice* slices, int n_slices, const float* gx, float* states, float* H,
                    cudaStream_t s);
// probs[n] = sigmoid(w . relu(H[n]) + b[0])
void vad_decoder(const float* H, const float* w, const float* b, int nb, float* probs, cudaStream_t s);

}  // namespace b2w
