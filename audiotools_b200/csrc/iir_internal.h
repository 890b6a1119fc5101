// iir_internal.h -- what csrc/iir.cu lends the loudness backward (csrc/lufs.cu, K21 in DESIGN.md).
#pragma once
#include <cstddef>
#include <cstdint>

namespace b2a {
namespace iir {

// Scratch of loudness_adjoint: the chunk states of the passes and the intermediate u [rows, Tp] float32
size_t loudness_adjoint_workspace_bytes(int64_t rows, int64_t Tp, int S);

// grad_x [B, C, T] = the first T samples of K^T (wt[row] m[e] K x~), where x~ is the row float32(gain[b] x) zero-extended
// to Tp samples, K the cascade `sos` ([S, 6] float32 on the device, a0 = 1), and m[e] the number of blocks
// [i blk_stride, i blk_stride + blk_len), 0 <= i < nblk, that contain sample e and that kept [B, nblk + 1] (a running
// count per item) counts as kept.  Six launches: the two passes of K19, the adjoint one reversed in time.
int loudness_adjoint(const float* x, const float* gain, int64_t B, int C, int64_t T, int64_t Tp, const float* sos,
                     int S, const double* wt, const int* kept, int nblk, int blk_stride, int blk_len, float* grad_x,
                     void* ws, void* stream);

}  // namespace iir
}  // namespace b2a
