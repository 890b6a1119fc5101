// dft_internal.h -- entry points of dft.cu used by other translation units of libb2a.
#pragma once
#include "b2a_common.h"

namespace b2a {
namespace dft {

// Overlap-add + window-envelope division of windowed frames [rows, n_frames, n_fft] (fold_kernel): out[row][i] =
// y[start + i] / env[start + i] for start + i < (n_frames + 2 pad_frames - 1) hop + n_fft, else 0.  divide = 0 skips the
// envelope division (the STFT's adjoint).  Enqueues one launch.
int launch_fold(const float* frames, const float* window, int64_t rows, int n_frames, int n_fft, int hop, int pad_frames,
                int64_t start, int64_t out_len, int divide, float* out, void* stream);

}  // namespace dft
}  // namespace b2a
