// truepeak_internal.h -- the 12-tap polyphase interpolator of the true-peak meter (truepeak.cu, K17 in DESIGN.md),
// shared with the limiter's envelope (limiter.cu, K18), whose definition is "K17's factor, taps and instants":
//
//   phase p >= 1     y[n, p] = sum_{d=-6..5} h_p[d] x[n - d]
//                    h_p[d] = float(sinc(u) * (1 + cos(pi u / 6)) / 2),  u = d + p / L  (designed in double here)
//
// A CTA stages its chunk plus a halo in shared memory; each thread copies RUN consecutive samples and their halo into
// registers (stage_run) and evaluates the phases at the instants it owns (phase).
#pragma once
#include "b2a_common.h"

namespace b2a {
namespace truepeak {

constexpr int TPB = 256;             // threads per CTA
constexpr int RUN = 16;              // consecutive instants n per thread
constexpr int CHUNK = TPB * RUN;     // samples of a row per CTA work item (tests cover T = CHUNK +- 1)
constexpr int HALO = 8;              // taps reach 6 samples ahead and 5 behind; 8 keeps the float4 reads aligned
constexpr int NTAP = 12;

struct Taps {
  float h[3][NTAP];  // phase p (1 .. L-1) at h[p - 1], tap d (-6 .. 5) at [d + 6]
};

// Taps of factor L (1, 2 or 4), designed in double and rounded to float; B2A_E_INVALID for any other L.
inline int design(int L, Taps* t) {
  B2A_REQUIRE(L == 1 || L == 2 || L == 4, B2A_E_INVALID, "true_peak: factor must be 1, 2 or 4, got %d", L);
  memset(t, 0, sizeof(*t));
  for (int p = 1; p < L; ++p)
    for (int d = -6; d <= 5; ++d) {
      const double u = d + (double)p / L, a = M_PI * u;  // |u| < 6 and u != 0
      t->h[p - 1][d + 6] = (float)(sin(a) / a * 0.5 * (1.0 + cos(a / 6.0)));
    }
  return B2A_OK;
}

// v[j] = s[j] for the RUN + 2 HALO staged samples of a run; s is 16-byte aligned shared memory.
__device__ __forceinline__ void stage_run(const float* s, float (&v)[RUN + 2 * HALO]) {
  const float4* s4 = reinterpret_cast<const float4*>(s);
#pragma unroll
  for (int j = 0; j < (RUN + 2 * HALO) / 4; ++j) {
    const float4 q = s4[j];
    v[4 * j] = q.x, v[4 * j + 1] = q.y, v[4 * j + 2] = q.z, v[4 * j + 3] = q.w;
  }
}

// y[n0 + k, p + 1] with v[k + HALO] = x[n0 + k]: the taps in a fixed FMA order, so every caller gets the same bits.
__device__ __forceinline__ float phase(const Taps& taps, int p, const float (&v)[RUN + 2 * HALO], int k) {
  float y = taps.h[p][0] * v[k + HALO + 6];
#pragma unroll
  for (int d = -5; d <= 5; ++d) y = fmaf(taps.h[p][d + 6], v[k + HALO - d], y);
  return y;
}

}  // namespace truepeak
}  // namespace b2a
