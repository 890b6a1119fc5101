// fft_warp.cuh -- register/warp-level FFT building blocks shared by spectral.cu and fftconv.cu.
//
//   DFT<R,S>           radix-R (2..32) DFT of register-resident complex values, natural order out
//   WPlan<LOG2N>       geometry of the warp-per-frame FFT: N = 2^LOG2N complex points, LPF = N/32 lanes
//                      per frame, 32 points per lane, passes = radix 32 then radix LPF
//   warp_fft           the forward N-point transform of a frame held by LPF lanes of one warp
//   warp_fft_tables    its role-constant twiddle tables (shared memory, [slot][lane])
//   load_frame         the windowed frame load in front of warp_fft (spectral.cu, loss.cu)
//   partner_lane       the lane holding Z[N - k] (the real-FFT untangles of spectral.cu, loss.cu, istft.cu)
#pragma once
#include "b2a_common.h"

namespace b2a {
namespace spectral {

// ---------------------------------------------------------------------------------------------
// small DFTs in registers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 rot_mi(float2 a) { return make_float2(a.y, -a.x); }  // a * (-i)

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return add2(a, b); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return add2(a, neg2(b)); }
// a * b = (a.x b.x - a.y b.y, a.x b.y + a.y b.x): the same two roundings per component as the scalar form
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return fma2(bcast2(a.x), b, mul2(bcast2(a.y), make_float2(-b.y, b.x)));
}

// cos(pi*j/16), j = 0..16
__device__ __forceinline__ constexpr float cos_pi16(int j) {
  return j == 0 ? 1.0f
       : j == 1 ? 0.98078528040323043f
       : j == 2 ? 0.92387953251128674f
       : j == 3 ? 0.83146961230254524f
       : j == 4 ? 0.70710678118654752f
       : j == 5 ? 0.55557023301960222f
       : j == 6 ? 0.38268343236508977f
       : j == 7 ? 0.19509032201612827f
       : j == 8 ? 0.0f
                : -cos_pi16(16 - j);
}

// cos(pi*j/32), j = 0..32 (the untangle twiddles exp(-i pi m / 32) of the N = 1024 transform as compile-time constants)
__device__ __forceinline__ constexpr float cos_pi32(int j) {
  return (j & 1) == 0 ? cos_pi16(j / 2)
       : j == 1 ? 0.99518472667219689f
       : j == 3 ? 0.95694033573220887f
       : j == 5 ? 0.88192126434835503f
       : j == 7 ? 0.77301045336273696f
       : j == 9 ? 0.63439328416364549f
       : j == 11 ? 0.47139673682599764f
       : j == 13 ? 0.29028467725446236f
       : j == 15 ? 0.09801714032956060f
                 : -cos_pi32(32 - j);
}

// o * W_R^k, W = exp(-2 pi i / R), 0 <= k < R/2, R in {2,4,8,16,32}
template <int R, int K>
__device__ __forceinline__ float2 mul_wr(float2 o) {
  constexpr int j = 32 * K / R;  // angle = pi*j/16, 0 <= j < 16
  if constexpr (j == 0) {
    return o;
  } else if constexpr (j == 8) {  // -i
    return make_float2(o.y, -o.x);
  } else if constexpr (j == 4) {  // (1 - i)/sqrt2
    constexpr float h = 0.70710678118654752f;
    return make_float2(h * (o.x + o.y), h * (o.y - o.x));
  } else if constexpr (j == 12) {  // (-1 - i)/sqrt2
    constexpr float h = 0.70710678118654752f;
    return make_float2(h * (o.y - o.x), -h * (o.x + o.y));
  } else {
    constexpr float c = cos_pi16(j);
    constexpr float sn = cos_pi16(j <= 8 ? 8 - j : j - 8);  // sin(pi j/16)
    return make_float2(fmaf(o.x, c, o.y * sn), fmaf(o.y, c, -o.x * sn));  // o * (c - i sn)
  }
}

// PRE: the first butterfly stage (pairs in[j], in[j + R S / 2] of the outermost call) was already applied by the
// caller, which could fuse it with the load (spectral.cu folds the window multiply into it).
template <int R, int S, bool PRE = false>
struct DFT {
  // out[K] = e + W o, out[K + R/2] = e - W o with W = exp(-2 pi i K / R) = c - i sn.  For a non-trivial W the sum is
  // formed with fused multiply-adds and the difference as 2e - sum: 6 instructions instead of 8 (complex multiply,
  // add, subtract).  The difference inherits one rounding of the sum (absolute error <= ulp(|e| + |o|), the size
  // of the usual butterfly error).
  template <int K>
  static __device__ __forceinline__ void comb(const float2 (&e)[R / 2], const float2 (&o)[R / 2], float2* out) {
    constexpr int j = 32 * K / R;  // angle = pi*j/16
    if constexpr (R == 2 && PRE) {
      out[K] = e[K];
      out[K + R / 2] = o[K];
    } else if constexpr (j == 0) {
      out[K] = add2(e[K], o[K]);
      out[K + R / 2] = add2(e[K], neg2(o[K]));
    } else if constexpr (j == 8) {  // W = -i
      out[K] = add2(e[K], rot_mi(o[K]));
      out[K + R / 2] = add2(e[K], neg2(rot_mi(o[K])));
    } else if constexpr (j == 4 || j == 12) {
      constexpr float h = 0.70710678118654752f;
      // j == 4: W o = h((o.x + o.y) + i(o.y - o.x));  j == 12: W o = h((o.y - o.x) - i(o.x + o.y))
      const float2 pq = add2(o[K], rot_mi(o[K]));  // (p, q) = (o.x + o.y, o.y - o.x)
      float2 s;
      if constexpr (j == 4) s = fma2(bcast2(h), pq, e[K]);
      else s = fma2(make_float2(h, -h), make_float2(pq.y, pq.x), e[K]);
      out[K] = s;
      out[K + R / 2] = fma2(bcast2(2.0f), e[K], neg2(s));
    } else {
      constexpr float c = cos_pi16(j);
      constexpr float sn = cos_pi16(j <= 8 ? 8 - j : j - 8);  // sin(pi j/16)
      // W o = (o.x c + o.y sn) + i (o.y c - o.x sn)
      const float2 s = fma2(o[K], bcast2(c), fma2(rot_mi(o[K]), bcast2(sn), e[K]));
      out[K] = s;
      out[K + R / 2] = fma2(bcast2(2.0f), e[K], neg2(s));
    }
    if constexpr (K + 1 < R / 2) comb<K + 1>(e, o, out);
  }
  // in: R values at in[0], in[S], ...; out: R values, natural frequency order
  static __device__ __forceinline__ void run(const float2* in, float2* out) {
    float2 e[R / 2], o[R / 2];
    DFT<R / 2, 2 * S, PRE>::run(in, e);
    DFT<R / 2, 2 * S, PRE>::run(in + S, o);
    comb<0>(e, o, out);
  }
};
template <int S, bool PRE>
struct DFT<1, S, PRE> {
  static __device__ __forceinline__ void run(const float2* in, float2* out) { out[0] = in[0]; }
};

template <int LOG2N>
struct WPlan {
  static constexpr int N = 1 << LOG2N;
  static constexpr int LPF = N / 32;   // lanes per frame
  static constexpr int FPW = 32 / LPF; // frames per warp in flight
  static constexpr int R1 = LPF;       // radix of pass 1 (1 => single pass)
  static constexpr int B1 = 32 / R1;   // pass-1 butterflies per lane
  static constexpr int NWARP = 8;
  static constexpr int G = NWARP * FPW;            // frames in flight per CTA
  // frames per tile: 16, except n_fft = 2048 where 8 keeps two CTAs per SM resident (97 KB of shared memory)
  static constexpr int FR = (G >= 16) ? G : (LOG2N == 10 ? 8 : 16);
  // LEAN (N = 1024: R1 = 32, B1 = 1): the 31 pass-1 twiddles W^(l t) of a lane are formed as W^(8a l) . W^(b l) from 10
  // table entries (t = 8a + b: slots 0..6 = W^(l b), b = 1..7; 7..9 = W^(8 l), W^(16 l), W^(24 l)), and the 16 untangle
  // twiddles exp(-i pi (l + 32 m) / N) as exp(-i pi l / N) . exp(-i pi m / 32) from ONE lane entry and compile-time
  // constants: 72 fewer shared-memory wavefronts per frame for 92 more SASS instructions on sm_90a, each twiddle with one
  // more rounding (<= 6e-8 relative).  On the H100 the full tables measured 2 % faster in the fused log-mel kernel, but
  // they move its outputs by up to 2e-6 (log10 units), which the golden gradient tests do not absorb (DESIGN.md K1).
  static constexpr bool LEAN = (LOG2N == 10);
  static constexpr int NTW = LEAN ? 10 : ((R1 >= 2) ? B1 * (R1 - 1) : 0);
  static constexpr int NUT = LEAN ? 1 : 16;  // untangle-twiddle slots per lane
  // floats per frame slot (16 B multiple): the padded exchange plane, later |X| (N+1 values + 3 zeros) plus
  // slack that the zero-weight tail of a padded mel band may read
  static constexpr int XB = ((N + N / 32 + 4 + 3) / 4) * 4 + (N >= 256 ? 128 : 32);
};

__device__ __forceinline__ float fast_sqrt(float v) {
#ifdef B2A_SIM
  return sqrtf(v);
#else
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));  // <= 2 ulp; |X| feeds a 1e-4 tolerance
  return r;
#endif
}

// Forward N-point FFT of the 32 register-resident points of a lane (element e = l + LPF m, natural
// order in and out): radix 32, warp-private transpose through `xb`, radix LPF.
__device__ __forceinline__ float fast_log2(float v) {
#ifdef B2A_SIM
  return log2f(v);
#else
  float r;
  asm("lg2.approx.f32 %0, %1;" : "=f"(r) : "f"(v));  // abs error <= 2^-22: 1.4e-7 in log10 units
  return r;
#endif
}

// PRE0: z[j], z[j + 16] (j < 16) already hold sum and difference of elements j and j + 16 (the first butterfly stage
// of the radix-32 pass).
template <int LOG2N, bool PRE0 = false>
__device__ __forceinline__ void warp_fft(float2 (&z)[32], float* xb, const float2* tw, int l) {
  using PL = WPlan<LOG2N>;
  constexpr int LPF = PL::LPF, R1 = PL::R1, B1 = PL::B1;
  {
    float2 o[32];
    DFT<32, 1, PRE0>::run(z, o);
#pragma unroll
    for (int t = 0; t < 32; ++t) z[t] = o[t];
  }
  if constexpr (R1 >= 2) {
    // exchange (transpose within the frame's lanes): write i = l*32 + t, read e = l + LPF m
#pragma unroll
    for (int t = 0; t < 32; ++t) xb[l * 33 + t] = z[t].x;
    __syncwarp();
#pragma unroll
    for (int m = 0; m < 32; ++m) { const int e = l + LPF * m; z[m].x = xb[e + (e >> 5)]; }
    __syncwarp();
#pragma unroll
    for (int t = 0; t < 32; ++t) xb[l * 33 + t] = z[t].y;
    __syncwarp();
#pragma unroll
    for (int m = 0; m < 32; ++m) { const int e = l + LPF * m; z[m].y = xb[e + (e >> 5)]; }
    __syncwarp();
    if constexpr (PL::LEAN) {
      const float2 w8 = tw[7 * LPF + l], w16 = tw[8 * LPF + l], w24 = tw[9 * LPF + l];
      z[8] = cmul(z[8], w8); z[16] = cmul(z[16], w16); z[24] = cmul(z[24], w24);
#pragma unroll
      for (int b = 1; b < 8; ++b) {
        const float2 wb = tw[(b - 1) * LPF + l];
        z[b] = cmul(z[b], wb);
        z[8 + b] = cmul(cmul(z[8 + b], wb), w8);
        z[16 + b] = cmul(cmul(z[16 + b], wb), w16);
        z[24 + b] = cmul(cmul(z[24 + b], wb), w24);
      }
    }
#pragma unroll
    for (int b = 0; b < B1; ++b) {  // pass 1: radix LPF, NS = 32
      if constexpr (!PL::LEAN) {
#pragma unroll
        for (int t = 1; t < R1; ++t)
          z[b + B1 * t] = cmul(z[b + B1 * t], tw[(b * (R1 - 1) + (t - 1)) * LPF + l]);
      }
      float2 o[R1];
      DFT<R1, B1>::run(&z[b], o);
#pragma unroll
      for (int t = 0; t < R1; ++t) z[b + B1 * t] = o[t];
    }
  }
}

// untangle twiddle exp(-i pi (l + LPF m) / N) of lane l, slot m < 16; `u0` = the lane's entry ut[l] (LEAN) -- loaded once
// per frame by the caller
template <int LOG2N, int M>
__device__ __forceinline__ float2 untangle_twiddle(const float2* ut, float2 u0, int l) {
  using PL = WPlan<LOG2N>;
  if constexpr (PL::LEAN) {
    if constexpr (M == 0) {
      return u0;
    } else {
      constexpr float c = cos_pi32(M), sn = cos_pi32(16 - M);  // exp(-i pi M / 32) = c - i sn
      return fma2(bcast2(u0.x), make_float2(c, -sn), mul2(bcast2(u0.y), make_float2(sn, c)));  // u0 * (c - i sn)
    }
  } else {
    return ut[M * PL::LPF + l];
  }
}

template <int LOG2N>
__device__ __forceinline__ float2 untangle_twiddle_m(const float2* ut, float2 u0, int l, int m) {
  switch (m) {  // called from fully unrolled loops: m is a compile-time constant after unrolling
    case 0: return untangle_twiddle<LOG2N, 0>(ut, u0, l);
    case 1: return untangle_twiddle<LOG2N, 1>(ut, u0, l);
    case 2: return untangle_twiddle<LOG2N, 2>(ut, u0, l);
    case 3: return untangle_twiddle<LOG2N, 3>(ut, u0, l);
    case 4: return untangle_twiddle<LOG2N, 4>(ut, u0, l);
    case 5: return untangle_twiddle<LOG2N, 5>(ut, u0, l);
    case 6: return untangle_twiddle<LOG2N, 6>(ut, u0, l);
    case 7: return untangle_twiddle<LOG2N, 7>(ut, u0, l);
    case 8: return untangle_twiddle<LOG2N, 8>(ut, u0, l);
    case 9: return untangle_twiddle<LOG2N, 9>(ut, u0, l);
    case 10: return untangle_twiddle<LOG2N, 10>(ut, u0, l);
    case 11: return untangle_twiddle<LOG2N, 11>(ut, u0, l);
    case 12: return untangle_twiddle<LOG2N, 12>(ut, u0, l);
    case 13: return untangle_twiddle<LOG2N, 13>(ut, u0, l);
    case 14: return untangle_twiddle<LOG2N, 14>(ut, u0, l);
    default: return untangle_twiddle<LOG2N, 15>(ut, u0, l);
  }
}

// ---- front end of a warp frame (spectral_warp_kernel and spectral_loss_kernel load it with the same instructions, so
//      the fused loss transforms exactly the frames stft() does)

// lane of the same frame that holds Z[N - k] for this lane's Z[k] (l = lane % LPF <-> LPF - l; lane 0 holds both itself)
template <int LPF>
__device__ __forceinline__ int partner_lane(int lane) {
  return (lane & ~(LPF - 1)) | ((LPF - (lane & (LPF - 1))) & (LPF - 1));
}

// windowed frame, element e = l + LPF m; the first butterfly stage of the radix-32 pass (elements m and m + 16) is
// formed right here with the window multiply fused in: a = s_m w_m, sum = fma(s_n, w_n, a), difference =
// fma(-s_n, w_n, a)  (3 instead of 4 instructions per component pair).  Feeds warp_fft<LOG2N, true>.
template <int LOG2N>
__device__ __forceinline__ void load_frame(const float* fs, const float* win, int hop, float2 (&z)[32], int l) {
  constexpr int LPF = WPlan<LOG2N>::LPF;
  if ((hop & 1) == 0) {
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      const int e0 = l + LPF * m, e1 = e0 + LPF * 16;
      const float2 s0 = *reinterpret_cast<const float2*>(fs + 2 * e0);
      const float2 w0 = *reinterpret_cast<const float2*>(win + 2 * e0);
      const float2 s1 = *reinterpret_cast<const float2*>(fs + 2 * e1);
      const float2 w1 = *reinterpret_cast<const float2*>(win + 2 * e1);
      const float2 a = mul2(s0, w0);
      z[m] = fma2(s1, w1, a);
      z[m + 16] = fma2(neg2(s1), w1, a);
    }
  } else {
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      const int e0 = l + LPF * m, e1 = e0 + LPF * 16;
      const float ax = fs[2 * e0] * win[2 * e0], ay = fs[2 * e0 + 1] * win[2 * e0 + 1];
      const float sx = fs[2 * e1], sy = fs[2 * e1 + 1], wx = win[2 * e1], wy = win[2 * e1 + 1];
      z[m] = make_float2(fmaf(sx, wx, ax), fmaf(sy, wy, ay));
      z[m + 16] = make_float2(fmaf(-sx, wx, ax), fmaf(-sy, wy, ay));
    }
  }
}

// role-constant tables of the warp FFT: pass-1 twiddles [NTW][LPF] and untangle twiddles [16][LPF]
// NUT: untangle-twiddle slots to fill (16 = the full table other kernels index directly; WPlan::NUT = the lean form)
template <int LOG2N, int NUT = 16>
__device__ __forceinline__ void warp_fft_tables(float2* tw, float2* ut) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N, LPF = PL::LPF, R1 = PL::R1;
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < PL::NTW * LPF; i += nt) {
    const int slot = i / LPF, ll = i - slot * LPF;
    int e;  // exponent of W_N
    if constexpr (PL::LEAN) {
      e = ll * (slot < 7 ? slot + 1 : 8 * (slot - 6));
    } else {
      const int b = slot / (R1 > 1 ? R1 - 1 : 1), t = slot - b * (R1 > 1 ? R1 - 1 : 1) + 1;
      e = (ll + LPF * b) * t;
    }
    float sn, cs;
    sincospif(-2.0f * (float)e / (float)N, &sn, &cs);
    tw[i] = make_float2(cs, sn);
  }
  for (int i = tid; i < NUT * LPF; i += nt) {
    const int m = i / LPF, ll = i - m * LPF;
    float sn, cs;  // exp(-i pi (ll + LPF m) / N)
    sincospif(-(float)(ll + LPF * m) / (float)N, &sn, &cs);
    ut[i] = make_float2(cs, sn);
  }
}

}  // namespace spectral
}  // namespace b2a
