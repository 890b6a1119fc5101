// fft_large.cu -- STFT / inverse STFT of the large power-of-two windows (forward 8192 .. 32768, inverse 4096 .. 32768)
// as FFTs on sm_90a.
//
// spectral.cu keeps a whole tile of frames plus a full window / twiddle plan in shared memory, which stops at 4096;
// the dense DFT of dft.cu would do O(n_fft^2) work per frame here.  These kernels give each frame ONE CTA and keep only
// that frame in shared memory (16384 complex points = 128 KB at n_fft = 32768); the window is read through L2 and the
// twiddles are computed (sincospif) where they are used.
//
// A real frame of n_fft = 2N samples is FFT-ed as N packed complex points z[n] = x[2n] + i x[2n+1] plus the untangle
//     X[k] = E[k] + W^k O[k],  X[N-k] = conj(E[k] - W^k O[k]),   E = (Z[k] + conj Z[N-k]) / 2,
//     O = (Z[k] - conj Z[N-k]) / 2i,  W = exp(-i pi / N),
// and the N-point complex FFT is split four-step as N = N1 x N2 with N2 = 1024, N1 = N / 1024 in {2 .. 16}:
//   1. column DFTs of length N1 in registers (thread per column n2, DFT<N1> of fft_warp.cuh), times W_N^(n2 k1);
//   2. row FFTs of length 1024, one warp per row (warp_fft<10> of fft_warp.cuh, its lean twiddle table);
//   3. result Z[k1 + N1 k2] sits at row k1, column k2 (rows padded to 1025 points: the strided reads of the untangle
//      are conflict-free), read there by the untangle.
// One warp per row: N1 warps per CTA (64 .. 512 threads).  The inverse runs the same steps backwards through
// IFFT(Z) = conj(FFT(conj Z)) / N, writes the windowed frames to the workspace in the layout fold_kernel (dft.cu)
// reads, and lets it do the overlap-add and the envelope division.
#include "b2a_common.h"
#include "dft_internal.h"
#include "fft_warp.cuh"
#include "grad_internal.h"
#include "spectral_internal.h"

namespace b2a {
namespace large {

using spectral::cmul;
using spectral::DFT;

constexpr int N2 = 1024;      // row length (the warp FFT)
constexpr int RS = N2 + 1;    // row stride in complex points
constexpr int TW_PTS = 10 * 32 + 32;  // warp_fft<10> lean twiddles (10 slots x 32 lanes) + its 32 untangle entries

template <int LOG2_NFFT>
struct Geo {
  static constexpr int NFFT = 1 << LOG2_NFFT;
  static constexpr int N = NFFT / 2;          // complex points
  static constexpr int L1 = LOG2_NFFT - 11;   // log2 N1
  static constexpr int N1 = 1 << L1;
  static constexpr int NT = 32 * N1;          // one warp per row
  static constexpr int CPT = N2 / NT;         // columns per thread in step 1
  static constexpr size_t SMEM = (size_t)(TW_PTS + N1 * RS) * sizeof(float2);
  static_assert(N1 >= 2 && N1 <= 16, "n_fft 4096 .. 32768");
};

// W_N^e = exp(-2 pi i e / N), 0 <= e < N
template <int N>
__device__ __forceinline__ float2 twiddle(int e) {
  float sn, cs;
  sincospif((float)e * (-2.0f / (float)N), &sn, &cs);
  return make_float2(cs, sn);
}

// Z[k] of the N-point transform, k in [0, N): row k mod N1, column k / N1
template <int LOG2_NFFT>
__device__ __forceinline__ int zpos(int k) {
  using G = Geo<LOG2_NFFT>;
  return (k & (G::N1 - 1)) * RS + (k >> G::L1);
}

// steps 1 + 2 of the four-step FFT over s (x[p] at row p / N2, column p mod N2 on entry)
template <int LOG2_NFFT>
__device__ __forceinline__ void fft_in_smem(float2* s, const float2* tw) {
  using G = Geo<LOG2_NFFT>;
  constexpr int N1 = G::N1;
  const int tid = threadIdx.x;
  // 1. columns: each thread owns its columns completely (reads and writes them in place)
#pragma unroll 1
  for (int c = 0; c < G::CPT; ++c) {
    const int n2 = tid + G::NT * c;
    float2 v[N1], o[N1];
#pragma unroll
    for (int n1 = 0; n1 < N1; ++n1) v[n1] = s[n1 * RS + n2];
    DFT<N1, 1>::run(v, o);
    s[n2] = o[0];
#pragma unroll
    for (int k1 = 1; k1 < N1; ++k1) s[k1 * RS + n2] = cmul(o[k1], twiddle<G::N>(n2 * k1));
  }
  __syncthreads();
  // 2. rows: warp w transforms row w in place (the row doubles as the warp FFT's exchange buffer)
  const int w = tid >> 5, l = tid & 31;
  float2* row = s + w * RS;
  float2 z[32];
#pragma unroll
  for (int m = 0; m < 32; ++m) z[m] = row[l + 32 * m];
  __syncwarp();
  spectral::warp_fft<10>(z, reinterpret_cast<float*>(row), tw, l);
#pragma unroll
  for (int m = 0; m < 32; ++m) row[l + 32 * m] = z[m];
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// forward: stft_out[row][k][f], k = 0 .. N (frame axis fastest), the framing of spectral.cu / dft.cu
// ---------------------------------------------------------------------------------------------
struct FwdParams {
  const float* x;
  const float* window;
  float2* out;
  int T, hop, pad, right_pad, pad_mode, drop_edge, n_frames;
  int origin, center;  // frame f starts at x-coordinate (f + drop_edge) hop + origin; center: src_index's framing flag
};

template <int LOG2_NFFT>
__global__ void __launch_bounds__(Geo<LOG2_NFFT>::NT, 1) stft_large_kernel(const FwdParams p) {
  using G = Geo<LOG2_NFFT>;
  constexpr int N = G::N, NFFT = G::NFFT;
  B2A_DYN_SMEM(smem);
  float2* tw = reinterpret_cast<float2*>(smem);
  float2* s = tw + TW_PTS;
  const int tid = threadIdx.x;
  const int row = (int)(blockIdx.x / (unsigned)p.n_frames);
  const int f = (int)(blockIdx.x - (unsigned)row * (unsigned)p.n_frames);
  spectral::warp_fft_tables<10, 1>(tw, tw + 10 * 32);

  const float* xr = p.x + (size_t)row * (size_t)p.T;
  const long long base = (long long)(f + p.drop_edge) * p.hop + p.origin;  // x-coordinate of sample 0
  const bool interior = base >= 0 && base + NFFT <= (long long)p.T;
  auto sample = [&](int n) -> float {
    if (interior) return __ldg(xr + (base + n));
    const int u = spectral::src_index((int)(base + n), p.T, p.pad, p.right_pad, p.pad_mode, p.center);
    return u >= 0 ? __ldg(xr + u) : 0.f;
  };
  // framing + window: point q = x[2q] + i x[2q+1] at row q / N2, column q mod N2
  for (int q = tid; q < N; q += G::NT) {
    const float a = sample(2 * q) * __ldg(p.window + 2 * q);
    const float b = sample(2 * q + 1) * __ldg(p.window + 2 * q + 1);
    s[(q >> 10) * RS + (q & (N2 - 1))] = make_float2(a, b);
  }
  __syncthreads();
  fft_in_smem<LOG2_NFFT>(s, tw);

  // untangle: bins k and N - k from Z[k], Z[N - k]
  float2* o = p.out + (size_t)row * (size_t)(N + 1) * (size_t)p.n_frames + f;
  for (int k = tid; k <= N / 2; k += G::NT) {
    const float2 zk = s[zpos<LOG2_NFFT>(k)], zn = s[zpos<LOG2_NFFT>((N - k) & (N - 1))];
    const float2 e = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));
    const float2 od = make_float2(0.5f * (zk.y + zn.y), -0.5f * (zk.x - zn.x));  // (Z[k] - conj Z[N-k]) / 2i
    float sn, cs;
    sincospif((float)k * (1.0f / (float)N), &sn, &cs);
    const float2 wo = cmul(od, make_float2(cs, -sn));
    o[(size_t)k * p.n_frames] = make_float2(e.x + wo.x, e.y + wo.y);
    if (2 * k != N) o[(size_t)(N - k) * p.n_frames] = make_float2(e.x - wo.x, wo.y - e.y);
  }
}

// ---------------------------------------------------------------------------------------------
// inverse: frames[row][f][n] = w[n] . irfft(spec[row][:, f])[n]  (torch.istft's per-frame inverse, norm 1/n_fft)
// ---------------------------------------------------------------------------------------------
struct InvParams {
  const float2* spec;
  const float* window;
  float* frames;
  int n_frames;
  int adjoint;  // 1: bin weights 1 instead of c_k / n_fft (the STFT's adjoint; the fold then skips the envelope)
};

template <int LOG2_NFFT>
__global__ void __launch_bounds__(Geo<LOG2_NFFT>::NT, 1) istft_large_kernel(const InvParams p) {
  using G = Geo<LOG2_NFFT>;
  constexpr int N = G::N, NFFT = G::NFFT;
  B2A_DYN_SMEM(smem);
  float2* tw = reinterpret_cast<float2*>(smem);
  float2* s = tw + TW_PTS;
  const int tid = threadIdx.x;
  const int row = (int)(blockIdx.x / (unsigned)p.n_frames);
  const int f = (int)(blockIdx.x - (unsigned)row * (unsigned)p.n_frames);
  spectral::warp_fft_tables<10, 1>(tw, tw + 10 * 32);

  // re-tangle: Z[k] = E + i O with E = (X[k] + conj X[N-k]) / 2, O = (X[k] - conj X[N-k]) / 2 . W^-k; stored as
  // conj(Z) / N (the forward FFT of the conjugate is N conj(z)).  The imaginary parts of DC and Nyquist do not
  // enter, as in a C2R transform.
  const float2* sp = p.spec + (size_t)row * (size_t)(N + 1) * (size_t)p.n_frames + f;
  const float inv_n = p.adjoint ? 1.0f : 1.0f / (float)N;  // adjoint: n_fft/2 x the inverse, DC / Nyquist doubled
  for (int k = tid; k <= N / 2; k += G::NT) {
    float2 xk = sp[(size_t)k * p.n_frames], xn = sp[(size_t)(N - k) * p.n_frames];
    if (k == 0) {
      xk.y = 0.f; xn.y = 0.f;
      if (p.adjoint) { xk.x *= 2.f; xn.x *= 2.f; }
    }
    const float2 e = make_float2(0.5f * (xk.x + xn.x), 0.5f * (xk.y - xn.y));
    const float2 d = make_float2(0.5f * (xk.x - xn.x), 0.5f * (xk.y + xn.y));
    float sn, cs;
    sincospif((float)k * (1.0f / (float)N), &sn, &cs);
    const float2 od = cmul(d, make_float2(cs, sn));
    // conj(Z[k]) = (e.x - od.y, -(e.y + od.x)),  conj(Z[N-k]) = (e.x + od.y, e.y - od.x)
    s[(k >> 10) * RS + (k & (N2 - 1))] = make_float2(inv_n * (e.x - od.y), -inv_n * (e.y + od.x));
    if (k != 0 && 2 * k != N) {
      const int q = N - k;
      s[(q >> 10) * RS + (q & (N2 - 1))] = make_float2(inv_n * (e.x + od.y), inv_n * (e.y - od.x));
    }
  }
  __syncthreads();
  fft_in_smem<LOG2_NFFT>(s, tw);

  // z[n] = conj(Y[n]): x[2n] = Y.x, x[2n+1] = -Y.y, windowed, one float2 per point
  float* fr = p.frames + ((size_t)row * p.n_frames + f) * (size_t)NFFT;
  for (int n = tid; n < N; n += G::NT) {
    const float2 y = s[zpos<LOG2_NFFT>(n)];
    *reinterpret_cast<float2*>(fr + 2 * n) =
        make_float2(__ldg(p.window + 2 * n) * y.x, -(__ldg(p.window + 2 * n + 1) * y.y));
  }
}

template <int LOG2_NFFT>
int launch_fwd(const FwdParams& p, int64_t rows, void* stream) {
  using G = Geo<LOG2_NFFT>;
  B2A_CUDA_OK(cudaFuncSetAttribute(stft_large_kernel<LOG2_NFFT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)G::SMEM));
  B2A_LAUNCH(stft_large_kernel<LOG2_NFFT>, dim3((unsigned)(rows * p.n_frames)), dim3(G::NT), G::SMEM, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

template <int LOG2_NFFT>
int launch_inv(const InvParams& p, int64_t rows, void* stream) {
  using G = Geo<LOG2_NFFT>;
  B2A_CUDA_OK(cudaFuncSetAttribute(istft_large_kernel<LOG2_NFFT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)G::SMEM));
  B2A_LAUNCH(istft_large_kernel<LOG2_NFFT>, dim3((unsigned)(rows * p.n_frames)), dim3(G::NT), G::SMEM, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

}  // namespace large
}  // namespace b2a

using namespace b2a::large;

static inline int log2_pow2(int n) {
  int l = 0;
  while ((1 << l) < n) ++l;
  return (1 << l) == n ? l : -1;
}

// the window lengths of these kernels: forward 8192 .. 32768, hop >= 1; inverse 4096 .. 32768, 1 <= hop <= n_fft
static bool supported(int n_fft, int hop, int inverse) {
  const int l = n_fft >= 2 ? log2_pow2(n_fft) : -1;
  if (hop < 1 || l > 15) return false;
  return inverse ? (l >= 12 && hop <= n_fft) : l >= 13;
}

static int launch_fwd_any(const FwdParams& p, int64_t rows, int n_fft, void* stream);

int b2a::large::stft(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window, int pad,
                     int right_pad, int pad_mode, int drop_edge, float* stft_out, void* stream) {
  B2A_REQUIRE(x && window && stft_out, B2A_E_INVALID, "stft_large: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1, B2A_E_INVALID, "stft_large: empty input");
  B2A_REQUIRE(T < (int64_t)1 << 30, B2A_E_UNSUPPORTED, "stft_large: rows longer than 2^30 samples");
  B2A_REQUIRE(supported(n_fft, hop, 0), B2A_E_UNSUPPORTED,
              "stft_large: window_length %d hop %d (powers of two 8192 .. 32768, hop >= 1)", n_fft, hop);
  int64_t nfr;
  const int rc = b2a::spectral::check_framing("stft_large", T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(rows * nfr < (int64_t)2147483647, B2A_E_UNSUPPORTED, "stft_large: too many frames");
  FwdParams p;
  p.x = x; p.window = window; p.out = reinterpret_cast<float2*>(stft_out);
  p.T = (int)T; p.hop = hop; p.pad = pad; p.right_pad = right_pad; p.pad_mode = pad_mode; p.drop_edge = drop_edge;
  p.n_frames = (int)nfr; p.origin = -(n_fft / 2) - pad; p.center = 1;
  return launch_fwd_any(p, rows, n_fft, stream);
}

static int launch_fwd_any(const FwdParams& p, int64_t rows, int n_fft, void* stream) {
  switch (n_fft) {
    case 4096: return launch_fwd<12>(p, rows, stream);
    case 8192: return launch_fwd<13>(p, rows, stream);
    case 16384: return launch_fwd<14>(p, rows, stream);
    default: return launch_fwd<15>(p, rows, stream);
  }
}

int b2a::large::forward_raw(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window,
                            int64_t origin, int64_t n_frames, float* out, void* stream) {
  B2A_REQUIRE(supported(n_fft, hop, 1), B2A_E_UNSUPPORTED, "stft_large: window_length %d hop %d", n_fft, hop);
  B2A_REQUIRE(T < (int64_t)1 << 30 && rows * n_frames < (int64_t)2147483647 && origin > -((int64_t)1 << 30) &&
                  origin < ((int64_t)1 << 30),
              B2A_E_UNSUPPORTED, "stft_large: too large");
  FwdParams p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.window = window; p.out = reinterpret_cast<float2*>(out);
  p.T = (int)T; p.hop = hop; p.pad_mode = B2A_PAD_CONSTANT; p.n_frames = (int)n_frames; p.origin = (int)origin;
  p.center = 0;
  return launch_fwd_any(p, rows, n_fft, stream);
}

int b2a::large::inverse_frames(const float* spec, int64_t rows, int64_t n_frames, int n_fft, const float* window,
                               float* frames, int adjoint, void* stream) {
  InvParams p;
  p.spec = reinterpret_cast<const float2*>(spec); p.window = window; p.frames = frames;
  p.n_frames = (int)n_frames; p.adjoint = adjoint ? 1 : 0;
  switch (n_fft) {
    case 4096: return launch_inv<12>(p, rows, stream);
    case 8192: return launch_inv<13>(p, rows, stream);
    case 16384: return launch_inv<14>(p, rows, stream);
    default: return launch_inv<15>(p, rows, stream);
  }
}

int b2a::large::istft(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window,
                      int pad_frames, int64_t start, int64_t out_len, float* out, void* ws, size_t ws_bytes,
                      void* stream) {
  B2A_REQUIRE(spec && window && out && ws, B2A_E_INVALID, "istft_large: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && n_frames >= 1 && out_len >= 1 && pad_frames >= 0 && start >= 0,
              B2A_E_INVALID, "istft_large: bad argument");
  B2A_REQUIRE(supported(n_fft, hop, 1), B2A_E_UNSUPPORTED,
              "istft_large: n_fft=%d hop=%d (powers of two 4096 .. 32768, 1 <= hop <= n_fft)", n_fft, hop);
  B2A_REQUIRE(ws_bytes >= (size_t)rows * (size_t)n_frames * (size_t)n_fft * sizeof(float), B2A_E_INVALID,
              "istft_large: workspace too small");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0 && ((uintptr_t)ws & 7) == 0, B2A_E_INVALID,
              "istft_large: spectra and workspace must be 8-byte aligned");
  B2A_REQUIRE(rows * n_frames < (int64_t)2147483647, B2A_E_UNSUPPORTED, "istft_large: too many frames");
  float* frames = reinterpret_cast<float*>(ws);
  const int rc = b2a::large::inverse_frames(spec, rows, n_frames, n_fft, window, frames, 0, stream);
  if (rc != B2A_OK) return rc;
  return b2a::dft::launch_fold(frames, window, rows, (int)n_frames, n_fft, hop, pad_frames, start, out_len, 1, out,
                               stream);
}
