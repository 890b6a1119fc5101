// spectral.cu -- fused framing -> window -> real FFT -> |.| -> banded mel -> post-op on sm_90a.
//
// Replaces the device work of AudioSignal.stft (ref:audiotools/core/audio_signal.py:1123-1212),
// AudioSignal.mel_spectrogram (:1333-1369), the log-mel of ref:audiotools/metrics/spectral.py:187-190
// and -- optionally, in the same pass over x -- the x*gain of EffectMixin.normalize
// (ref:audiotools/core/effects.py:219).  The reference materialises the complex STFT
// ([64,2,1025,862] c64 = 905 MB at BASELINE cfg2), |.|, a transpose and a matmul; here the
// spectrum of a frame never leaves the SM.
//
// One CTA (256 threads) owns FR consecutive frames of one row:
//   1. the contiguous sample span those frames cover ((FR-1)*hop + n_fft samples) is loaded ONCE
//      into shared memory (coalesced 128-bit loads; optional *gain and write-back of the scaled
//      waveform for the samples the CTA owns); edge tiles resolve torch's two nested paddings
//      (F.pad(pad, pad+right_pad, mode) then stft(center=True) reflect) per sample, bit-exact in
//      the frame/sample indexing;
//   2. G = 256/(N/16) frames are transformed concurrently, N = n_fft/2: the real frame is packed
//      as N complex points, each thread keeps 16 of them in registers, and a Stockham
//      auto-sort FFT runs as 2-3 radix-16/8/4/2 passes with one shared-memory exchange between
//      passes (reads are always lane-consecutive; the strided pass-0 write is padded 17/16).
//      Twiddles depend only on the thread's role, so they are computed once per CTA (sincospif)
//      and kept in shared memory in [slot][thread] order (conflict-free);
//   3. the N-point spectrum is untangled into the n_fft/2+1 real-FFT bins; optional stft_out;
//   4. |X| -> banded mel projection in FP32 (each Slaney filter touches 2..63 of the 1025 bins:
//      2013 non-zeros of 131200 at 44.1k/2048/128, so the banded FP32 sum costs 64x fewer FLOPs
//      than a dense tensor-core GEMM and is exact to FP32 rounding) -> post-op -> tile in shared
//      memory -> coalesced store along the frame axis.
#include "b2a_common.h"
#include "fft_warp.cuh"
#include "grad_internal.h"
#include "spectral_internal.h"

namespace b2a {
namespace spectral {

constexpr int THREADS = 256;
constexpr int E = 16;  // complex points per thread

// ---------------------------------------------------------------------------------------------
// compile-time FFT plan for N = 2^LOG2N complex points, 16 points per thread
// ---------------------------------------------------------------------------------------------
template <int LOG2N>
struct Plan {
  static constexpr int N = 1 << LOG2N;
  static constexpr int TPF = N / E;          // threads per frame
  static constexpr int G = THREADS / TPF;    // frames in flight per CTA
  static constexpr int P = (LOG2N + 3) / 4;  // passes
  static constexpr int radix(int p) {        // 16,16,...,rest
    return (p < LOG2N / 4) ? 16 : (1 << (LOG2N % 4));
  }
  static constexpr int ns(int p) { return 1 << (4 * p); }  // product of earlier radices
  // twiddle slots of pass p (p >= 1): (16/R) butterflies x (R-1) factors
  static constexpr int slots(int p) { return p == 0 ? 0 : (E / radix(p)) * (radix(p) - 1); }
  static constexpr int slot_off(int p) {
    int o = 0;
    for (int i = 1; i < p; ++i) o += slots(i);
    return o;
  }
  static constexpr int NSLOT = slot_off(P);
  static constexpr int BUF = N + N / 16 + 1;  // padded complex work buffer per frame
  static constexpr int MAG = N + 4;           // floats per frame (N+1 used)
  // frames per CTA: enough rounds to amortise the span load, bounded shared memory
  static constexpr int FR = (G >= 16) ? G : ((LOG2N >= 11) ? 2 * G : ((LOG2N == 10) ? 4 * G : 16));
};

// Stage the contiguous sample span of a tile into shared memory (x * gain) and write back the part
// of the scaled waveform this CTA owns ([n0*hop, (n0+FR)*hop) -- the last tile up to T).
__device__ __forceinline__ void stage_span(const Params& p, float* sp, int row, int tile, int n0, int FR, int ws,
                                           float g) {
  const int tid = threadIdx.x, T = p.T, hop = p.hop, span = p.span;
  const float* xr = p.x + (size_t)row * (size_t)T;
  // ---- stage the sample span (x * gain), write back the owned part of the scaled waveform
  const int own_lo = n0 * hop;  // only used when y_out (pad == 0, drop_edge == 0)
  const int own_hi = (tile == p.n_tiles - 1) ? T : min(T, (n0 + FR) * hop);
  const bool interior = (ws >= 0) && (ws + span <= T);
  if (interior) {
    const float* src = xr + ws;
    const bool vec = ((((uintptr_t)src) & 15) == 0) && ((span & 3) == 0) &&
                     (!p.y_out || (((uintptr_t)(p.y_out + (size_t)row * T + ws)) & 15) == 0);
    if (vec) {
      for (int i = tid * 4; i < span; i += (int)blockDim.x * 4) {
        float4 v = *reinterpret_cast<const float4*>(src + i);
        if (p.gain) { v.x *= g; v.y *= g; v.z *= g; v.w *= g; }
        *reinterpret_cast<float4*>(sp + i) = v;
        if (p.y_out) {
          const int w = ws + i;
          if (w >= own_lo && w + 3 < own_hi) {
            *reinterpret_cast<float4*>(p.y_out + (size_t)row * T + w) = v;
          } else {
            float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (w + e >= own_lo && w + e < own_hi) p.y_out[(size_t)row * T + w + e] = vv[e];
          }
        }
      }
    } else {
      for (int i = tid; i < span; i += (int)blockDim.x) {
        float v = __ldg(src + i);
        if (p.gain) v *= g;
        sp[i] = v;
        const int w = ws + i;
        if (p.y_out && w >= own_lo && w < own_hi) p.y_out[(size_t)row * T + w] = v;
      }
    }
  } else {
    for (int i = tid; i < span; i += (int)blockDim.x) {
      const int w = ws + i;
      const int u = src_index(w, T, p.pad, p.right_pad, p.pad_mode);
      float v = (u >= 0) ? __ldg(xr + u) : 0.f;
      if (p.gain) v *= g;
      sp[i] = v;
      if (p.y_out && w >= own_lo && w < own_hi) p.y_out[(size_t)row * T + w] = v;  // w in [0,T) => u == w
    }
  }
  if (p.y_out) {  // owned samples the span does not cover (only when hop > n_fft/2)
    for (int w = max(own_lo, ws + span) + tid; w < own_hi; w += (int)blockDim.x) {
      float v = __ldg(xr + w);
      if (p.gain) v *= g;
      p.y_out[(size_t)row * T + w] = v;
    }
  }
}

// y_out[w] = x[w] * g for the samples this CTA owns (requires pad == drop_edge == 0, so span[i] = x[ws+i])
__device__ __forceinline__ void writeback_scaled(const Params& p, const float* sp, int row, int tile, int n0, int FR,
                                                 int ws, float g) {
  const int tid = threadIdx.x, T = p.T, hop = p.hop, span = p.span;
  const int own_lo = n0 * hop;
  const int own_hi = (tile == p.n_tiles - 1) ? T : min(T, (n0 + FR) * hop);
  float* yr = p.y_out + (size_t)row * (size_t)T;
  const int lo = max(own_lo, ws), hi = min(own_hi, ws + span);  // part covered by the span
  const bool vec = (((lo - ws) & 3) == 0) && ((((uintptr_t)(yr + lo)) & 15) == 0);
  if (vec) {
    const int n4 = (hi - lo) >> 2;
    for (int i = tid; i < n4; i += (int)blockDim.x) {
      float4 v = *reinterpret_cast<const float4*>(sp + (lo - ws) + 4 * i);
      v.x *= g; v.y *= g; v.z *= g; v.w *= g;
      st_stream4(yr + lo + 4 * i, v);
    }
    for (int w = lo + 4 * n4 + tid; w < hi; w += (int)blockDim.x) yr[w] = sp[w - ws] * g;
  } else {
    for (int w = lo + tid; w < hi; w += (int)blockDim.x) yr[w] = sp[w - ws] * g;
  }
  const float* xr = p.x + (size_t)row * (size_t)T;
  for (int w = max(own_lo, ws + span) + tid; w < own_hi; w += (int)blockDim.x) yr[w] = __ldg(xr + w) * g;
}

template <int TPF>
__device__ __forceinline__ void group_sync(int g) {
  if constexpr (TPF >= 64) {
    B2A_BAR_SYNC(1 + g, TPF);
  } else {
    __syncwarp();
  }
}

template <int LOG2N>
__device__ __forceinline__ int buf_phys(int i) { return i + (i >> 4); }

// one Stockham pass p >= 1 on the 16 register-resident points of this thread
template <int LOG2N, int PASS>
__device__ __forceinline__ void fft_pass(float2 (&v)[E], float2* buf, const float2* tw, int q) {
  using PL = Plan<LOG2N>;
  constexpr int R = PL::radix(PASS), NS = PL::ns(PASS), B = E / R, TPF = PL::TPF;
#pragma unroll
  for (int b = 0; b < B; ++b) {
    // twiddle: v[b + B t] *= W_{NS*R}^{k t}
#pragma unroll
    for (int t = 1; t < R; ++t) {
      float2 w = tw[(PL::slot_off(PASS) + b * (R - 1) + (t - 1)) * TPF + q];
      v[b + B * t] = cmul(v[b + B * t], w);
    }
    float2 out[R];
    DFT<R, B>::run(&v[b], out);
    const int j = q + TPF * b;
    const int k = j & (NS - 1);
    const int base = (j - k) * R + k;
#pragma unroll
    for (int t = 0; t < R; ++t) buf[buf_phys<LOG2N>(base + t * NS)] = out[t];
  }
}

template <int LOG2N>
__global__ void __launch_bounds__(THREADS) spectral_kernel(Params p) {
  using PL = Plan<LOG2N>;
  constexpr int N = PL::N, TPF = PL::TPF, G = PL::G, FR = PL::FR, P = PL::P;
  B2A_DYN_SMEM(smem);
  float* sp = reinterpret_cast<float*>(smem);                        // sample span
  float* win = reinterpret_cast<float*>(smem + p.off_win);           // [n_fft]
  float2* tw = reinterpret_cast<float2*>(smem + p.off_tw);           // [NSLOT][TPF]
  float2* ut = reinterpret_cast<float2*>(smem + p.off_ut);           // [N/2+1]  exp(-i pi k / N)
  float2* bufs = reinterpret_cast<float2*>(smem + p.off_buf);        // [G][BUF]
  float* mags = reinterpret_cast<float*>(smem + p.off_mag);          // [G][MAG]
  float* melt = reinterpret_cast<float*>(smem + p.off_mel);          // [n_mels][FR+1]

  const int tid = threadIdx.x;
  const int row = blockIdx.x / p.n_tiles;
  const int tile = blockIdx.x - row * p.n_tiles;
  const int n0 = tile * FR;  // first output frame of this CTA
  const int hop = p.hop, n_fft = 2 * N;
  const float g = p.gain ? __ldg(p.gain + row / p.rows_per_gain) : 1.0f;
  const int ws = (n0 + p.drop_edge) * hop - N - p.pad;  // x-coordinate of span[0]

  // ---- tables (role-dependent only)
  for (int i = tid; i < n_fft; i += THREADS) win[i] = __ldg(p.window + i);
  for (int i = tid; i < PL::NSLOT * TPF; i += THREADS) {
    const int slot = i / TPF, q = i - slot * TPF;
    int pass = 1;
#pragma unroll
    for (int pp = 1; pp < P; ++pp)
      if (slot >= PL::slot_off(pp)) pass = pp;
    const int R = PL::radix(pass), NS = PL::ns(pass);
    const int s = slot - PL::slot_off(pass);
    const int b = s / (R - 1), t = s - b * (R - 1) + 1;
    const int k = (q + TPF * b) & (NS - 1);
    float sn, cs;
    sincospif(-2.0f * (float)(k * t) / (float)(NS * R), &sn, &cs);
    tw[i] = make_float2(cs, sn);
  }
  for (int i = tid; i <= N / 2; i += THREADS) {
    float sn, cs;
    sincospif(-(float)i / (float)N, &sn, &cs);
    ut[i] = make_float2(cs, sn);
  }

  stage_span(p, sp, row, tile, n0, FR, ws, g);
  __syncthreads();

  const int grp = tid / TPF, q = tid - grp * TPF;
  float2* buf = bufs + grp * PL::BUF;
  float* mag = mags + grp * PL::MAG;
  const int F = N + 1;

  for (int rd = 0; rd < FR / G; ++rd) {
    const int f = rd * G + grp;  // frame within the tile
    const int n = n0 + f;        // output frame index
    const bool live = n < p.n_frames;
    const float* fs = sp + f * hop;

    // ---- pass 0: windowed real frame packed as N complex points, radix-16, no twiddles
    float2 v[E];
    if ((hop & 1) == 0) {
#pragma unroll
      for (int m = 0; m < E; ++m) {
        const int e = q + TPF * m;
        const float2 s2 = *reinterpret_cast<const float2*>(fs + 2 * e);
        const float2 w2 = *reinterpret_cast<const float2*>(win + 2 * e);
        v[m] = make_float2(s2.x * w2.x, s2.y * w2.y);
      }
    } else {
#pragma unroll
      for (int m = 0; m < E; ++m) {
        const int e = q + TPF * m;
        v[m] = make_float2(fs[2 * e] * win[2 * e], fs[2 * e + 1] * win[2 * e + 1]);
      }
    }
    {
      float2 out[E];
      DFT<E, 1>::run(v, out);
#pragma unroll
      for (int t = 0; t < E; ++t) buf[buf_phys<LOG2N>(q * E + t)] = out[t];
    }
    group_sync<TPF>(grp);
    // ---- passes 1..P-1
    if constexpr (P >= 2) {
#pragma unroll
      for (int m = 0; m < E; ++m) v[m] = buf[buf_phys<LOG2N>(q + TPF * m)];
      group_sync<TPF>(grp);
      fft_pass<LOG2N, 1>(v, buf, tw, q);
      group_sync<TPF>(grp);
    }
    if constexpr (P >= 3) {
#pragma unroll
      for (int m = 0; m < E; ++m) v[m] = buf[buf_phys<LOG2N>(q + TPF * m)];
      group_sync<TPF>(grp);
      fft_pass<LOG2N, 2>(v, buf, tw, q);
      group_sync<TPF>(grp);
    }

    // ---- untangle the packed transform into the real-FFT bins k and N-k
    for (int k = q; k <= N / 2; k += TPF) {
      const float2 zk = buf[buf_phys<LOG2N>(k)];
      const float2 zn = buf[buf_phys<LOG2N>((N - k) & (N - 1))];
      const float2 xe = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));  // (Zk + conj Zn)/2
      const float2 xo = make_float2(0.5f * (zk.y + zn.y), 0.5f * (zn.x - zk.x));  // (Zk - conj Zn)/(2i)
      const float2 tt = cmul(ut[k], xo);
      const float2 xk = cadd(xe, tt);
      const float2 d = csub(xe, tt);
      const float2 xnk = make_float2(d.x, -d.y);  // conj(Xe - T)
      if (p.stft_out && live) {
        float2* o = p.stft_out + (size_t)row * F * p.n_frames + n;
        o[(size_t)k * p.n_frames] = xk;
        o[(size_t)(N - k) * p.n_frames] = xnk;
      }
      mag[k] = sqrtf(fmaf(xk.x, xk.x, xk.y * xk.y));
      mag[N - k] = sqrtf(fmaf(xnk.x, xnk.x, xnk.y * xnk.y));
    }
    group_sync<TPF>(grp);

    // ---- banded mel projection + post-op for this frame
    if (p.mel_out) {
      for (int m = q; m < p.n_mels; m += TPF) {
        const int lo = __ldg(p.mel_lo + m), hi = __ldg(p.mel_hi + m);
        const float* wrow = p.mel_fb + (size_t)m * F;
        float acc = 0.f;
        for (int k = lo; k < hi; ++k) acc = fmaf(__ldg(wrow + k), mag[k], acc);
        if (p.post == B2A_POST_LOG10) {
          float c = fmaxf(acc, p.post_eps);
          c = (p.post_power == 2.0f) ? c * c : powf(c, p.post_power);
          acc = log10f(c);
        } else if (p.post == B2A_POST_LN) {
          acc = logf(acc + p.post_eps);
        }
        melt[m * (FR + 1) + f] = acc;
      }
    }
    group_sync<TPF>(grp);
  }

  if (p.mel_out) {
    __syncthreads();
    const int nf = min(FR, p.n_frames - n0);
    float* o = p.mel_out + (size_t)row * p.n_mels * p.n_frames + n0;
    for (int i = tid; i < p.n_mels * FR; i += THREADS) {
      const int m = i / FR, f = i - m * FR;
      if (f < nf) o[(size_t)m * p.n_frames + f] = melt[m * (FR + 1) + f];
    }
  }
}

template <int LOG2N>
static int launch(Params& p, void* stream) {
  using PL = Plan<LOG2N>;
  p.span = (PL::FR - 1) * p.hop + p.n_fft;
  p.n_tiles = (p.n_frames + PL::FR - 1) / PL::FR;
  int o = align16(p.span * 4);
  p.off_win = o; o = align16(o + p.n_fft * 4);
  p.off_tw = o; o = align16(o + PL::NSLOT * PL::TPF * 8 + 16);
  p.off_ut = o; o = align16(o + (PL::N / 2 + 1) * 8);
  p.off_buf = o; o = align16(o + PL::G * PL::BUF * 8);
  p.off_mag = o; o = align16(o + PL::G * PL::MAG * 4);
  p.off_mel = o; o = align16(o + (p.mel_out ? p.n_mels * (PL::FR + 1) * 4 : 0));
  p.smem_bytes = o;
  B2A_REQUIRE(o <= 227 * 1024, B2A_E_UNSUPPORTED,
              "spectral: n_fft=%d hop=%d n_mels=%d needs %d bytes of shared memory (> 227 KB)", p.n_fft, p.hop,
              p.n_mels, o);
  B2A_REQUIRE((int64_t)p.rows * p.n_tiles < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spectral: grid too large");
  B2A_CUDA_OK(cudaFuncSetAttribute(spectral_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  B2A_LAUNCH(spectral_kernel<LOG2N>, dim3((unsigned)(p.rows * p.n_tiles)), dim3(THREADS), (size_t)o, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}


// =============================================================================================
// Warp-per-frame kernel (n_fft 64 .. 2048): the fast path.
//
// A frame of N = n_fft/2 packed complex points is owned by LPF = N/32 lanes of ONE warp, 32 points
// per lane, and transformed with two Stockham passes: radix 32, then radix LPF.  Nothing in the
// FFT crosses a warp, so there is no CTA barrier between the span load and the final tile store:
//   pass 0   32 points/lane straight from the staged span (x window), radix-32 DFT in registers
//   exchange one warp-private 32 x 32 transpose through shared memory (two float planes, stride 33:
//            conflict-free), __syncwarp only
//   pass 1   role-constant twiddles (shared memory, [slot][lane]), radix-LPF DFTs in registers;
//            the lane ends up with Z[l + LPF m], m = 0..31, in natural order
//   untangle Z[N-k] lives in lane LPF-l, register 31-m: one warp shuffle per pair, each lane
//            produces the real-FFT bins k and N-k for its 16 k < N/2
//   mel      |X| -> the (dead) exchange plane -> banded FP32 gather, post-op, tile in smem
// =============================================================================================
// MODE 0: no STFT output (mel / log-mel only: the bench path; the per-bin store code is compiled out);
// MODE 1: STFT-only launch that parks the complex frames in shared memory and writes them transposed;
// MODE 2: generic (STFT straight from registers, with or without mel).

// B2A_K1_PROBE (tests/probes/k1_phase_probe.py only): lane 0 of every warp stamps clock64() at the 11 phase boundaries
// of its first K1_PROBE_TILES tiles.  Without the macro the stamps compile to nothing.
#ifdef B2A_K1_PROBE
__device__ unsigned long long* g_k1_probe;  // [grid][8 warps][K1_PROBE_TILES][11] clock64 stamps of lane 0
#define K1_PROBE_TILES 64
#define K1_STAMP(k)                                                                                   \
  do {                                                                                                \
    if (g_k1_probe && lane == 0 && it_probe < K1_PROBE_TILES)                                         \
      g_k1_probe[(((size_t)blockIdx.x * 8 + warp) * K1_PROBE_TILES + it_probe) * 11 + (k)] = clock64(); \
  } while (0)
#else
#define K1_STAMP(k) do { } while (0)
#endif

template <int LOG2N, int MODE>
__global__ void __launch_bounds__(256, 2) spectral_warp_kernel(Params p) {
  using PL = WPlan<LOG2N>;
  constexpr bool STAGED = (MODE == 1), DIRECT = (MODE == 2);
  constexpr int N = PL::N, LPF = PL::LPF, FPW = PL::FPW, G = PL::G, FR = PL::FR;
  static_assert(FR == G && FR % 8 == 0, "one round per tile: the |X| slot of a frame is its index in the tile");
  B2A_DYN_SMEM(smem);
  float* sp = reinterpret_cast<float*>(smem);
  float* win = reinterpret_cast<float*>(smem + p.off_win);   // [n_fft]
  float2* tw = reinterpret_cast<float2*>(smem + p.off_tw);   // [NTW][LPF]
  float2* ut = reinterpret_cast<float2*>(smem + p.off_ut);   // [16][LPF]
  float* xbs = reinterpret_cast<float*>(smem + p.off_buf);   // [G][XB]
  float* mpk = reinterpret_cast<float*>(smem + p.off_mpk);
  int4* mseg = reinterpret_cast<int4*>(smem + p.off_mseg);   // (offset, lo4, n4, -)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int hop = p.hop, n_fft = 2 * N, F = N + 1;
  const int l = lane & (LPF - 1);  // lane within the frame
  const int fw = lane / LPF;       // frame within the warp
  const int total_tiles = p.rows * p.n_tiles;

  // ---- first tile's samples in flight while the (row-independent) tables are built ONCE per CTA
  int t = blockIdx.x;
  __shared__ __align__(8) unsigned long long s_bar;  // mbarrier the TMA span copies complete on
  if (tid == 0) mbar_init(&s_bar, 1);
  __syncthreads();
  bool by_tma;
  unsigned tma_parity = 0;
  {
    const int row = t / p.n_tiles, tile = t - row * p.n_tiles;
    by_tma = stage_span_async(p, sp, row,
                              (tile * FR + p.drop_edge) * hop + p.origin + (p.row_origin ? __ldg(p.row_origin + row) : 0),
                              &s_bar);
  }
  // the window is kept HALVED: the real-FFT untangle needs (Zk +- conj Zn)/2, and a power-of-two scale commutes with
  // every rounding of the (linear) transform, so the 0.5 factors vanish from the untangle with bit-identical results
  for (int i = tid; i < n_fft; i += 256) win[i] = 0.5f * __ldg(p.window + i);
  for (int i = tid; i < G * p.xb_stride; i += 256) xbs[i] = 0.f;  // the slack behind each |X| slot must stay finite (0 x w)
  warp_fft_tables<LOG2N, PL::NUT>(tw, ut);
  // banded mel weights in shared memory.  The projection runs once per tile, AFTER the tile's FFTs, with the
  // work transposed: lane (f, j) of warp w handles frame f (8 at a time) and filter m = 4*(w + 8*i) + j in
  // step i, so one 128-bit weight load is broadcast to 8 frames and the |X| loads of the 8 frames interleave
  // conflict-free.  Row m = its 4-aligned band [lo4, lo4 + 4*n4), zero padded to the widest of the 4 CONSECUTIVE
  // filters of its (warp, step) so that all lanes of a warp run the same trip count (neighbouring filters have
  // nearly equal widths: 6 % padding at 44.1 kHz / 2048 / 128 against 49 % when a step took every 8th filter).
  const bool packed = p.mel_out && p.mel_packed_len > 0;
  __shared__ int s_clamp;
  if (packed) {
    for (int m = tid; m < p.n_mels; m += 256) {
      const int lo4 = __ldg(p.mel_lo + m) & ~3;
      int n4 = (((__ldg(p.mel_hi + m) + 3) & ~3) - lo4) >> 2;
      mseg[m] = make_int4(0, lo4, n4 < 0 ? 0 : n4, 0);
    }
    __syncthreads();
    if (tid == 0) {  // offsets (float4 units) and padded widths
      int run = 0, reach = 0;
      for (int w = 0; w < 8; ++w)
        for (int i = 0; 4 * (w + 8 * i) < p.n_mels; ++i) {
          int mx = 0;
          for (int j = 0; j < 4; ++j) { const int m = 4 * (w + 8 * i) + j; if (m < p.n_mels) mx = max(mx, mseg[m].z); }
          mx = (mx + 1) & ~1;  // even width: the projection loop is unrolled by two without a remainder
          for (int j = 0; j < 4; ++j) {
            const int m = 4 * (w + 8 * i) + j;
            if (m < p.n_mels) { mseg[m].x = run; mseg[m].w = mx; run += mx; reach = max(reach, mseg[m].y + 4 * mx); }
          }
        }
      s_clamp = reach > PL::XB;  // a zero-padded row would read past its frame's |X| slot: clamp the index
    }
    __syncthreads();
    for (int m = warp; m < p.n_mels; m += 8) {
      const int4 sg = mseg[m];
      const float* wrow = p.mel_fb + (size_t)m * F;
      for (int i = lane; i < 4 * sg.w; i += 32) {
        const int k = sg.y + i;
        mpk[4 * sg.x + i] = (i < 4 * sg.z && k < F) ? __ldg(wrow + k) : 0.f;
      }
    }
  }

  float* xb = xbs + (warp * FPW + fw) * p.xb_stride;
  const int src_lane = partner_lane<LPF>(lane);  // holder of Z[N - k]

#ifdef B2A_K1_PROBE
  int it_probe = 0;
#endif
  bool first = true;
#pragma unroll 1
  for (; t < total_tiles; t += gridDim.x) {
    const int row = t / p.n_tiles, tile = t - row * p.n_tiles;
    const int n0 = tile * FR;
    const int ws = (n0 + p.drop_edge) * hop + p.origin + (p.row_origin ? __ldg(p.row_origin + row) : 0);
    const float g = p.gain ? __ldg(p.gain + row / p.rows_per_gain) : 1.0f;
    const float ga = fabsf(g);
    K1_STAMP(0);
    // this tile's span was issued by the previous iteration (or the prologue)
    if (by_tma) { mbar_wait(&s_bar, tma_parity); tma_parity ^= 1u; }
    K1_STAMP(1);
    // a TMA span is visible to each thread once its wait returns; a span staged with plain stores (and, on the first
    // tile, the tables) needs the CTA barrier.  Nothing else is ordered here: the |X| slots the previous tile's mel
    // phase reads are rewritten only after this tile's barrier before its TMA issue.  (The simulator's copy is
    // synchronous and its wait a no-op, so there the barrier is what orders the copy before the reads.)
#ifdef B2A_SIM
    __syncthreads();
#else
    if (!by_tma || first) __syncthreads();
#endif
    first = false;
    K1_STAMP(2);
    if (p.y_out) writeback_scaled(p, sp, row, tile, n0, FR, ws, g);  // (sp is re-filled only after the barrier
                                                                      //  inside the last round, below)
    K1_STAMP(3);

#pragma unroll 1
    for (int rd = 0; rd < FR / G; ++rd) {
      const int f = rd * G + warp * FPW + fw;
      const int n = n0 + f;
      const bool live = n < p.n_frames;
      const float* fs = sp + f * hop;

      // ---- windowed frame with the first radix-32 butterfly fused in
      float2 z[32];
      load_frame<LOG2N>(fs, win, hop, z, l);
      K1_STAMP(4);
      if (rd == FR / G - 1) {
        // every warp holds its last frame in registers: the span buffer is dead, so the next tile's
        // samples stream in (one TMA bulk copy) underneath this round's FFTs and mel projection
        __syncthreads();
        const int tn = t + gridDim.x;
        by_tma = false;
        if (tn < total_tiles) {
          const int rown = tn / p.n_tiles, tilen = tn - rown * p.n_tiles;
          by_tma = stage_span_async(
              p, sp, rown, (tilen * FR + p.drop_edge) * hop + p.origin + (p.row_origin ? __ldg(p.row_origin + rown) : 0),
              &s_bar);
        }
      }
      K1_STAMP(5);
      warp_fft<LOG2N, true>(z, xb, tw, l);  // z[m] = Z[l + LPF m]

      // ---- untangle -> real-FFT bins k = l + LPF m (m < 16) and N - k ; magnitudes into xb
      const float2 u0 = ut[l];  // exp(-i pi l / N): the lane's base untangle twiddle (the only table entry when lean)
      float2* so = (DIRECT && p.stft_out) ? p.stft_out + (size_t)row * F * p.n_frames + n : nullptr;
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const float2 zk = z[m];
        float2 zn;
        zn.x = __shfl_sync(0xffffffffu, z[31 - m].x, src_lane);
        zn.y = __shfl_sync(0xffffffffu, z[31 - m].y, src_lane);
        if (l == 0) zn = z[(32 - m) & 31];
        const int k = l + LPF * m;
        const float2 xe = add2(zk, make_float2(zn.x, -zn.y));               // (Zk + conj Zn)/2   (window halved above)
        const float2 xo = add2(make_float2(zk.y, -zk.x), make_float2(zn.y, zn.x));  // (Zk - conj Zn)/(2i)
        // X[k] = Xe + W Xo, X[N-k]* = Xe - W Xo: a twiddled butterfly, fused like the ones of the transform
        const float2 w = untangle_twiddle_m<LOG2N>(ut, u0, l, m);
        const float2 xk = fma2(bcast2(w.x), xo, fma2(make_float2(-w.y, w.y), make_float2(xo.y, xo.x), xe));
        const float2 d = fma2(bcast2(2.0f), xe, neg2(xk));
        if constexpr (STAGED) {  // park the complex bins in the frame's own slot (the exchange plane is dead now)
          float2* xc = reinterpret_cast<float2*>(xb);
          xc[k] = make_float2(g * xk.x, g * xk.y);
          xc[N - k] = make_float2(g * d.x, -g * d.y);
        } else {
          if constexpr (DIRECT) {
            if (so && live) {
              so[(size_t)k * p.n_frames] = make_float2(g * xk.x, g * xk.y);
              so[(size_t)(N - k) * p.n_frames] = make_float2(g * d.x, -g * d.y);
            }
          }
          xb[k] = fast_sqrt(fmaf(xk.x, xk.x, xk.y * xk.y));
          xb[N - k] = fast_sqrt(fmaf(d.x, d.x, d.y * d.y));
        }
      }
      if (l == 0) {  // k = N/2 pairs with itself: X = conj(Z[N/2])
        const float2 zh = make_float2(2.0f * z[16].x, 2.0f * z[16].y);  // undo the halved window: X = conj(Z[N/2])
        if constexpr (STAGED) {
          reinterpret_cast<float2*>(xb)[N / 2] = make_float2(g * zh.x, -g * zh.y);
        } else {
          if constexpr (DIRECT) {
            if (so && live) so[(size_t)(N / 2) * p.n_frames] = make_float2(g * zh.x, -g * zh.y);
          }
          xb[N / 2] = fast_sqrt(fmaf(zh.x, zh.x, zh.y * zh.y));
          xb[N + 1] = 0.f; xb[N + 2] = 0.f; xb[N + 3] = 0.f;  // read (x 0 weight) by 4-wide band loads
        }
      }
      __syncwarp();

    }
    K1_STAMP(6);

    // ---- mel phase of the tile: |X| of all FR frames sit in the xb slots (slot = frame within the tile)
    //      Each lane stores its cells straight from registers: the 8 lanes of a filter write 8 consecutive frames (the
    //      same 32-byte runs a staged tile store would write), so no tile buffer, and no barrier after the projection:
    //      the next tile's barrier before its TMA issue already orders these |X| reads before the slots are rewritten.
    const int nf = min(FR, p.n_frames - n0);
    float* mo = p.mel_out ? p.mel_out + (size_t)row * p.n_mels * p.n_frames + n0 : nullptr;
    if (p.mel_out) {
      __syncthreads();
      K1_STAMP(7);
      const int fl = lane & 7, jq = lane >> 3;
      const float lscale = p.post_power * 0.30102999566398120f;  // log10(c^power) = power * log10(2) * log2(c)
      if (packed) {
        const float4* mpk4 = reinterpret_cast<const float4*>(mpk);
        for (int fc = 0; fc < FR; fc += 8) {
          const int f = fc + fl;
          const float* xf = xbs + f * p.xb_stride;
          if (!s_clamp) {  // the padded rows stay inside the frame's |X| slot (always, for the stock filterbanks)
            for (int mm = 4 * warp + jq; mm < p.n_mels; mm += 32) {
              const int4 sg = mseg[mm];  // (row offset, lo4, own n4, padded even n4: the same for the 4 filters of a step)
              const float4* w4 = mpk4 + sg.x;
              const float4* v4 = reinterpret_cast<const float4*>(xf + sg.y);
              float2 a01 = make_float2(0.f, 0.f), a23 = a01;  // packed accumulator pairs (fma on (re, im) pairs)
              for (int it = 0; it < sg.w; it += 2) {
                const float4 wa = w4[it], wb = w4[it + 1], va = v4[it], vb = v4[it + 1];
                a01 = fma2(make_float2(wa.x, wa.y), make_float2(va.x, va.y), a01);
                a23 = fma2(make_float2(wb.x, wb.y), make_float2(vb.x, vb.y), a23);
                a01 = fma2(make_float2(wa.z, wa.w), make_float2(va.z, va.w), a01);
                a23 = fma2(make_float2(wb.z, wb.w), make_float2(vb.z, vb.w), a23);
              }
              float acc = ((a01.x + a01.y) + (a23.x + a23.y)) * ga;
              if (p.post == B2A_POST_LOG10) acc = lscale * fast_log2(fmaxf(acc, p.post_eps));
              else if (p.post == B2A_POST_LN) acc = logf(acc + p.post_eps);
              if (f < nf) mo[(size_t)mm * p.n_frames + f] = acc;
            }
          } else {  // a zero-padded row would read past the slot: clamp the index
            const int lim = PL::XB - 4;
            for (int mm = 4 * warp + jq; mm < p.n_mels; mm += 32) {
              const int4 sg = mseg[mm];
              const float4* w4 = mpk4 + sg.x;
              float a0 = 0.f, a1 = 0.f;
              for (int it = 0; it < sg.w; ++it) {
                const float4 w = w4[it];
                const float4 v = *reinterpret_cast<const float4*>(xf + min(sg.y + 4 * it, lim));
                a0 = fmaf(w.x, v.x, a0); a1 = fmaf(w.y, v.y, a1);
                a0 = fmaf(w.z, v.z, a0); a1 = fmaf(w.w, v.w, a1);
              }
              float acc = (a0 + a1) * ga;
              if (p.post == B2A_POST_LOG10) acc = lscale * fast_log2(fmaxf(acc, p.post_eps));
              else if (p.post == B2A_POST_LN) acc = logf(acc + p.post_eps);
              if (f < nf) mo[(size_t)mm * p.n_frames + f] = acc;
            }
          }
        }
      } else {  // band table does not fit in shared memory: weights from global
        for (int fc = 0; fc < FR; fc += 8) {
          const int f = fc + fl;
          const float* xf = xbs + f * p.xb_stride;
          for (int mm = 4 * warp + jq; mm < p.n_mels; mm += 32) {
            float acc = mel_band(p.mel_fb, p.mel_lo, p.mel_hi, F, mm, xf) * ga;
            if (p.post == B2A_POST_LOG10) acc = lscale * fast_log2(fmaxf(acc, p.post_eps));
            else if (p.post == B2A_POST_LN) acc = logf(acc + p.post_eps);
            if (f < nf) mo[(size_t)mm * p.n_frames + f] = acc;
          }
        }
      }
    }

    K1_STAMP(8);
    if constexpr (STAGED) {
      __syncthreads();  // all frames of the tile are parked in their slots
      // transposed write of the tile's complex frames: 32 lanes = 32/FR bins x FR consecutive frames, i.e. runs of
      // FR * 8 bytes instead of one 8-byte store per sector (the layout is [rows, F, n_frames], frame fastest)
      const int nf = min(FR, p.n_frames - n0);
      float2* o = p.stft_out + (size_t)row * F * p.n_frames + n0;
      for (int i = tid; i < F * FR; i += 256) {
        const int k = i / FR, f = i - k * FR;
        if (f < nf) o[(size_t)k * p.n_frames + f] = reinterpret_cast<const float2*>(xbs + f * p.xb_stride)[k];
      }
      // (the next iteration's barrier, after its span wait, orders these reads before the slots are reused)
    }
    K1_STAMP(9);
    K1_STAMP(10);
#ifdef B2A_K1_PROBE
    ++it_probe;
#endif
  }
}

#ifdef B2A_K1_PROBE
static int g_k1_last[3];  // occupancy (CTAs / SM), grid and dynamic shared memory of the last n_fft 2048 mel launch
#endif

template <int LOG2N>
static int launch_warp(Params& p, void* stream) {
  using PL = WPlan<LOG2N>;
  p.span = (PL::FR - 1) * p.hop + p.n_fft;
  p.n_tiles = (p.n_frames + PL::FR - 1) / PL::FR;
  int o = align16(p.span * 4);
  p.off_win = o; o = align16(o + p.n_fft * 4);
  p.off_tw = o; o = align16(o + PL::NTW * PL::LPF * 8 + 16);
  p.off_ut = o; o = align16(o + PL::NUT * PL::LPF * 8);
  // STFT-only launches park the complex frame (N+1 float2) in the frame's slot and write it out transposed; that
  // needs 2N+4 floats per slot instead of XB -- only if two CTAs per SM still fit
  p.xb_stride = PL::XB;
  p.stage_stft = 0;
  if (p.stft_out && !p.mel_out) {
    const int wide = ((2 * PL::N + 4 + 3) / 4) * 4;
    if (wide >= PL::XB && o + PL::G * wide * 4 + 64 <= 112 * 1024) { p.xb_stride = wide; p.stage_stft = 1; }
  }
  p.off_buf = o; o = align16(o + PL::G * p.xb_stride * 4);
  p.off_mag = o;
  p.off_mel = o;  // (mel cells are stored from registers: no tile buffer)
  const int base = o;
  p.off_mpk = o; p.off_mseg = o;
  if (p.mel_out && p.mel_packed_len > 0) {
    p.off_mpk = o; o = align16(o + p.mel_packed_len * 4);
    p.off_mseg = o; o = align16(o + p.n_mels * 16);
    if (o > 227 * 1024) { o = base; p.mel_packed_len = 0; }  // does not fit: read the weights from global
  }
  p.smem_bytes = o;
  B2A_REQUIRE(o <= 227 * 1024, B2A_E_UNSUPPORTED,
              "spectral: n_fft=%d hop=%d n_mels=%d needs %d bytes of shared memory (> 227 KB)", p.n_fft, p.hop,
              p.n_mels, o);
  const int64_t total = (int64_t)p.rows * p.n_tiles;
  B2A_REQUIRE(total < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spectral: too many tiles");
  auto kern = p.stage_stft ? spectral_warp_kernel<LOG2N, 1>
                           : (p.stft_out ? spectral_warp_kernel<LOG2N, 2> : spectral_warp_kernel<LOG2N, 0>);
  B2A_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  // persistent: as many CTAs as are resident at once (2 per SM by registers / shared memory), each loops over tiles
  int64_t grid;
  const int rc = persistent_grid(kern, o, total, &grid);
  if (rc != B2A_OK) return rc;
#ifdef B2A_K1_PROBE
  if (LOG2N == 10 && !p.stft_out) {
    B2A_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&g_k1_last[0], kern, 256, (size_t)o));
    g_k1_last[1] = (int)grid; g_k1_last[2] = o;
  }
#endif
  B2A_LAUNCH(kern, dim3((unsigned)grid), dim3(256), (size_t)o, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// raw-framing forward FFT of blocks (the FFT convolution, the inverse STFT's backward): out[rows, F, n_frames]
int frames_fft(const float* x, int rows, int T, int n_fft, int hop, const float* window, int origin,
               const int32_t* row_origin, int pad_mode, int n_frames, float2* out, void* stream) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.window = window; p.stft_out = out;
  p.rows = rows; p.T = T; p.n_fft = n_fft; p.hop = hop; p.pad_mode = pad_mode; p.n_frames = n_frames;
  p.rows_per_gain = 1; p.center = 0; p.origin = origin; p.row_origin = row_origin;
  switch (n_fft) {
    case 64: return launch_warp<5>(p, stream);
    case 128: return launch_warp<6>(p, stream);
    case 256: return launch_warp<7>(p, stream);
    case 512: return launch_warp<8>(p, stream);
    case 1024: return launch_warp<9>(p, stream);
    case 2048: return launch_warp<10>(p, stream);
  }
  return b2a::fail(B2A_E_UNSUPPORTED, "frames_fft: block size %d", n_fft);
}

int check_framing(const char* who, int64_t T, int n_fft, int hop, int pad, int right_pad, int pad_mode, int drop_edge,
                  int64_t* n_frames) {
  B2A_REQUIRE(pad >= 0 && right_pad >= 0 && drop_edge >= 0, B2A_E_INVALID, "%s: negative padding", who);
  B2A_REQUIRE(pad_mode >= 0 && pad_mode <= 2, B2A_E_UNSUPPORTED, "%s: pad mode %d", who, pad_mode);
  const int64_t Lp = T + 2 * (int64_t)pad + right_pad;
  // torch raises for these (reflect padding wider than the signal)
  B2A_REQUIRE(n_fft / 2 < Lp, B2A_E_INVALID, "%s: n_fft/2 (%d) must be < padded length (%lld)", who, n_fft / 2,
              (long long)Lp);
  B2A_REQUIRE(pad_mode != B2A_PAD_REFLECT || (pad + right_pad) < T || (pad + right_pad) == 0, B2A_E_INVALID,
              "%s: reflect padding (%d) must be < signal length (%lld)", who, pad + right_pad, (long long)T);
  *n_frames = b2a_stft_num_frames(T, n_fft, hop, pad, right_pad, drop_edge);
  B2A_REQUIRE(*n_frames >= 1, B2A_E_INVALID, "%s: no frames", who);
  return B2A_OK;
}

}  // namespace spectral
}  // namespace b2a

extern "C" int64_t b2a_stft_num_frames(int64_t T, int n_fft, int hop, int pad, int right_pad, int drop_edge) {
  if (T < 1 || n_fft < 2 || hop < 1 || pad < 0 || right_pad < 0 || drop_edge < 0) return -1;
  // torch.stft(center=True): 1 + (len + 2*(n_fft/2) - n_fft) / hop  with len = T + 2 pad + right_pad
  // (an odd window length loses one sample: 2*(n_fft/2) - n_fft = -(n_fft & 1))
  int64_t n = 1 + (T + 2 * (int64_t)pad + right_pad - (n_fft & 1)) / hop - 2 * (int64_t)drop_edge;
  return n;
}

// The one route table (include/b2a.h).  Each family's entry points keep their own, wider or equal, range checks.
extern "C" int b2a_stft_route(int n_fft, int hop, int inverse) {
  if (n_fft < 2 || hop < 1 || (inverse && hop > n_fft)) return B2A_ROUTE_NONE;
  if ((n_fft & (n_fft - 1)) == 0) {
    if (n_fft >= (inverse ? 64 : 32) && n_fft <= (inverse ? 2048 : 4096)) return B2A_ROUTE_FFT;
    if (n_fft >= 4096 && n_fft <= 32768) return B2A_ROUTE_LARGE;
  }
  return n_fft <= 8192 ? B2A_ROUTE_DENSE : B2A_ROUTE_NONE;
}

// b2a_spectral_f32 on B2A_ROUTE_FFT: everything in one launch of the fused kernel.
static int spectral_fft(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window, int pad,
                        int right_pad, int pad_mode, int drop_edge, const float* gain, int rows_per_gain, float* y_out,
                        const float* mel_fb, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels,
                        int mel_packed_len, int post, float post_eps, float post_power, float* mel_out,
                        float* stft_out, void* stream) {
  using namespace b2a::spectral;
  B2A_REQUIRE(x && window, B2A_E_INVALID, "spectral: null x/window");
  B2A_REQUIRE(mel_out || stft_out, B2A_E_INVALID, "spectral: neither mel_out nor stft_out requested");
  B2A_REQUIRE(rows >= 1 && T >= 1, B2A_E_INVALID, "spectral: empty input");
  B2A_REQUIRE(T < (int64_t)1 << 30, B2A_E_UNSUPPORTED, "spectral: rows longer than 2^30 samples");
  B2A_REQUIRE(n_fft >= 32 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0, B2A_E_UNSUPPORTED,
              "spectral: window_length must be a power of two in [32, 4096] (got %d)", n_fft);
  B2A_REQUIRE(hop >= 1, B2A_E_INVALID, "spectral: hop_length must be >= 1");
  int64_t nfr;
  const int rc = check_framing("spectral", T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(!y_out || (pad == 0 && right_pad == 0 && drop_edge == 0), B2A_E_UNSUPPORTED,
              "spectral: y_out needs pad == right_pad == drop_edge == 0");
  B2A_REQUIRE(!gain || rows_per_gain >= 1, B2A_E_INVALID, "spectral: rows_per_gain");
  B2A_REQUIRE(!mel_out || (mel_fb && mel_lo && mel_hi && n_mels >= 1), B2A_E_INVALID, "spectral: mel arguments");
  B2A_REQUIRE(post >= 0 && post <= 2, B2A_E_INVALID, "spectral: post-op %d", post);
  Params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.window = window; p.gain = gain; p.y_out = y_out;
  p.mel_fb = mel_fb; p.mel_lo = mel_lo; p.mel_hi = mel_hi; p.mel_out = mel_out;
  p.stft_out = reinterpret_cast<float2*>(stft_out);
  p.rows = (int)rows; p.T = (int)T; p.n_fft = n_fft; p.hop = hop; p.pad = pad; p.right_pad = right_pad;
  p.pad_mode = pad_mode; p.drop_edge = drop_edge; p.n_frames = (int)nfr; p.n_mels = n_mels;
  p.mel_packed_len = (mel_out && mel_packed_len > 0) ? mel_packed_len : 0;
  p.center = 1; p.origin = -(n_fft / 2) - pad; p.row_origin = nullptr;
  p.rows_per_gain = gain ? rows_per_gain : 1; p.post = post; p.post_eps = post_eps; p.post_power = post_power;
  switch (n_fft) {
    case 32: return launch<4>(p, stream);
    case 64: return launch_warp<5>(p, stream);
    case 128: return launch_warp<6>(p, stream);
    case 256: return launch_warp<7>(p, stream);
    case 512: return launch_warp<8>(p, stream);
    case 1024: return launch_warp<9>(p, stream);
    case 2048: return launch_warp<10>(p, stream);
    case 4096: return launch<11>(p, stream);  // 64 lanes per frame: CTA-cooperative kernel
  }
  return b2a::fail(B2A_E_UNSUPPORTED, "spectral: n_fft %d", n_fft);
}

extern "C" size_t b2a_spectral_workspace_bytes(int64_t rows, int64_t T, int n_fft, int hop, int pad, int right_pad,
                                                int drop_edge, int stft_scratch, int scaled_scratch) {
  const int r = b2a_stft_route(n_fft, hop, 0);
  const int64_t nfr = b2a_stft_num_frames(T, n_fft, hop, pad, right_pad, drop_edge);
  if (rows < 1 || nfr < 1 || r == B2A_ROUTE_NONE || r == B2A_ROUTE_FFT) return 0;
  size_t bytes = 0;
  if (stft_scratch) bytes += (size_t)rows * (size_t)(n_fft / 2 + 1) * (size_t)nfr * 2 * sizeof(float);
  if (scaled_scratch) bytes += (size_t)rows * (size_t)T * sizeof(float);
  return bytes;
}

// b2a_spectral_f32 on B2A_ROUTE_LARGE / DENSE: the gain pass, the STFT of all frames, then the mel from that STFT.
// The outputs the caller did not ask for go to ws: the STFT at its start, the scaled signal after it.
static int spectral_materialised(int route, const float* x, int64_t rows, int64_t T, int n_fft, int hop,
                                 const float* window, const float* matrix, int pad, int right_pad, int pad_mode,
                                 int drop_edge, const float* gain, int rows_per_gain, float* y_out,
                                 const float* mel_fb, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels,
                                 int post, float post_eps, float post_power, float* mel_out, float* stft_out,
                                 void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(mel_out || stft_out, B2A_E_INVALID, "spectral: neither mel_out nor stft_out requested");
  // the framing is checked before the gain pass, with the message the STFT's own check gives
  int64_t nfr;
  int rc = b2a::spectral::check_framing(route == B2A_ROUTE_LARGE ? "stft_large" : "stft_dense", T, n_fft, hop, pad,
                                        right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  const size_t need = b2a_spectral_workspace_bytes(rows, T, n_fft, hop, pad, right_pad, drop_edge, !stft_out,
                                                   gain && !y_out);
  B2A_REQUIRE(ws_bytes >= need && (ws || need == 0), B2A_E_INVALID, "spectral: workspace too small");
  B2A_REQUIRE(((uintptr_t)ws & 7) == 0, B2A_E_INVALID, "spectral: workspace must be 8-byte aligned");
  const int F = n_fft / 2 + 1;
  char* scratch = static_cast<char*>(ws);
  float* stft = stft_out;
  if (!stft) {
    stft = reinterpret_cast<float*>(scratch);
    scratch += (size_t)rows * F * (size_t)nfr * 2 * sizeof(float);
  }
  if (gain) {
    B2A_REQUIRE(rows_per_gain >= 1 && rows % rows_per_gain == 0, B2A_E_INVALID, "spectral: rows_per_gain");
    float* scaled = y_out ? y_out : reinterpret_cast<float*>(scratch);
    rc = b2a_gain_f32(x, scaled, rows / rows_per_gain, rows_per_gain * T, gain, stream);
    if (rc != B2A_OK) return rc;
    x = scaled;
  }
  rc = route == B2A_ROUTE_LARGE
           ? b2a::large::stft(x, rows, T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge, stft, stream)
           : b2a::dft::stft(x, rows, T, n_fft, hop, matrix, pad, right_pad, pad_mode, drop_edge, stft, stream);
  if (rc != B2A_OK || !mel_out) return rc;
  return b2a::dft::mel_from_stft(stft, rows, F, nfr, mel_fb, mel_lo, mel_hi, n_mels, post, post_eps, post_power,
                                 mel_out, stream);
}

extern "C" int b2a_spectral_f32(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window,
                                const float* matrix, int pad, int right_pad, int pad_mode, int drop_edge,
                                const float* gain, int rows_per_gain, float* y_out, const float* mel_fb,
                                const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, int mel_packed_len, int post,
                                float post_eps, float post_power, float* mel_out, float* stft_out, void* ws,
                                size_t ws_bytes, void* stream) {
  const int route = b2a_stft_route(n_fft, hop, 0);
  if (route == B2A_ROUTE_FFT)
    return spectral_fft(x, rows, T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge, gain, rows_per_gain, y_out,
                        mel_fb, mel_lo, mel_hi, n_mels, mel_packed_len, post, post_eps, post_power, mel_out, stft_out,
                        stream);
  if (route == B2A_ROUTE_LARGE || route == B2A_ROUTE_DENSE)
    return spectral_materialised(route, x, rows, T, n_fft, hop, window, matrix, pad, right_pad, pad_mode, drop_edge,
                                 gain, rows_per_gain, y_out, mel_fb, mel_lo, mel_hi, n_mels, post, post_eps, post_power,
                                 mel_out, stft_out, ws, ws_bytes, stream);
  return b2a::fail(B2A_E_UNSUPPORTED,
                   "spectral: n_fft=%d hop=%d (hop >= 1; powers of two up to 32768, any other length up to 8192)",
                   n_fft, hop);
}

extern "C" int b2a_spectral_tc_enable(int on) {
  if (on == 0) return 0;
  return b2a::fail(B2A_E_UNSUPPORTED,
                   "spectral_tc_enable: the tensor-core spectral kernel was removed; the FP32 kernel runs every launch");
}

#ifdef B2A_K1_PROBE
// Phase-clock probe of spectral_warp_kernel<10, *> (tests/probes/k1_phase_probe.py): not part of include/b2a.h and
// compiled only with -DB2A_K1_PROBE.  `buf` (device, or null to stop recording): [grid][8][K1_PROBE_TILES][11] u64.
extern "C" int b2a_k1_probe_set(void* buf) {
  B2A_CUDA_OK(cudaMemcpyToSymbol(b2a::spectral::g_k1_probe, &buf, sizeof(buf)));
  return B2A_OK;
}
extern "C" int b2a_k1_probe_tiles() { return K1_PROBE_TILES; }
// (occupancy in CTAs per SM, grid, dynamic shared memory bytes) of the last n_fft 2048 mel launch
extern "C" void b2a_k1_probe_last(int* out) {
  for (int i = 0; i < 3; ++i) out[i] = b2a::spectral::g_k1_last[i];
}
#endif
