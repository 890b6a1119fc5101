// istft.cu -- inverse STFT on sm_90a: spectra -> inverse real FFT -> window -> overlap-add -> / envelope.
//
// Replaces AudioSignal.istft (ref:audiotools/core/audio_signal.py:1214-1296), i.e. torch.istft(center=True,
// onesided, window of n_fft samples):
//     y[t]   = sum_n  w[t - n hop] * irfft(X[:, n])[t - n hop]        (t - n hop in [0, n_fft))
//     env[t] = sum_n  w[t - n hop]^2
//     out[i] = y[start + i] / env[start + i]   for start + i < expected = (N-1) hop + n_fft,  else 0
// with N frames (match_stride puts `pad_frames` zero frames back on either side, :1276-1279; they count in the
// envelope exactly as in torch) and start = n_fft/2 (+ the match_stride trim).
//
// One persistent kernel, no intermediate in HBM (torch materialises the [rows, N, n_fft] frame tensor, folds it,
// folds the window and divides: 4 passes over 4x the signal):
//   * a CTA owns a run of consecutive frame groups of one row (a "segment"); a group is G = 8 * FPW frames, one
//     frame per LPF = n_fft/64 lanes of a warp (fft_warp.cuh, the forward kernel's transform run on conj input);
//   * the group's spectra are staged into shared memory with frame-contiguous global reads (the layout is
//     [rows, F, N], frame fastest), each frame slot is then consumed by its own lanes only, reused as the FFT's
//     exchange plane and finally holds the windowed frame;
//   * the overlap-add is a gather: a thread owns residues r mod hop and walks the hop index, summing the
//     <= ceil(n_fft/hop) slots that cover a sample plus the carry of the previous group (samples that later
//     frames still touch are carried in shared memory, double buffered); finished samples are divided by the
//     envelope (recomputed from the window: <= ceil(n_fft/hop) terms) and written once, coalesced.
//   * a segment starts `warm` groups early with a zero carry so that segments are independent (redundancy
//     (R-1)/(seg_groups*G) frames); the work list is sized to ~4 items per resident CTA.
// Bytes: read spectra 8 F N + write 4 T per row -- the algorithmic minimum.
#include "b2a_common.h"
#include "fft_warp.cuh"
#include "grad_internal.h"

namespace b2a {
namespace istft {

using namespace b2a::spectral;

struct Params {
  const float2* spec;   // [rows, N+1, n_frames]
  const float* window;  // [n_fft]
  float* out;           // [rows, out_len]
  int rows, n_frames, pad_frames, hop;
  int adjoint;          // 1: the STFT's adjoint (bin weights 1, no envelope division), see b2a::istft::run
  int groups_total;     // groups that cover every sample below `expected`
  int seg_groups, segs_per_row, warm;
  long long start, out_len, expected;
  int off_tw, off_ut, off_win, off_carry, off_reg, FS;
};

template <int LOG2N>
__global__ void __launch_bounds__(256, 2) istft_kernel(const Params p) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N, LPF = PL::LPF, FPW = PL::FPW, G = 8 * FPW, NFFT = 2 * N;
  B2A_DYN_SMEM(smem);
  float2* tw = reinterpret_cast<float2*>(smem + p.off_tw);
  float2* ut = reinterpret_cast<float2*>(smem + p.off_ut);
  float* win = reinterpret_cast<float*>(smem + p.off_win);
  float* carry = reinterpret_cast<float*>(smem + p.off_carry);  // [2][NFFT]
  float* reg = reinterpret_cast<float*>(smem + p.off_reg);      // [G][FS]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int FS = p.FS, hop = p.hop;
  warp_fft_tables<LOG2N>(tw, ut);
  for (int i = tid; i < NFFT; i += 256) win[i] = __ldg(p.window + i);
  __syncthreads();
  const int NP = p.n_frames + 2 * p.pad_frames;  // frames incl. the zero frames of match_stride
  const int g_own = warp * FPW + lane / LPF, l = lane % LPF;
  float* slot = reg + g_own * FS;
  // 1/N of the transform and the 1/2 of the even/odd split; the adjoint wants sum_k Re(G_k e^{i theta}) = n_fft/2 times
  // the inverse of the DC / Nyquist-doubled spectrum
  const float inv_n = p.adjoint ? 0.5f : 0.5f / (float)N;
  const int src_lane = partner_lane<LPF>(lane);  // holder of the partner element N - k
  const int tail = NFFT - hop;                   // samples a group hands to the next one
  const int items = p.rows * p.segs_per_row;
  // gather roles: RL residue lanes x QL hop lanes (hop >= 256: every thread owns residues and walks all hops)
  const int RL = hop < 256 ? hop : 256, QL = 256 / RL;
  const int r_first = tid < RL * QL ? tid % RL : hop, q_first = tid / RL;
  const bool vec4 = (hop & 3) == 0 && (FS & 3) == 0;
  const int RL4 = (hop >> 2) < 256 ? max(hop >> 2, 1) : 256, QL4 = 256 / RL4;
  const int r4_first = tid < RL4 * QL4 ? tid % RL4 : hop, q4_first = tid / RL4;
#pragma unroll 1
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int row = item / p.segs_per_row, seg = item - row * p.segs_per_row;
    const int gs = seg * p.seg_groups;
    const int ge = min(gs + p.seg_groups, p.groups_total);
    const int gw = max(gs - p.warm, 0);
    const float2* srow = p.spec + (size_t)row * (size_t)(N + 1) * (size_t)p.n_frames;
    float* orow = p.out + (size_t)row * (size_t)p.out_len;
    for (int i = tid; i < NFFT; i += 256) carry[i] = 0.f;
    int cur = 0;
#pragma unroll 1
    for (int gidx = gw; gidx < ge; ++gidx) {
      const int g0 = gidx * G;  // first frame (padded numbering) of the group
      __syncthreads();          // previous group's gather is done with the slots; carry[cur] is complete
      // ---- 1. spectra of frames g0 .. g0+G-1 -> slots (frame-contiguous global reads)
      for (int i = tid; i < (N + 1) * G; i += 256) {
        const int k = i / G, g = i - k * G;
        const int n = g0 + g - p.pad_frames;
        float2 v = make_float2(0.f, 0.f);
        if (n >= 0 && n < p.n_frames) v = __ldg(srow + (size_t)k * p.n_frames + n);
        if (k == 0 || k == N) {
          v.y = 0.f;  // a C2R transform ignores the imaginary parts of DC and Nyquist
          if (p.adjoint) v.x *= 2.f;  // weight 1 on every bin: DC / Nyquist get 2x the 1/2 of the interior pairs
        }
        reinterpret_cast<float2*>(reg + g * FS)[k] = v;
      }
      __syncthreads();
      // ---- 2. Z[e] = Xe[e] + i Xo[e] from the bins X[e], X[N-e]; inverse = conj(FFT(conj Z))/N.  e = l + LPF m.
      //      A pair (k, N-k), k = l + LPF m < N/2, yields both Z[k] (this lane, register m) and Z[N-k], which lives in
      //      lane (LPF - l), register 31 - m (lane 0: itself, register 32 - m): computed once, handed over by shuffle.
      //      The common factor 1/2 of Xe, Xo is folded into the final scale (exact: a power of two).
      const bool live = (g0 + g_own - p.pad_frames >= 0) && (g0 + g_own - p.pad_frames < p.n_frames);
      float2 z[32];
      {
        const float2* S = reinterpret_cast<const float2*>(slot);
        float2 pb[16];  // conj(Z[N-k]) of pair m
#pragma unroll
        for (int m = 0; m < 16; ++m) {
          const int k = l + LPF * m;
          const float2 xk = S[k], xn = S[N - k];
          const float2 xe = make_float2(xk.x + xn.x, xk.y - xn.y);  // 2 Xe
          const float2 tt = make_float2(xk.x - xn.x, xk.y + xn.y);
          const float2 w = ut[k];                                   // exp(-i pi k / N)
          const float2 xo = make_float2(fmaf(w.x, tt.x, w.y * tt.y), fmaf(w.x, tt.y, -w.y * tt.x));  // 2 Xo = conj(w) tt
          z[m] = make_float2(xe.x - xo.y, -(xe.y + xo.x));          // conj(Xe + i Xo)
          pb[m] = make_float2(xe.x + xo.y, xe.y - xo.x);            // conj(conj Xe + i conj Xo)
        }
        float2 zh;  // element N/2 (lane 0, register 16): k = N/2 pairs with itself, w = -i
        {
          const float2 xh = S[N / 2];
          const float2 xe = make_float2(2.0f * xh.x, 0.f), tt = make_float2(0.f, 2.0f * xh.y);
          const float2 xo = make_float2(-tt.y, tt.x);               // conj(-i) tt = i tt
          zh = make_float2(xe.x - xo.y, -(xe.y + xo.x));
        }
#pragma unroll
        for (int m = 0; m < 16; ++m) {
          float2 rv;
          rv.x = __shfl_sync(0xffffffffu, pb[m].x, src_lane);
          rv.y = __shfl_sync(0xffffffffu, pb[m].y, src_lane);
          if (l == 0) rv = (m < 15) ? pb[m + 1] : zh;
          z[31 - m] = rv;
        }
      }
      __syncwarp();  // every lane of this frame holds its bins: the slot may now serve as the exchange plane
      // ---- 3. transform, window, park the frame in its slot
      warp_fft<LOG2N>(z, slot, tw, l);
      __syncwarp();
#pragma unroll
      for (int m = 0; m < 32; ++m) {
        const int n = l + LPF * m;  // time samples 2n, 2n+1
        const float2 wv = *reinterpret_cast<const float2*>(win + 2 * n);
        float2 v = make_float2(z[m].x * inv_n * wv.x, -z[m].y * inv_n * wv.y);
        if (!live) v = make_float2(0.f, 0.f);
        *reinterpret_cast<float2*>(slot + 2 * n) = v;
      }
      __syncthreads();
      // ---- 4. overlap-add (gather) + envelope + write.  Sample t = (g0 + q) hop + r.
      const float* cin = carry + cur * NFFT;
      float* cout = carry + (cur ^ 1) * NFFT;
      const bool emit = gidx >= gs;
      if (vec4) {
        // hop, FS and the carry offsets are multiples of 4: a thread owns 4 consecutive residues (one dmax for all
        // four, see the launch code) and moves float4s -- 4x fewer shared-memory and address instructions
        for (int r = 4 * r4_first; r < hop; r += 4 * RL4) {
          const int dmax = (NFFT - 1 - r) / hop;
          const int qn = G + dmax;
          float4 ef = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int d = 0; d <= dmax; ++d) {
            const float4 wv = *reinterpret_cast<const float4*>(win + d * hop + r);
            ef.x = fmaf(wv.x, wv.x, ef.x); ef.y = fmaf(wv.y, wv.y, ef.y);
            ef.z = fmaf(wv.z, wv.z, ef.z); ef.w = fmaf(wv.w, wv.w, ef.w);
          }
          const float4 inv_ef = p.adjoint ? make_float4(1.f, 1.f, 1.f, 1.f)
                                          : make_float4(1.0f / ef.x, 1.0f / ef.y, 1.0f / ef.z, 1.0f / ef.w);
          for (int q = q4_first; q < qn; q += QL4) {
            const int trel = q * hop + r;
            float4 acc = trel < tail ? *reinterpret_cast<const float4*>(cin + trel) : make_float4(0.f, 0.f, 0.f, 0.f);
            const int jlo = max(q - dmax, 0), jhi = min(q, G - 1);
            for (int j = jlo; j <= jhi; ++j) {
              const float4 v = *reinterpret_cast<const float4*>(reg + j * FS + (q - j) * hop + r);
              acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            if (q >= G) {
              *reinterpret_cast<float4*>(cout + trel - G * hop) = acc;
              continue;
            }
            if (!emit) continue;
            const long long t = (long long)(g0 + q) * hop + r;
            const long long i = t - p.start;
            const int dlo = max(g0 + q - (NP - 1), 0), dhi = min(dmax, g0 + q);
            const bool interior = (dlo == 0 && dhi == dmax);
            if (interior && i >= 0 && i + 3 < p.out_len && t + 3 < p.expected &&
                ((reinterpret_cast<uintptr_t>(orow + i) & 15) == 0)) {
              *reinterpret_cast<float4*>(orow + i) =
                  make_float4(acc.x * inv_ef.x, acc.y * inv_ef.y, acc.z * inv_ef.z, acc.w * inv_ef.w);
            } else {  // signal ends, unaligned rows: per sample, same arithmetic as the scalar path
              const float a4[4] = {acc.x, acc.y, acc.z, acc.w};
              const float ie4[4] = {inv_ef.x, inv_ef.y, inv_ef.z, inv_ef.w};
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const long long iu = i + u;
                if (iu < 0 || iu >= p.out_len) continue;
                float v = 0.f;
                if (t + u < p.expected) {
                  if (interior) {
                    v = a4[u] * ie4[u];
                  } else {
                    float env = 0.f;
                    for (int d = dlo; d <= dhi; ++d) { const float wv = win[d * hop + r + u]; env = fmaf(wv, wv, env); }
                    v = p.adjoint ? a4[u] : a4[u] / env;
                  }
                }
                orow[iu] = v;
              }
            }
          }
        }
      } else
      for (int r = r_first; r < hop; r += RL) {
        const int dmax = (NFFT - 1 - r) / hop;  // frames n with (q - n) in [0, dmax] cover residue r of hop q
        const int qn = G + dmax;                // hops of this group's span that hold residue r
        // envelope of residue r where all dmax+1 covering frames exist (everywhere but the signal's two ends)
        float env_full = 0.f;
        for (int d = 0; d <= dmax; ++d) { const float wv = win[d * hop + r]; env_full = fmaf(wv, wv, env_full); }
        const float inv_env_full = p.adjoint ? 1.f : 1.0f / env_full;
        for (int q = q_first; q < qn; q += QL) {
          const int trel = q * hop + r;
          float acc = trel < tail ? cin[trel] : 0.f;
          const int jlo = max(q - dmax, 0), jhi = min(q, G - 1);
          for (int j = jlo; j <= jhi; ++j) acc += reg[j * FS + (q - j) * hop + r];
          if (q < G) {
            if (emit) {
              const long long t = (long long)(g0 + q) * hop + r;
              const long long i = t - p.start;
              if (i >= 0 && i < p.out_len) {
                float v = 0.f;
                if (t < p.expected) {
                  // env[t] = sum over frames n' = g0 + q - d, d in [0, dmax], 0 <= n' < NP
                  const int dlo = max(g0 + q - (NP - 1), 0), dhi = min(dmax, g0 + q);
                  if (dlo == 0 && dhi == dmax) {
                    v = acc * inv_env_full;
                  } else {
                    float env = 0.f;
                    for (int d = dlo; d <= dhi; ++d) { const float wv = win[d * hop + r]; env = fmaf(wv, wv, env); }
                    v = p.adjoint ? acc : acc / env;
                  }
                }
                orow[i] = v;
              }
            }
          } else {
            cout[trel - G * hop] = acc;
          }
        }
      }
      cur ^= 1;
    }
    // ---- the last segment zero-fills what lies beyond the last group (torch pads with zeros)
    if (ge == p.groups_total) {
      const long long first = (long long)p.groups_total * G * hop - p.start;
      for (long long i = (first > 0 ? first : 0) + tid; i < p.out_len; i += 256) orow[i] = 0.f;
    }
    __syncthreads();  // carry[] and the slots are rewritten by the next item
  }
}

template <int LOG2N>
static int launch(Params& p, void* stream) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N, G = 8 * PL::FPW, NFFT = 2 * N;
  int FS = NFFT + 2;
  if (FS < PL::XB) FS = PL::XB;
  FS = (FS + 3) & ~3;  // multiple of 4: float4 access in the gather
  p.FS = FS;
  int o = 0;
  p.off_tw = o; o = align16(o + PL::NTW * PL::LPF * 8 + 16);
  p.off_ut = o; o = align16(o + 16 * PL::LPF * 8);
  p.off_win = o; o = align16(o + NFFT * 4);
  p.off_carry = o; o = align16(o + 2 * NFFT * 4);
  p.off_reg = o; o = align16(o + G * FS * 4);
  B2A_REQUIRE(o <= 227 * 1024, B2A_E_UNSUPPORTED, "istft: n_fft=%d needs %d bytes of shared memory", NFFT, o);
  B2A_CUDA_OK(cudaFuncSetAttribute(istft_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  int64_t cap;  // resident CTAs: the work list below is sized from them
  const int rc = persistent_grid(istft_kernel<LOG2N>, o, INT64_MAX, &cap);
  if (rc != B2A_OK) return rc;
  // groups: every sample below `expected` (and below start + out_len) must be finalised by some group
  const int NP = p.n_frames + 2 * p.pad_frames;
  long long need = p.start + p.out_len;
  if (need > p.expected) need = p.expected;
  const long long hops = (need + p.hop - 1) / p.hop;  // hop indices 0 .. hops-1 hold the wanted samples
  p.groups_total = (int)((hops + G - 1) / G);
  if (p.groups_total < 1) p.groups_total = 1;
  (void)NP;
  const int R = (NFFT + p.hop - 1) / p.hop;
  p.warm = (R - 1 + G - 1) / G;
  // ~4 work items per resident CTA, but segments of at least 4x the warm-up so the recomputation stays small
  long long seg = ((long long)p.rows * p.groups_total + 4 * cap - 1) / (4 * cap);
  if (seg < 4 * p.warm) seg = 4 * p.warm;
  if (seg < 1) seg = 1;
  if (seg > p.groups_total) seg = p.groups_total;
  p.seg_groups = (int)seg;
  p.segs_per_row = (p.groups_total + p.seg_groups - 1) / p.seg_groups;
  const int64_t items = (int64_t)p.rows * p.segs_per_row;
  B2A_REQUIRE(items < (int64_t)2147483647, B2A_E_UNSUPPORTED, "istft: too many work items");
  const unsigned grid = (unsigned)(items < cap ? items : cap);
  B2A_LAUNCH(istft_kernel<LOG2N>, dim3(grid), dim3(256), (size_t)o, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

static bool supported(int n_fft, int hop) {
  if (n_fft < 64 || n_fft > 2048 || (n_fft & (n_fft - 1))) return false;
  return hop >= 1 && hop <= n_fft;
}

}  // namespace istft
}  // namespace b2a

int b2a::istft::run(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window,
                    int pad_frames, int64_t start, int64_t out_len, float* out, int adjoint, void* stream) {
  B2A_REQUIRE(spec && window && out, B2A_E_INVALID, "istft: null pointer");
  B2A_REQUIRE(rows >= 1 && n_frames >= 1 && out_len >= 1 && pad_frames >= 0 && start >= 0, B2A_E_INVALID,
              "istft: bad argument");
  B2A_REQUIRE(supported(n_fft, hop), B2A_E_UNSUPPORTED,
              "istft: n_fft=%d hop=%d (power-of-two n_fft in [64, 2048], 1 <= hop <= n_fft)", n_fft, hop);
  B2A_REQUIRE(rows < ((int64_t)1 << 24) && n_frames < ((int64_t)1 << 28) && out_len < ((int64_t)1 << 40),
              B2A_E_UNSUPPORTED, "istft: too large");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0, B2A_E_INVALID, "istft: spectra must be 8-byte aligned");
  Params p;
  memset(&p, 0, sizeof(p));
  p.spec = reinterpret_cast<const float2*>(spec);
  p.window = window; p.out = out;
  p.rows = (int)rows; p.n_frames = (int)n_frames; p.pad_frames = pad_frames; p.hop = hop; p.adjoint = adjoint ? 1 : 0;
  p.start = start; p.out_len = out_len;
  p.expected = (long long)(n_frames + 2 * pad_frames - 1) * hop + n_fft;
  switch (n_fft) {
    case 64: return launch<5>(p, stream);
    case 128: return launch<6>(p, stream);
    case 256: return launch<7>(p, stream);
    case 512: return launch<8>(p, stream);
    case 1024: return launch<9>(p, stream);
    default: return launch<10>(p, stream);
  }
}

extern "C" size_t b2a_istft_workspace_bytes(int64_t rows, int64_t n_frames, int n_fft, int hop) {
  const int r = b2a_stft_route(n_fft, hop, 1);
  if (rows < 1 || n_frames < 1 || r == B2A_ROUTE_NONE || r == B2A_ROUTE_FFT) return 0;
  return (size_t)rows * (size_t)n_frames * (size_t)n_fft * sizeof(float);
}

extern "C" int b2a_istft_f32(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop,
                             const float* window, const float* matrix, int pad_frames, int64_t start, int64_t out_len,
                             float* out, void* ws, size_t ws_bytes, void* stream) {
  switch (b2a_stft_route(n_fft, hop, 1)) {
    case B2A_ROUTE_FFT:
      return b2a::istft::run(spec, rows, n_frames, n_fft, hop, window, pad_frames, start, out_len, out, 0, stream);
    case B2A_ROUTE_LARGE:
      return b2a::large::istft(spec, rows, n_frames, n_fft, hop, window, pad_frames, start, out_len, out, ws, ws_bytes,
                               stream);
    case B2A_ROUTE_DENSE:
      return b2a::dft::istft(spec, rows, n_frames, n_fft, hop, window, matrix, pad_frames, start, out_len, out, ws,
                             ws_bytes, stream);
  }
  return b2a::fail(B2A_E_UNSUPPORTED,
                   "istft: n_fft=%d hop=%d (1 <= hop <= n_fft; powers of two up to 32768, any other length up to 8192)",
                   n_fft, hop);
}
