// fftconv.cu -- per-row FIR / circular convolution of [rows, T] waveforms by uniformly partitioned
// overlap-save FFT convolution on sm_90a.
//
// One engine serves every "long filter" of the hot path:
//   * DSPMixin.low_pass / high_pass   (ref:audiotools/core/dsp.py:153-215 -> julius.LowPassFilter:
//                                      windowed-sinc, 103 .. 44983 taps, replicate padding)
//   * EffectMixin.equalizer / mel_filterbank (ref:audiotools/core/effects.py:386-433 -> julius.SplitBands,
//                                      641 taps @44.1k/6 bands; the band split + weighted sum collapses
//                                      into ONE FIR per item)
//   * EffectMixin.convolve            (ref:audiotools/core/effects.py:66-123: CIRCULAR convolution with
//                                      period T, IR rolled to its peak, scaled by 1/max|IR|)
// The reference does these with torch.fft.rfft of the whole (non power of two) signal or with julius'
// block FFT; here:   out[row][n] = post * sum_k g[filt][k] * xv[row][n - k + c[filt]],   n in [0, T)
// where xv extends x by zero / replicate / circular (period T) indexing.
//
//   1. H[filt][f][p]   = rFFT_2048([g_p, 0])            p-th 1024-tap partition   (spectral.cu kernel)
//   2. X[row][f][b]    = rFFT_2048(xv[(b-1)*1024 .. (b+1)*1024))                   (spectral.cu kernel)
//   3. Y[row][f][b]    = sum_p H[f][p] * X[f][b-p]       a complex FIR along the block index, per bin
//   4. out[b*1024 ..]  = irFFT_2048(Y[.][b])[1024:]      warp-per-block inverse FFT + epilogue
// Rows are processed in chunks so that X and Y stay L2-friendly (<= 256 MB of workspace).
#include "b2a_common.h"
#include "fft_warp.cuh"
#include "spectral_internal.h"

namespace b2a {
namespace fftconv {

using namespace b2a::spectral;

constexpr int LP = 1024;    // partition length == new samples per block
constexpr int NFFT = 2048;  // block size
constexpr int NF = 1025;    // bins
constexpr int LOG2N = 10;   // 1024 complex points per block FFT

__global__ void fill_windows_kernel(float* ones, float* half) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NFFT) {
    ones[i] = 1.0f;
    half[i] = i < LP ? 1.0f : 0.0f;
  }
}

__global__ void row_origin_kernel(const int32_t* __restrict__ offset, int offset0, int rows_per_filt, int rows,
                                  int row0, int32_t* __restrict__ row_origin) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) row_origin[r] = offset0 + (offset ? offset[(row0 + r) / rows_per_filt] : 0);
}

// Y[row][f][b] = sum_p H[filt][f][p] * X[row][f][b + P-1 - p]   (complex FIR along the block index)
//
// Register-tiled: a thread owns 4 consecutive blocks b and slides an 8-element complex window over
// q = P-1-p, so 4 new X values and 4 taps are loaded for 16 complex MACs (64 FMAs).  The (row, f) line of X
// is staged in shared memory de-interleaved by (index mod 4): the 4 new window elements of all lanes are then
// unit-stride 64-bit loads (conflict-free); the reversed taps g[q] = H[P-1-q] are broadcast loads.
constexpr int FIR_R = 4;

__device__ __forceinline__ void cmac(float2& a, const float2 g, const float2 x) {
  a.x = fmaf(g.x, x.x, a.x); a.x = fmaf(-g.y, x.y, a.x);
  a.y = fmaf(g.x, x.y, a.y); a.y = fmaf(g.y, x.x, a.y);
}

__global__ void __launch_bounds__(128)
freq_fir_kernel(const float2* __restrict__ X, const float2* __restrict__ H, float2* __restrict__ Y, int NB,
                int NBX, int P, int rows_per_filt, int row0, int SP) {
  B2A_DYN_SMEM(smem);
  float2* xs = reinterpret_cast<float2*>(smem);  // [4][SP]: xs[i & 3][i >> 2] = X[b0 + i]
  float2* gs = xs + 4 * SP;                      // [P4]
  const int f = blockIdx.y, row = blockIdx.z;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int P4 = (P + 3) & ~3;
  const int b0 = blockIdx.x * nt * FIR_R;
  const float2* xr = X + ((size_t)row * NF + f) * NBX + b0;
  const float2* hr = H + ((size_t)((row0 + row) / rows_per_filt) * NF + f) * P;
  const int avail = NBX - b0;
  for (int i = tid; i < 4 * SP; i += nt)
    xs[(i & 3) * SP + (i >> 2)] = i < avail ? __ldg(xr + i) : make_float2(0.f, 0.f);
  for (int q = tid; q < P4; q += nt) gs[q] = q < P ? __ldg(hr + (P - 1 - q)) : make_float2(0.f, 0.f);
  __syncthreads();
  float2 w0 = xs[tid], w1 = xs[SP + tid], w2 = xs[2 * SP + tid], w3 = xs[3 * SP + tid];
  float2 a0 = make_float2(0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
#pragma unroll 2
  for (int q = 0; q < P4; q += 4) {
    const int n = tid + (q >> 2) + 1;
    const float2 v0 = xs[n], v1 = xs[SP + n], v2 = xs[2 * SP + n], v3 = xs[3 * SP + n];
    const float2 g0 = gs[q], g1 = gs[q + 1], g2 = gs[q + 2], g3 = gs[q + 3];
    cmac(a0, g0, w0); cmac(a0, g1, w1); cmac(a0, g2, w2); cmac(a0, g3, w3);
    cmac(a1, g0, w1); cmac(a1, g1, w2); cmac(a1, g2, w3); cmac(a1, g3, v0);
    cmac(a2, g0, w2); cmac(a2, g1, w3); cmac(a2, g2, v0); cmac(a2, g3, v1);
    cmac(a3, g0, w3); cmac(a3, g1, v0); cmac(a3, g2, v1); cmac(a3, g3, v2);
    w0 = v0; w1 = v1; w2 = v2; w3 = v3;
  }
  const int b = b0 + FIR_R * tid;
  float2* yr = Y + ((size_t)row * NF + f) * NB + b;
  if (b < NB) yr[0] = a0;
  if (b + 1 < NB) yr[1] = a1;
  if (b + 2 < NB) yr[2] = a2;
  if (b + 3 < NB) yr[3] = a3;
}

struct InvParams {
  const float2* Y;       // [rows, NF, NB]  (or the signal spectra X when H1 is set)
  const float2* H1;      // single-partition filters [n_filt, NF]: the product X * H is formed on load (no Y pass)
  const float* x;        // [rows_total, T] (for subtract_from_input)
  const float* post;     // [n_filt] nullable
  const int32_t* bypass; // [n_filt] nullable: non-zero = out = x for the rows of this filter
  float* out;            // [rows_total, T]
  int rows, row0, T, NB, rows_per_filt, subtract;
  int off_tw, off_ut, off_buf;
};

// The packed complex input of the inverse real FFT of one block: bin k of the block spectrum is yr[k * fs] (times
// hr[k] when hr is set).  Z[e] = Xe[e] + i Xo[e] from the real-FFT bins X[e], X[N-e]; the inverse transform is
// conj(FFT(conj(Z)))/N, so z holds conj(Z).   e = l + 32 m
template <int N>
__device__ __forceinline__ void inverse_input(float2 (&z)[32], const float2* __restrict__ yr, size_t fs,
                                              const float2* __restrict__ hr, const float2* ut, int l) {
#pragma unroll
  for (int m = 0; m < 32; ++m) {
    const int e = l + 32 * m;
    // for e > N/2 use the pair (k = N-e): Z[e] = conj(Xe[k]) + i conj(Xo[k])
    const int k = (m < 16) ? e : N - e;
    float2 xk = __ldg(yr + (size_t)k * fs);
    float2 xn = __ldg(yr + (size_t)(N - k) * fs);
    if (hr) {  // one partition: Y = H * X, multiplied here instead of in a pass of its own
      xk = cmul(xk, __ldg(hr + k));
      xn = cmul(xn, __ldg(hr + (N - k)));
    }
    // Xe = (X[k] + conj X[N-k])/2 ; T = (X[k] - conj X[N-k])/2 ; Xo = conj(W_k) T, W_k = exp(-i pi k/N)
    const float2 xe = make_float2(0.5f * (xk.x + xn.x), 0.5f * (xk.y - xn.y));
    const float2 tt = make_float2(0.5f * (xk.x - xn.x), 0.5f * (xk.y + xn.y));
    float2 w;
    if (k == N / 2) w = make_float2(0.f, -1.f);
    else w = ut[(k >> 5) * 32 + (k & 31)];  // table index m' * LPF + l' with k = l' + 32 m'
    const float2 xo = make_float2(fmaf(w.x, tt.x, w.y * tt.y), fmaf(w.x, tt.y, -w.y * tt.x));  // conj(w) * tt
    float2 zz = make_float2(xe.x - xo.y, xe.y + xo.x);  // Xe + i Xo
    if (m >= 16 && e != N / 2) zz = make_float2(xe.x + xo.y, -xe.y + xo.x);  // conj(Xe) + i conj(Xo)
    z[m] = make_float2(zz.x, -zz.y);  // conj for the inverse-by-forward trick
  }
}

// inverse real FFT of block spectra, one warp per block, keeping the last LP samples (overlap-save)
__global__ void __launch_bounds__(256, 2) ifft_blocks_kernel(InvParams p) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N;
  B2A_DYN_SMEM(smem);
  float2* tw = reinterpret_cast<float2*>(smem + p.off_tw);
  float2* ut = reinterpret_cast<float2*>(smem + p.off_ut);
  float* xbs = reinterpret_cast<float*>(smem + p.off_buf);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  warp_fft_tables<LOG2N>(tw, ut);
  __syncthreads();
  float* xb = xbs + warp * PL::XB;
  const int l = lane;
  const int groups = (p.NB + 7) / 8;
  const int total = p.rows * groups;
  const float inv_n = 1.0f / (float)N;
#pragma unroll 1
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int row = t / groups, b = (t - row * groups) * 8 + warp;
    if (b >= p.NB) continue;  // warp-uniform
    if (p.bypass && __ldg(p.bypass + (p.row0 + row) / p.rows_per_filt)) {  // not selected by the mask: out = x
      const float* xs = p.x + (size_t)(p.row0 + row) * p.T;
      float* os = p.out + (size_t)(p.row0 + row) * p.T;
      for (int i = l; i < LP; i += 32) { const int s = b * LP + i; if (s < p.T) os[s] = __ldg(xs + s); }
      continue;
    }
    const float2* yr = p.Y + (size_t)row * NF * p.NB + b;
    const float2* hr = p.H1 ? p.H1 + (size_t)((p.row0 + row) / p.rows_per_filt) * NF : nullptr;
    float2 z[32];
    inverse_input<N>(z, yr, (size_t)p.NB, hr, ut, l);
    warp_fft<LOG2N>(z, xb, tw, l);
    // z[m] = conj(N * zt[n]), n = l + 32 m; samples x[2n] = Re zt, x[2n+1] = Im zt; keep n >= N/2
    const int grow = p.row0 + row;
    const float post = p.post ? __ldg(p.post + grow / p.rows_per_filt) : 1.0f;
    float* orow = p.out + (size_t)grow * p.T;
    const float* xrow = p.x + (size_t)grow * p.T;
#pragma unroll
    for (int m = 16; m < 32; ++m) {
      const int n = l + 32 * m;
      const int s0 = b * LP + 2 * n - LP;
      float v0 = z[m].x * inv_n * post, v1 = -z[m].y * inv_n * post;
      if (s0 < p.T) {
        if (p.subtract) v0 = __ldg(xrow + s0) - v0;
        orow[s0] = v0;
      }
      if (s0 + 1 < p.T) {
        if (p.subtract) v1 = __ldg(xrow + s0 + 1) - v1;
        orow[s0 + 1] = v1;
      }
    }
    __syncwarp();
  }
}

// per CTA of 256 threads: first index of max|h| over the first Leff samples, and 1 / max(max|h|, 1e-5), stored at
// idx_out[blockIdx.x] and scale_out[blockIdx.x]
__device__ __forceinline__ void ir_peak(const float* __restrict__ h, int Leff, int32_t* __restrict__ idx_out,
                                        float* __restrict__ scale_out, int roll) {
  __shared__ float sv[256];
  __shared__ int si[256];
  float best = -1.f;
  int bi = 0;
  for (int i = threadIdx.x; i < Leff; i += 256) {
    const float a = fabsf(h[i]);
    if (a > best) { best = a; bi = i; }  // strictly greater: keeps the first maximum of this thread's stride
  }
  sv[threadIdx.x] = best;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      const float o = sv[threadIdx.x + s];
      const int oi = si[threadIdx.x + s];
      if (o > sv[threadIdx.x] || (o == sv[threadIdx.x] && oi < si[threadIdx.x])) {
        sv[threadIdx.x] = o;
        si[threadIdx.x] = oi;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    idx_out[blockIdx.x] = roll ? si[0] : 0;
    scale_out[blockIdx.x] = 1.0f / fmaxf(sv[0], 1e-5f);
  }
}

// per IR of rows L apart: ir_peak
__global__ void __launch_bounds__(256)
ir_peak_kernel(const float* __restrict__ ir, int L, int Leff, int32_t* __restrict__ idx_out,
               float* __restrict__ scale_out, int roll) {
  ir_peak(ir + (size_t)blockIdx.x * L, Leff, idx_out, scale_out, roll);
}

struct Layout {
  size_t ones, half, H, X, Y, rorg, peak_idx, peak_scale, total;
  int P, NB, NBX, chunk;
};
static inline size_t al(size_t v) { return (v + 255) & ~(size_t)255; }
// Spectra of one chunk of rows (X and, with several partitions, Y): rows are processed in chunks whose spectra take at
// most 256 MB, which bounds the workspace.
constexpr size_t CHUNK_BUDGET_MB = 256;

static Layout layout(int64_t rows, int64_t T, int64_t n_filt, int64_t L) {
  Layout w;
  w.P = (int)((L + LP - 1) / LP);
  w.NB = (int)((T + LP - 1) / LP);
  w.NBX = w.NB + w.P - 1;
  // one partition: the product is formed inside the inverse kernel, Y is never written (see run())
  const size_t per_row = (size_t)NF * (w.NBX + (w.P > 1 ? w.NB : 0)) * 8;
  int64_t chunk = (int64_t)((CHUNK_BUDGET_MB << 20) / per_row);
  if (chunk < 1) chunk = 1;
  if (chunk > rows) chunk = rows;
  if (chunk > 65535) chunk = 65535;
  w.chunk = (int)chunk;
  size_t o = 0;
  w.ones = o; o = al(o + NFFT * 4);
  w.half = o; o = al(o + NFFT * 4);
  w.H = o; o = al(o + (size_t)n_filt * NF * w.P * 8);
  w.X = o; o = al(o + (size_t)w.chunk * NF * w.NBX * 8);
  w.Y = o; o = al(o + (w.P > 1 ? (size_t)w.chunk * NF * w.NB * 8 : 0));
  w.rorg = o; o = al(o + (size_t)w.chunk * 4);
  w.peak_idx = o; o = al(o + (size_t)n_filt * 4);
  w.peak_scale = o; o = al(o + (size_t)n_filt * 4);
  w.total = o;
  return w;
}

static int run(const float* x, int64_t rows, int64_t T, const float* g, int64_t n_filt, int64_t L, int rows_per_filt,
               const int32_t* offset, int offset0, int pad_mode, const float* post_scale, int subtract,
               const int32_t* bypass, float* out, char* ws, const Layout& w, void* stream) {
  float* ones = (float*)(ws + w.ones);
  float* half = (float*)(ws + w.half);
  float2* H = (float2*)(ws + w.H);
  float2* X = (float2*)(ws + w.X);
  float2* Y = (float2*)(ws + w.Y);
  int32_t* rorg = (int32_t*)(ws + w.rorg);
  B2A_LAUNCH(fill_windows_kernel, dim3(NFFT / 256), dim3(256), 0, stream, ones, half);
  // 1. filter partitions: frame p = g[p*LP, p*LP + 2048) x [1..1 0..0], zero beyond L
  int rc = frames_fft(g, (int)n_filt, (int)L, NFFT, LP, half, 0, nullptr, B2A_PAD_CONSTANT, w.P, H, stream);
  if (rc != B2A_OK) return rc;
  using PL = WPlan<LOG2N>;
  InvParams ip;
  memset(&ip, 0, sizeof(ip));
  int o = 0;
  ip.off_tw = o; o += (PL::NTW * PL::LPF * 8 + 31) & ~15;
  ip.off_ut = o; o += (16 * PL::LPF * 8 + 15) & ~15;
  ip.off_buf = o; o += 8 * PL::XB * 4;
  B2A_CUDA_OK(cudaFuncSetAttribute(ifft_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  for (int64_t r0 = 0; r0 < rows; r0 += w.chunk) {
    const int nr = (int)((rows - r0 < w.chunk) ? rows - r0 : w.chunk);
    B2A_LAUNCH(row_origin_kernel, dim3((nr + 255) / 256), dim3(256), 0, stream, offset, offset0, rows_per_filt, nr,
               (int)r0, rorg);
    // 2. block b' covers xv[(b' - P)*LP + c, +2048)
    rc = frames_fft(x + (size_t)r0 * T, nr, (int)T, NFFT, LP, ones, -w.P * LP, rorg, pad_mode, w.NBX, X, stream);
    if (rc != B2A_OK) return rc;
    // 3. complex FIR along the block index
    if (w.P > 1) {
      int nt = ((w.NB + FIR_R - 1) / FIR_R + 31) / 32 * 32;
      if (nt > 128) nt = 128;
      const int P4 = (w.P + 3) & ~3;
      int SP = nt + P4 / 4 + 1;
      SP += (8 - (SP & 15)) & 15;  // SP = 8 mod 16: the 4 phase rows of a staging store hit distinct banks
      const size_t fir_smem = (size_t)(4 * SP + P4) * sizeof(float2);
      B2A_REQUIRE(fir_smem <= 48 * 1024, B2A_E_UNSUPPORTED, "fftconv: %d partitions do not fit", w.P);
      B2A_LAUNCH(freq_fir_kernel, dim3((w.NB + nt * FIR_R - 1) / (nt * FIR_R), NF, nr), dim3(nt), fir_smem, stream,
                 (const float2*)X, (const float2*)H, Y, w.NB, w.NBX, w.P, rows_per_filt, (int)r0, SP);
    }
    // 4. inverse FFT + overlap-save + epilogue
    // one partition (NBX == NB): the inverse kernel multiplies X by H while loading, Y is never written
    ip.Y = (w.P > 1) ? Y : X; ip.H1 = (w.P > 1) ? nullptr : H;
    ip.x = x; ip.post = post_scale; ip.out = out; ip.bypass = bypass;
    ip.rows = nr; ip.row0 = (int)r0; ip.T = (int)T; ip.NB = w.NB; ip.rows_per_filt = rows_per_filt;
    ip.subtract = subtract;
    const int64_t total = (int64_t)nr * ((w.NB + 7) / 8);
    const int64_t cap = (int64_t)num_sms() * 2;
    B2A_LAUNCH(ifft_blocks_kernel, dim3((unsigned)(total < cap ? total : cap)), dim3(256), (size_t)o, stream, ip);
  }
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

}  // namespace fftconv
}  // namespace b2a

using namespace b2a::fftconv;

extern "C" size_t b2a_fftconv_workspace_bytes(int64_t rows, int64_t T, int64_t n_filt, int64_t L) {
  if (rows < 1 || T < 1 || n_filt < 1 || L < 1) return 0;
  return layout(rows, T, n_filt, L).total;
}

extern "C" int b2a_fftconv_f32(const float* x, int64_t rows, int64_t T, const float* g, int64_t n_filt, int64_t L,
                               int rows_per_filt, const int32_t* offset, int offset0, int pad_mode,
                               const float* post_scale, int subtract_from_input, const int32_t* bypass, float* out,
                               void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(x && g && out && ws, B2A_E_INVALID, "fftconv: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && n_filt >= 1 && L >= 1 && rows_per_filt >= 1, B2A_E_INVALID, "fftconv: bad shape");
  B2A_REQUIRE((rows + rows_per_filt - 1) / rows_per_filt <= n_filt, B2A_E_INVALID,
              "fftconv: %lld rows / %d per filter need more than %lld filters", (long long)rows, rows_per_filt,
              (long long)n_filt);
  B2A_REQUIRE(T < ((int64_t)1 << 30) && L < ((int64_t)1 << 30), B2A_E_UNSUPPORTED, "fftconv: too long");
  B2A_REQUIRE(pad_mode == B2A_PAD_CONSTANT || pad_mode == B2A_PAD_REPLICATE || pad_mode == 3, B2A_E_INVALID,
              "fftconv: pad_mode %d (1 zero, 2 replicate, 3 circular)", pad_mode);
  B2A_REQUIRE(out != x, B2A_E_INVALID, "fftconv: in-place is not supported");
  const Layout w = layout(rows, T, n_filt, L);
  B2A_REQUIRE(ws_bytes >= w.total, B2A_E_INVALID, "fftconv: workspace too small (%zu < %zu)", ws_bytes, w.total);
  return run(x, rows, T, g, n_filt, L, rows_per_filt, offset, offset0, pad_mode, post_scale, subtract_from_input, bypass,
             out, (char*)ws, w, stream);
}

/* EffectMixin.convolve (ref:audiotools/core/effects.py:66-123): out = (x (*) roll(ir, -argmax|ir|)) / max(max|ir|, 1e-5),
 * circular with period T.  ir: [n_ir, L] (mono IRs, one per rows_per_ir rows); only its first min(L, T) samples count. */
extern "C" size_t b2a_circconv_workspace_bytes(int64_t rows, int64_t T, int64_t n_ir, int64_t L) {
  if (rows < 1 || T < 1 || n_ir < 1 || L < 1) return 0;
  return layout(rows, T, n_ir, L < T ? L : T).total;
}

extern "C" int b2a_circconv_f32(const float* x, int64_t rows, int64_t T, const float* ir, int64_t n_ir, int64_t L,
                                int rows_per_ir, int roll_to_peak, const int32_t* bypass, float* out, void* ws,
                                size_t ws_bytes, void* stream) {
  B2A_REQUIRE(x && ir && out && ws, B2A_E_INVALID, "circconv: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && n_ir >= 1 && L >= 1 && rows_per_ir >= 1, B2A_E_INVALID, "circconv: bad shape");
  const int64_t Leff = L < T ? L : T;  // the reference truncates the IR to the signal length
  const Layout w = layout(rows, T, n_ir, Leff);
  B2A_REQUIRE(ws_bytes >= w.total, B2A_E_INVALID, "circconv: workspace too small (%zu < %zu)", ws_bytes, w.total);
  char* base = (char*)ws;
  int32_t* pidx = (int32_t*)(base + w.peak_idx);
  float* pscale = (float*)(base + w.peak_scale);
  B2A_LAUNCH(ir_peak_kernel, dim3((unsigned)n_ir), dim3(256), 0, stream, ir, (int)L, (int)Leff, pidx, pscale,
             roll_to_peak);
  // y[n] = sum_j h[j] x[(n - (j - idx)) mod T]  ==  causal conv with offset c = idx, circular indexing
  B2A_REQUIRE(L == Leff, B2A_E_INVALID, "circconv: pass the IR already truncated to the signal length (L=%lld > T=%lld)",
              (long long)L, (long long)T);
  return run(x, rows, T, ir, n_ir, Leff, rows_per_ir, pidx, 0, 3, pscale, 0, bypass, out, base, w, stream);
}

/* Adjoint of b2a_circconv_f32.  The forward is y[n] = s sum_j h[j] x[(n - j + idx) mod T]; its adjoint
 * gx[m] = s sum_j h[j] g[(m + j - idx) mod T] is the same engine with the taps reversed (h~[k] = h[L-1-k]) and the
 * per-IR offset L-1-idx; idx and s come from ir_peak_kernel exactly as in the forward.  The reversal is a kernel of its
 * own (reverse_taps_kernel) so that the shared filter-FFT stage stays caller-agnostic.  Bypassed rows copy g. */
namespace b2a {
namespace fftconv {

__global__ void __launch_bounds__(256) reverse_taps_kernel(const float* __restrict__ ir, int L,
                                                           const int32_t* __restrict__ pidx, float* __restrict__ rev,
                                                           int32_t* __restrict__ off) {
  const float* h = ir + (size_t)blockIdx.x * L;
  float* o = rev + (size_t)blockIdx.x * L;
  for (int k = threadIdx.x; k < L; k += 256) o[k] = h[L - 1 - k];
  if (threadIdx.x == 0) off[blockIdx.x] = L - 1 - pidx[blockIdx.x];
}

}  // namespace fftconv
}  // namespace b2a

extern "C" size_t b2a_circconv_backward_workspace_bytes(int64_t rows, int64_t T, int64_t n_ir, int64_t L) {
  if (rows < 1 || T < 1 || n_ir < 1 || L < 1) return 0;
  const int64_t Leff = L < T ? L : T;
  return layout(rows, T, n_ir, Leff).total + al((size_t)n_ir * Leff * 4) + al((size_t)n_ir * 4);
}

extern "C" int b2a_circconv_backward_f32(const float* grad_out, int64_t rows, int64_t T, const float* ir, int64_t n_ir,
                                         int64_t L, int rows_per_ir, int roll_to_peak, const int32_t* bypass,
                                         float* grad_x, void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(grad_out && ir && grad_x && ws, B2A_E_INVALID, "circconv_backward: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && n_ir >= 1 && L >= 1 && rows_per_ir >= 1, B2A_E_INVALID,
              "circconv_backward: bad shape");
  B2A_REQUIRE(L <= T, B2A_E_INVALID,
              "circconv_backward: pass the IR already truncated to the signal length (L=%lld > T=%lld)", (long long)L,
              (long long)T);
  B2A_REQUIRE(grad_out != grad_x, B2A_E_INVALID, "circconv_backward: in-place is not supported");
  const Layout w = layout(rows, T, n_ir, L);
  B2A_REQUIRE(ws_bytes >= b2a_circconv_backward_workspace_bytes(rows, T, n_ir, L), B2A_E_INVALID,
              "circconv_backward: workspace too small");
  char* base = (char*)ws;
  int32_t* pidx = (int32_t*)(base + w.peak_idx);
  float* pscale = (float*)(base + w.peak_scale);
  float* rev = (float*)(base + w.total);
  int32_t* off = (int32_t*)(base + w.total + al((size_t)n_ir * L * 4));
  B2A_LAUNCH(ir_peak_kernel, dim3((unsigned)n_ir), dim3(256), 0, stream, ir, (int)L, (int)L, pidx, pscale, roll_to_peak);
  B2A_LAUNCH(reverse_taps_kernel, dim3((unsigned)n_ir), dim3(256), 0, stream, ir, (int)L, (const int32_t*)pidx, rev, off);
  return run(grad_out, rows, T, rev, n_ir, L, rows_per_ir, off, 0, 3, pscale, 0, bypass, grad_x, base, w, stream);
}

/* b2a_circconv_path_f32: a circular convolution whose impulse response moves along a path of K waypoints, one IR
 * every `hop` samples (DESIGN.md K22).  Waypoint k sits at tau_k = k hop; the output is the receiver-time crossfade
 *     y[row][t] = s sum_k v_k(t) sum_j h_k[j] x[(t - j + idx) mod T],   v_k(t) = max(0, 1 - |t - tau_k| / hop),
 * v_{K-1}(t) = 1 for t >= tau_{K-1}, with idx and s from waypoint 0 (ir_peak_kernel), so the weights sum to 1 and a
 * change in propagation delay along the path stays in the output.
 *
 * It is the overlap-save engine above with the FIR stage split by waypoint.  X is computed once per row.  Waypoint k
 * is non-zero on (tau_{k-1}, tau_{k+1}), so its FIR runs only over the output blocks that meet that span
 * (path_blocks); hop >= LP means a block meets at most 3 waypoints, and waypoints k and k + 3 never share a block.
 * Each waypoint therefore writes its own slot k % 3 of Y3 with no overlap, and the inverse kernel transforms the 2 or
 * 3 slots of a block, weights each sample by v_k and sums them in waypoint order: no atomics, no read-modify-write. */
namespace b2a {
namespace fftconv {

// The output blocks [lo, hi] on which waypoint k's weight is non-zero: those meeting (tau_{k-1}, tau_{k+1}), from block
// 0 for the first waypoint and up to the last block for the last one.
__device__ __forceinline__ void path_blocks(int k, int K, int hop, int NB, int& lo, int& hi) {
  lo = k == 0 ? 0 : ((k - 1) * hop + 1) / LP;
  hi = k == K - 1 ? NB - 1 : min(((k + 1) * hop - 1) / LP, NB - 1);
}

// v_k(t): hop - |t - tau_k| is exact, so the weights of two neighbours are each rounded once.
__device__ __forceinline__ float path_weight(int k, int K, int hop, int t) {
  const int d = t - k * hop;
  if (k == K - 1 && d >= 0) return 1.0f;
  const int a = d < 0 ? -d : d;
  return a >= hop ? 0.0f : (float)(hop - a) / (float)hop;
}

constexpr int PATH_R = 8;  // output blocks per thread and register tile

// Y3[row][k % 3][b][f] = sum_p H[item][k][c][f][p] * X[row][f][b + P-1 - p] over the blocks b of waypoint k, for the
// row's IR ir = item * ir_channels + c.  One thread
// per bin f walks the waypoint's blocks in tiles of PATH_R and slides a window over X, so each tap and each new X value
// is loaded once per tile.  The sum runs in freq_fir_kernel's order (q = P-1-p ascending, one fmaf chain per output),
// so a waypoint's block spectra are bit-identical to the static engine's.  The [b][f] layout makes the stores and the
// inverse kernel's loads unit-stride.
__global__ void __launch_bounds__(128)
path_fir_kernel(const float2* __restrict__ X, const float2* __restrict__ H, float2* __restrict__ Y3, int NB, int NBX,
                int P, int K, int hop, int rows_per_ir, int ir_channels, int row0) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= NF) return;
  const int k = blockIdx.y, row = blockIdx.z;
  int lo, hi;
  path_blocks(k, K, hop, NB, lo, hi);
  const int ir = (row0 + row) / rows_per_ir - row0 / rows_per_ir;  // chunks start on an item boundary
  const int filt = ((ir / ir_channels) * K + k) * ir_channels + ir % ir_channels;
  const float2* xr = X + ((size_t)row * NF + f) * NBX;
  const float2* hr = H + ((size_t)filt * NF + f) * P;
  float2* yr = Y3 + ((size_t)row * 3 + k % 3) * NB * NF + f;
  const float2 zero = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int b0 = lo; b0 <= hi; b0 += PATH_R) {
    float2 w[PATH_R], a[PATH_R];
#pragma unroll
    for (int r = 0; r < PATH_R; ++r) {
      w[r] = b0 + r < NBX ? __ldg(xr + b0 + r) : zero;  // w[r] = X[b0 + r + q]
      a[r] = zero;
    }
#pragma unroll 2
    for (int q = 0; q < P; ++q) {
      const float2 g = __ldg(hr + (P - 1 - q));
#pragma unroll
      for (int r = 0; r < PATH_R; ++r) cmac(a[r], g, w[r]);
#pragma unroll
      for (int r = 0; r < PATH_R - 1; ++r) w[r] = w[r + 1];
      const int i = b0 + PATH_R + q;
      w[PATH_R - 1] = i < NBX ? __ldg(xr + i) : zero;
    }
#pragma unroll
    for (int r = 0; r < PATH_R; ++r)
      if (b0 + r <= hi) yr[(size_t)(b0 + r) * NF] = a[r];
  }
}

struct PathInvParams {
  const float2* Y3;      // [rows, 3, NB, NF]
  const float* x;        // [rows_total, T]
  const float* post;     // [n_ir]
  const int32_t* bypass; // [n_ir] nullable: non-zero = out = x for the rows of this IR
  float* out;            // [rows_total, T]
  int rows, row0, T, NB, K, hop, rows_per_ir;
  int off_tw, off_ut, off_buf;
};

// One warp per output block: the inverse FFT of each waypoint active on the block, weighted per sample by v_k and
// summed in waypoint order, then scaled by the row's post.
__global__ void __launch_bounds__(256, 2) path_ifft_kernel(PathInvParams p) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N;
  B2A_DYN_SMEM(smem);
  float2* tw = reinterpret_cast<float2*>(smem + p.off_tw);
  float2* ut = reinterpret_cast<float2*>(smem + p.off_ut);
  float* xbs = reinterpret_cast<float*>(smem + p.off_buf);
  const int tid = threadIdx.x, l = tid & 31, warp = tid >> 5;
  warp_fft_tables<LOG2N>(tw, ut);
  __syncthreads();
  float* xb = xbs + warp * PL::XB;
  const int groups = (p.NB + 7) / 8;
  const int total = p.rows * groups;
  const float inv_n = 1.0f / (float)N;
#pragma unroll 1
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int row = t / groups, b = (t - row * groups) * 8 + warp;
    if (b >= p.NB) continue;  // warp-uniform
    const int grow = p.row0 + row;
    float* orow = p.out + (size_t)grow * p.T;
    if (p.bypass && __ldg(p.bypass + grow / p.rows_per_ir)) {
      const float* xs = p.x + (size_t)grow * p.T;
      for (int i = l; i < LP; i += 32) { const int s = b * LP + i; if (s < p.T) orow[s] = __ldg(xs + s); }
      continue;
    }
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    const int kc = b * LP / p.hop;  // the waypoints meeting block b are among kc - 1 .. kc + 2
    const int k1 = min(kc + 2, p.K - 1);
#pragma unroll 1
    for (int k = max(kc - 1, 0); k <= k1; ++k) {
      int lo, hi;
      path_blocks(k, p.K, p.hop, p.NB, lo, hi);
      if (b < lo || b > hi) continue;  // warp-uniform
      float2 z[32];
      inverse_input<N>(z, p.Y3 + (((size_t)row * 3 + k % 3) * p.NB + b) * NF, 1, nullptr, ut, l);
      warp_fft<LOG2N>(z, xb, tw, l);
      // z[m] = conj(N * zt[n]), n = l + 32 m; samples x[2n] = Re zt, x[2n+1] = Im zt; keep n >= N/2
#pragma unroll
      for (int m = 16; m < 32; ++m) {
        const int s0 = b * LP + 2 * (l + 32 * m) - LP;
        acc[2 * (m - 16)] += path_weight(k, p.K, p.hop, s0) * (z[m].x * inv_n);
        acc[2 * (m - 16) + 1] += path_weight(k, p.K, p.hop, s0 + 1) * (-z[m].y * inv_n);
      }
      __syncwarp();
    }
    const float post = __ldg(p.post + grow / p.rows_per_ir);
#pragma unroll
    for (int m = 16; m < 32; ++m) {
      const int s0 = b * LP + 2 * (l + 32 * m) - LP;
      if (s0 < p.T) orow[s0] = acc[2 * (m - 16)] * post;
      if (s0 + 1 < p.T) orow[s0 + 1] = acc[2 * (m - 16) + 1] * post;
    }
  }
}

// per IR i = item * ir_channels + c of an [items][K][ir_channels][L] bank: ir_peak of its first waypoint
__global__ void __launch_bounds__(256)
path_peak_kernel(const float* __restrict__ ir, int K, int ir_channels, int L, int32_t* __restrict__ idx_out,
                 float* __restrict__ scale_out, int roll) {
  const int item = blockIdx.x / ir_channels, c = blockIdx.x - item * ir_channels;
  ir_peak(ir + ((size_t)item * K * ir_channels + c) * L, L, idx_out, scale_out, roll);
}

struct PathLayout {
  size_t ones, half, H, X, Y3, rorg, peak_idx, peak_scale, total;
  int P, NB, NBX, chunk;  // chunk: rows per chunk, whole items of ir_channels * rows_per_ir rows
};

// Per item: the spectra of its ir_channels x K waypoints; per row: X and the three Y3 slots.  A chunk of whole items
// takes at most CHUNK_BUDGET_MB of spectra, or one item when a single one needs more.
static PathLayout path_layout(int64_t rows, int64_t T, int64_t K, int64_t L, int64_t rows_per_ir,
                              int64_t ir_channels) {
  PathLayout w;
  w.P = (int)((L + LP - 1) / LP);
  w.NB = (int)((T + LP - 1) / LP);
  w.NBX = w.NB + w.P - 1;
  const int64_t n_ir = rows / rows_per_ir, item_rows = rows_per_ir * ir_channels, items = rows / item_rows;
  const size_t per_item = ((size_t)ir_channels * K * w.P + (size_t)item_rows * (w.NBX + 3 * (size_t)w.NB)) * NF * 8;
  int64_t chunk = (int64_t)((CHUNK_BUDGET_MB << 20) / per_item);
  if (chunk < 1) chunk = 1;
  if (chunk > items) chunk = items;
  if (chunk * item_rows > 65535) chunk = 65535 / item_rows;
  w.chunk = (int)(chunk * item_rows);
  size_t o = 0;
  w.ones = o; o = al(o + NFFT * 4);
  w.half = o; o = al(o + NFFT * 4);
  w.H = o; o = al(o + (size_t)chunk * ir_channels * K * w.P * NF * 8);
  w.X = o; o = al(o + (size_t)w.chunk * NF * w.NBX * 8);
  w.Y3 = o; o = al(o + (size_t)w.chunk * 3 * w.NB * NF * 8);
  w.rorg = o; o = al(o + (size_t)w.chunk * 4);
  w.peak_idx = o; o = al(o + (size_t)n_ir * 4);
  w.peak_scale = o; o = al(o + (size_t)n_ir * 4);
  w.total = o;
  return w;
}

static int run_path(const float* x, int64_t rows, int64_t T, const float* ir, int64_t K, int64_t L, int rows_per_ir,
                    int ir_channels, int hop, int roll_to_peak, const int32_t* bypass, float* out, char* ws,
                    const PathLayout& w, void* stream) {
  float* ones = (float*)(ws + w.ones);
  float* half = (float*)(ws + w.half);
  float2* H = (float2*)(ws + w.H);
  float2* X = (float2*)(ws + w.X);
  float2* Y3 = (float2*)(ws + w.Y3);
  int32_t* rorg = (int32_t*)(ws + w.rorg);
  int32_t* pidx = (int32_t*)(ws + w.peak_idx);
  float* pscale = (float*)(ws + w.peak_scale);
  const int64_t n_ir = rows / rows_per_ir, item_rows = (int64_t)rows_per_ir * ir_channels;
  // roll and scale of every IR's first waypoint
  B2A_LAUNCH(path_peak_kernel, dim3((unsigned)n_ir), dim3(256), 0, stream, ir, (int)K, ir_channels, (int)L, pidx,
             pscale, roll_to_peak);
  B2A_LAUNCH(fill_windows_kernel, dim3(NFFT / 256), dim3(256), 0, stream, ones, half);
  using PL = WPlan<LOG2N>;
  PathInvParams ip;
  memset(&ip, 0, sizeof(ip));
  int o = 0;
  ip.off_tw = o; o += (PL::NTW * PL::LPF * 8 + 31) & ~15;
  ip.off_ut = o; o += (16 * PL::LPF * 8 + 15) & ~15;
  ip.off_buf = o; o += 8 * PL::XB * 4;
  B2A_CUDA_OK(cudaFuncSetAttribute(path_ifft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  for (int64_t r0 = 0; r0 < rows; r0 += w.chunk) {
    const int nr = (int)((rows - r0 < w.chunk) ? rows - r0 : w.chunk);
    const int64_t b0 = r0 / item_rows, nb = nr / item_rows;
    // 1. partitions of every waypoint of the chunk's items, a contiguous run of filters: [nb][K][ir_channels][NF][P]
    int rc = frames_fft(ir + (size_t)b0 * K * ir_channels * L, (int)(nb * K * ir_channels), (int)L, NFFT, LP, half, 0,
                        nullptr, B2A_PAD_CONSTANT, w.P, H, stream);
    if (rc != B2A_OK) return rc;
    // 2. block spectra of the rows, circular, shifted by waypoint 0's peak
    B2A_LAUNCH(row_origin_kernel, dim3((nr + 255) / 256), dim3(256), 0, stream, (const int32_t*)pidx, 0, rows_per_ir,
               nr, (int)r0, rorg);
    rc = frames_fft(x + (size_t)r0 * T, nr, (int)T, NFFT, LP, ones, -w.P * LP, rorg, 3, w.NBX, X, stream);
    if (rc != B2A_OK) return rc;
    // 3. each waypoint's FIR over its own blocks
    B2A_LAUNCH(path_fir_kernel, dim3((NF + 127) / 128, (unsigned)K, nr), dim3(128), 0, stream, (const float2*)X,
               (const float2*)H, Y3, w.NB, w.NBX, w.P, (int)K, hop, rows_per_ir, ir_channels, (int)r0);
    // 4. inverse FFTs, crossfade, scale
    ip.Y3 = Y3; ip.x = x; ip.post = pscale; ip.bypass = bypass; ip.out = out;
    ip.rows = nr; ip.row0 = (int)r0; ip.T = (int)T; ip.NB = w.NB; ip.K = (int)K; ip.hop = hop;
    ip.rows_per_ir = rows_per_ir;
    const int64_t total = (int64_t)nr * ((w.NB + 7) / 8);
    const int64_t cap = (int64_t)num_sms() * 2;
    B2A_LAUNCH(path_ifft_kernel, dim3((unsigned)(total < cap ? total : cap)), dim3(256), (size_t)o, stream, ip);
  }
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

}  // namespace fftconv
}  // namespace b2a

extern "C" size_t b2a_circconv_path_workspace_bytes(int64_t rows, int64_t T, int64_t K, int64_t L, int rows_per_ir,
                                                    int ir_channels, int hop) {
  if (rows < 1 || T < 1 || K < 1 || L < 1 || rows_per_ir < 1 || ir_channels < 1 ||
      rows % ((int64_t)rows_per_ir * ir_channels) || hop < 1)
    return 0;
  return path_layout(rows, T, K, L < T ? L : T, rows_per_ir, ir_channels).total;
}

extern "C" int b2a_circconv_path_f32(const float* x, int64_t rows, int64_t T, const float* ir, int64_t K, int64_t L,
                                     int rows_per_ir, int ir_channels, int hop, int roll_to_peak,
                                     const int32_t* bypass, float* out, void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(x && ir && out && ws, B2A_E_INVALID, "circconv_path: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && K >= 1 && L >= 1 && rows_per_ir >= 1 && ir_channels >= 1, B2A_E_INVALID,
              "circconv_path: bad shape");
  B2A_REQUIRE(rows % ((int64_t)rows_per_ir * ir_channels) == 0, B2A_E_INVALID,
              "circconv_path: %lld rows are not whole items of %d IRs of %d rows", (long long)rows, ir_channels,
              rows_per_ir);
  B2A_REQUIRE(T < ((int64_t)1 << 30), B2A_E_UNSUPPORTED, "circconv_path: too long");
  B2A_REQUIRE(hop >= LP, B2A_E_INVALID, "circconv_path: hop %d < %d samples (a block would meet more than 3 waypoints)",
              hop, LP);
  B2A_REQUIRE(K == (T - 1) / hop + 1, B2A_E_INVALID,
              "circconv_path: %lld waypoints %d samples apart do not cover T=%lld (need %lld)", (long long)K, hop,
              (long long)T, (long long)((T - 1) / hop + 1));
  B2A_REQUIRE(L <= T, B2A_E_INVALID,
              "circconv_path: pass the IRs already truncated to the signal length (L=%lld > T=%lld)", (long long)L,
              (long long)T);
  B2A_REQUIRE(K <= 65535 && K * ir_channels * L < ((int64_t)1 << 31), B2A_E_UNSUPPORTED,
              "circconv_path: %lld waypoints of %d x %lld samples are too many", (long long)K, ir_channels,
              (long long)L);
  B2A_REQUIRE(out != x, B2A_E_INVALID, "circconv_path: in-place is not supported");
  const PathLayout w = path_layout(rows, T, K, L, rows_per_ir, ir_channels);
  B2A_REQUIRE(ws_bytes >= w.total, B2A_E_INVALID, "circconv_path: workspace too small (%zu < %zu)", ws_bytes, w.total);
  return run_path(x, rows, T, ir, K, L, rows_per_ir, ir_channels, hop, roll_to_peak, bypass, out, (char*)ws, w,
                  stream);
}
