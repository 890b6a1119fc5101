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
    // Z[e] = Xe[e] + i Xo[e] from the real-FFT bins X[e], X[N-e]; the inverse transform is
    // conj(FFT(conj(Z)))/N, so feed conj(Z).   e = l + 32 m
    float2 z[32];
#pragma unroll
    for (int m = 0; m < 32; ++m) {
      const int e = l + 32 * m;
      // for e > N/2 use the pair (k = N-e): Z[e] = conj(Xe[k]) + i conj(Xo[k])
      const int k = (m < 16) ? e : N - e;
      float2 xk = __ldg(yr + (size_t)k * p.NB);
      float2 xn = __ldg(yr + (size_t)(N - k) * p.NB);
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

// per item: first index of max|h| over the first Leff samples, and 1 / max(max|h|, 1e-5)
__global__ void __launch_bounds__(256)
ir_peak_kernel(const float* __restrict__ ir, int L, int Leff, int32_t* __restrict__ idx_out,
               float* __restrict__ scale_out, int roll) {
  __shared__ float sv[256];
  __shared__ int si[256];
  const float* h = ir + (size_t)blockIdx.x * L;
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
