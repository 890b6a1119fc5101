// rir.cu -- shoebox-room impulse responses by the image-source method (Allen & Berkley 1979), one per (item,
// microphone) row of a batch (K20 in DESIGN.md).
//
//   Distances are in samples (metres * fs / c).  For integers m = (mx, my, mz) and parities (q, j, k) in {0, 1}^3 the
//   image offset along x is X = (1 - 2q) s_x - r_x + 2 mx Lx (likewise y, z); d = |(X, Y, Z)|.  Its order is
//   |2mx - q| + |2my - j| + |2mz - k|, its gain
//     g = bx0^|mx-q| bx1^|mx| by0^|my-j| by1^|my| bz0^|mz-k| bz1^|mz| / (4 pi d c / fs),
//   and it adds g h(i - d) at every sample i in [floor(d) - Tw/2 + 1, floor(d) + Tw/2] inside [0, L), where
//     h(t) = cos^2(pi t / Tw) sinc(pi t),  Tw = 2 floor(0.004 fs + 1/2)
//   (the Hann-windowed fractional delay 1/2 (1 - cos(2 pi (n + 1 - f) / Tw)) sinc(pi (n + 1 - f - Tw/2)) of tap n,
//   f = d - floor(d), written in t = i - d).  Images with floor(d) >= L, or an order above max_order >= 0, are unused.
//
// One launch, no host sync, no atomics.  A CTA owns one row and a tile of TT output samples; a warp owns 32 * PER
// consecutive samples of it, a lane every 32nd.  The images that reach the tile have floor(d) in a spherical shell
// [t0 - Tw/2, t0 + TT + Tw/2 - 1).  The CTA walks the (mx, q, my, j, k) lines of that shell, NT at a time; each
// thread finds its line's mz values inside the shell (at most two runs, in closed form, widened by one on either
// side and then filtered per image on the exact floor(d)), a block scan gives every image a slot, and the images are
// staged in shared memory CAP at a time: d, the fractional delay and the gain in double, rounded to float once.  Every
// warp then adds the staged images that reach its samples, in slot order, with a compensated float sum.
//
// A tap is evaluated in float from the image's e = d - D (D the nearest integer) and k = i - D:
//   sinc(pi (k - e)) = -(-1)^k sin(pi e) / (pi (k - e)),  cos(pi (k - e) / Tw) = cos(pi k/Tw) cos(pi e/Tw)
//                                                                              + sin(pi k/Tw) sin(pi e/Tw),
// with cos / sin(pi k / Tw) from a per-CTA table, so the large argument pi (k - e) is never rounded; (-1)^i is applied
// once per sample at the end.  A sample's sum depends only on its row's geometry and the tile size: reruns and a batch
// against its items one at a time are bit-identical.
//
// Hybrid (t_d and seed given): the image sources for the early part only, a statistical tail after it.  With n_d =
// ceil(t_d fs), ism_kernel keeps the images with floor(d) < min(L, n_d); tail_kernel then adds, at every sample
// n >= n_d - Tw/2, w(n) sqrt(E(n)) xi(seed, c, n):
//   E(n) = c / (4 pi V fs) (1/4pi) int exp(-n sum_a lambda_a |u_a|) dOmega(u),  lambda_a = -(ln b_a0 + ln b_a1) / L_a
// (L_a in samples), the expected energy per sample of the image arrivals at n; w^2 = 1/2 (1 - cos(pi x)), x = (n - n_d
// + Tw/2 + 1/2) / Tw, over the Tw samples centred on n_d, then 1; xi a standard normal from a SplitMix64 counter
// (key = mix(mix(seed) + c), z = mix(key + n gamma)) by Box-Muller.  A wall with beta = 0 gives E = 0.
//   ln E is evaluated in double at nodes n_k = tau (1.1^k - 1), tau = max(1, 1 / sum lambda) samples, by a tanh-sinh
// rule (65 x 65 points) in u_z (uniform on [0, 1]) and the azimuth over one octant, with its derivative, and
// interpolated between nodes by a cubic Hermite (relative error below 1e-5: (ln E)'''' falls off like 12 / n^4).  Each
// CTA evaluates the nodes its tile spans, so the tail too depends only on its row's geometry, seed and microphone.
//
// Bands (K > 1): K octave bands with their own beta [B, 6, K] and air absorption [B, K] (dB/m).  The
// first K' bands (lower crossover below fs / 2) are computed in one pass: ism_tile<K'> enumerates each tile's images
// once and keeps K' compensated sums per sample, and the rows it writes are r_k - r_{k+1} (k < K' - 1) and r_{K'-1};
// tail_kernel adds each band's tail the same way.  The crossovers (Engine.fftconv) and band_sum_kernel then form
// y = r_{K'-1} + sum_k LP_k * (r_k - r_{k+1}) (DESIGN.md K20 "Bands").
//
// Directivity (mic_dir [B, C, 4] and / or src_dir [B, 4] given): first-order patterns D(u) = p + (1 - p) u.v.  An image
// with offset (X, Y, Z) and parities (q, j, k) is also scaled by D_m((X, Y, Z) / d) D_s(-((1-2q) X, (1-2j) Y,
// (1-2k) Z) / d), in double while it is staged, before its gain is tested for 0; the tail's quadrature weights are
// scaled by M(u) S(u), M = p_m^2 + (1 - p_m)^2 sum_a v_ma^2 u_a^2 (S likewise), the parts of D_m^2 and of D_s^2
// averaged over the parity classes that survive an integrand even in every u_a (DESIGN.md K20 "Directivity").  The
// directional path is a template flag, so the kernels without it are unchanged.
#include "b2a_common.h"

namespace b2a {
namespace rir {

constexpr int WARPS = 4;
constexpr int NT = 32 * WARPS;   // threads per CTA
constexpr int PER = 4;           // samples per lane
constexpr int WS = 32 * PER;     // samples per warp
constexpr int TT = NT * PER;     // samples per CTA (tile)
constexpr int CAP = 256;         // images staged in shared memory at a time
constexpr int TW_MAX = 3072;     // largest window: fs up to 384 kHz
constexpr int FAR = -(1 << 30);  // floor(d) of a staged slot that holds no image
constexpr int MAX_BANDS = 8;     // octave bands, 125 Hz .. 16 kHz

struct Geo {
  const double *room, *src, *mics, *beta;  // beta [B, 6, K]
  const double* td;        // per item: the diffuse tail starts at ceil(td fs); null: images only
  const uint64_t* seed;    // per item: the tail's noise
  const double* air;       // [B, K] air absorption in dB/m; null: none
  int C, L, Tw, max_order;
  int K, KB;               // bands per item in beta / air (1: frequency-flat); bands computed (the first KB)
  double fs, c;
  float* out;              // [KB, B C, L]: rows k < KB - 1 hold r_k - r_{k+1}, row KB - 1 holds r_{KB-1}
  const double* mic_dir;   // [B, C, 4] (p, v_x, v_y, v_z) per microphone; null: omnidirectional
  const double* src_dir;   // [B, 4] the same per item's source; null: omnidirectional
};

struct __align__(16) Img {
  int fl, D;      // floor(d); the nearest integer to d
  float e, gs;    // d - D; -(-1)^D g sin(pi e) / pi
  float g0, ce;   // (-1)^D g (the tap at t = 0); cos(pi e / Tw)
  float se, pad;  // sin(pi e / Tw)
};

// b^|n| by squaring (b^0 = 1, also for b = 0)
__device__ __forceinline__ double ipow(double b, int64_t n) {
  double r = 1.0;
  for (uint64_t e = (uint64_t)(n < 0 ? -n : n); e; e >>= 1, b *= b)
    if (e & 1) r *= b;
  return r;
}

__device__ __forceinline__ int64_t floor_div2(int64_t a) { return a >= 0 ? a / 2 : -((-a + 1) / 2); }

// The image sum of one tile for the first NB bands of a row.  The images are enumerated once; each staged image carries
// the last band's gains in its Img record and the other bands' in bgs, and every band keeps its own compensated sums.
// A band skips an image whose gain rounds to 0 in float, so band NB - 1 adds exactly the images ism_kernel adds for its
// beta, in the same order and with the same arithmetic: with one band this is ism_kernel.  DIR scales every band's
// gain by the patterns of the row's microphone and the item's source (a null table: p = 1).
template <int NB, bool DIR>
__device__ __forceinline__ void ism_tile(const Geo& g) {
  __shared__ float2 tab[TW_MAX + 1];
  __shared__ Img img[CAP];
  __shared__ float2 bgs[NB > 1 ? NB - 1 : 1][CAP];  // bands 0 .. NB - 2: (gs, g0) of the staged images
  __shared__ double wall[6][NB], att[NB];             // beta per wall and band; air absorption per sample of distance
  __shared__ int64_t wtot[WARPS];
  __shared__ double pat[8];  // DIR: p_m, v_m, p_s, v_s (in shared memory: no registers held across the tile)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row = blockIdx.y, b = row / g.C, rows = gridDim.y;
  const int t0 = blockIdx.x * TT, Tw = g.Tw, half = Tw / 2;
  const double ks = g.fs / g.c;  // samples per metre
  const double Lx = g.room[3 * b] * ks, Ly = g.room[3 * b + 1] * ks, Lz = g.room[3 * b + 2] * ks;
  const double sx = g.src[3 * b] * ks, sy = g.src[3 * b + 1] * ks, sz = g.src[3 * b + 2] * ks;
  const double rx = g.mics[3 * row] * ks, ry = g.mics[3 * row + 1] * ks, rz = g.mics[3 * row + 2] * ks;
  const double gscale = ks / (4.0 * M_PI);  // g = product of the betas * gscale / d

  for (int i = tid; i < 6 * NB; i += NT) wall[i / NB][i % NB] = g.beta[(6 * b + i / NB) * g.K + i % NB];
  // 10^(-a d_m / 20) = exp(-att d), d in samples
  for (int i = tid; i < NB; i += NT) att[i] = g.air ? g.air[b * g.K + i] * (M_LN10 / 20.0) / ks : 0.0;
  if (DIR && tid < 8) {
    const double* t = tid < 4 ? g.mic_dir + 4 * row : g.src_dir + 4 * b;
    pat[tid] = (tid < 4 ? g.mic_dir : g.src_dir) ? t[tid & 3] : (tid & 3) == 0;
  }
  for (int i = tid; i <= Tw; i += NT) {
    double s, c;
    sincospi((double)(i - half) / Tw, &s, &c);
    tab[i] = make_float2((float)c, (float)s);
  }
  // the shell: floor(d) in [dlo, dhi)
  const double dlo = (double)t0 - half;
  const double lim = g.td ? fmin((double)g.L, ceil(g.td[b] * g.fs)) : (double)g.L;  // images with floor(d) < lim
  const double dhi = fmin((double)t0 + TT + half - 1, lim);
  if (dhi <= dlo) {  // a tile past the images (only with a diffuse tail)
    for (int bd = 0; bd < NB; ++bd)
      for (int i = t0 + tid; i < min(t0 + TT, g.L); i += NT) g.out[(bd * rows + row) * g.L + i] = 0.f;
    return;
  }
  const double reach = dhi * (1.0 + 1e-12) + 1e-6;  // lines with rho >= reach have no image in the shell
  int64_t Mx = (int64_t)ceil(dhi / (2 * Lx)) + 1, My = (int64_t)ceil(dhi / (2 * Ly)) + 1;
  if (g.max_order >= 0) {  // |2 mx - q| <= max_order
    Mx = min(Mx, (int64_t)(g.max_order / 2 + 1));
    My = min(My, (int64_t)(g.max_order / 2 + 1));
  }
  const int64_t ny = 2 * (2 * My + 1), n_lines = 2 * (2 * Mx + 1) * ny * 2;
  const int wb = t0 + warp * WS;  // the warp's first sample

  float acc[NB][PER], cmp[NB][PER];
#pragma unroll
  for (int bd = 0; bd < NB; ++bd)
#pragma unroll
    for (int s = 0; s < PER; ++s) acc[bd][s] = 0.f, cmp[bd][s] = 0.f;
  __syncthreads();

  for (int64_t l0 = 0; l0 < n_lines; l0 += NT) {
    // this thread's line and its mz runs [za, zb], [zc, zd]
    const int64_t line = l0 + tid;
    int64_t za = 0, zb = -1, zc = 0, zd = -1, mx = 0, my = 0;
    int q = 0, j = 0, k = 0;
    double X = 0, Y = 0, Zc = 0, pxy[NB];
#pragma unroll
    for (int bd = 0; bd < NB; ++bd) pxy[bd] = 0;
    if (line < n_lines) {
      k = (int)(line & 1);
      const int64_t r2 = line >> 1, ix = r2 / ny, iy = r2 % ny;
      q = (int)(ix & 1), mx = (ix >> 1) - Mx, j = (int)(iy & 1), my = (iy >> 1) - My;
      X = (q ? -sx : sx) - rx + 2.0 * mx * Lx;
      Y = (j ? -sy : sy) - ry + 2.0 * my * Ly;
      const double rho2 = X * X + Y * Y;
      int64_t olo = INT64_MIN / 4, ohi = INT64_MAX / 4;
      bool any = rho2 < reach * reach;
      if (g.max_order >= 0) {
        const int64_t rem = g.max_order - (2 * mx - q < 0 ? q - 2 * mx : 2 * mx - q) -
                            (2 * my - j < 0 ? j - 2 * my : 2 * my - j);
        any = any && rem >= 0;
        olo = -floor_div2(rem - k), ohi = floor_div2(k + rem);  // |2 mz - k| <= rem
      }
      if (any) {
        Zc = (k ? -sz : sz) - rz;
        const double zmax = sqrt(reach * reach - rho2);
        const double zmin = dlo > 0 && dlo * dlo > rho2 ? sqrt(dlo * dlo - rho2) : 0.0;
        const double inv = 1.0 / (2 * Lz);
        za = (int64_t)floor((-zmax - Zc) * inv) - 1, zb = (int64_t)ceil((-zmin - Zc) * inv) + 1;
        zc = (int64_t)floor((zmin - Zc) * inv) - 1, zd = (int64_t)ceil((zmax - Zc) * inv) + 1;
        if (zb >= zc - 1) zb = zd, zc = 0, zd = -1;  // one run
        za = max(za, olo), zb = min(zb, ohi), zc = max(zc, olo), zd = min(zd, ohi);
#pragma unroll
        for (int bd = 0; bd < NB; ++bd)
          pxy[bd] = ipow(wall[0][bd], mx - q) * ipow(wall[1][bd], mx) * ipow(wall[2][bd], my - j) *
                    ipow(wall[3][bd], my) * gscale;
      }
    }
    const int64_t n1 = zb >= za ? zb - za + 1 : 0, cnt = n1 + (zd >= zc ? zd - zc + 1 : 0);
    // block scan of the counts: this thread's images take slots [off, off + cnt) of the round
    int64_t v = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    if (lane == 31) wtot[warp] = v;
    __syncthreads();
    int64_t off = v - cnt, total = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      off += w < warp ? wtot[w] : 0;
      total += wtot[w];
    }
    for (int64_t c0 = 0; c0 < total; c0 += CAP) {
      const int64_t lo = off > c0 ? off : c0, hi = min(off + cnt, c0 + CAP);
      for (int64_t sl = lo; sl < hi; ++sl) {
        const int64_t n = sl - off, mz = n < n1 ? za + n : zc + (n - n1);
        const double Z = Zc + 2.0 * mz * Lz;
        const double d = sqrt(X * X + Y * Y + Z * Z);
        const double fl = floor(d);
        double dir = 1.0;
        if (DIR) {  // D_m(u_m) D_s(w): u_m = (X, Y, Z) / d, w the direction the source emitted the ray in
          const volatile double* pt = pat;  // read at the image, not held in registers across the loop
          const double um = X * pt[1] + Y * pt[2] + Z * pt[3];                            // d u_m.v_m
          const double us = -((q ? -X : X) * pt[5] + (j ? -Y : Y) * pt[6] + (k ? -Z : Z) * pt[7]);  // d w.v_s
          dir = (pt[0] * d + (1.0 - pt[0]) * um) * (pt[4] * d + (1.0 - pt[4]) * us) / (d * d);
        }
        double gd[NB];
        bool live = false;
#pragma unroll
        for (int bd = 0; bd < NB; ++bd) {
          gd[bd] = pxy[bd] * ipow(wall[4][bd], mz - k) * ipow(wall[5][bd], mz) / d;
          if (g.air) gd[bd] *= exp(-att[bd] * d);
          if (DIR) gd[bd] *= dir;
          live = live || (float)gd[bd] != 0.f;
        }
        Img im;
        im.fl = FAR;
        if (fl >= dlo && fl < dhi && live) {
          const double D = d - fl > 0.5 ? fl + 1 : fl, e = d - D;
          const bool odd = fmod(D, 2.0) != 0.0;
          double se, ce, sw, cw;
          sincospi(e, &se, &ce);
          sincospi(e / Tw, &sw, &cw);
#pragma unroll
          for (int bd = 0; bd < NB - 1; ++bd) {
            const double sg = odd ? -gd[bd] : gd[bd];  // (-1)^D g
            bgs[bd][sl - c0] = make_float2((float)(-sg * se / M_PI), (float)sg);
          }
          const double sg = odd ? -gd[NB - 1] : gd[NB - 1];
          im.fl = (int)fl, im.D = (int)D, im.e = (float)e, im.gs = (float)(-sg * se / M_PI), im.g0 = (float)sg;
          im.ce = (float)cw, im.se = (float)sw, im.pad = 0.f;
        }
        img[sl - c0] = im;
      }
      __syncthreads();
      const int n_img = (int)min((int64_t)CAP, total - c0);
      for (int m = 0; m < n_img; ++m) {
        const Img im = img[m];
        if (im.fl + half < wb || im.fl - half + 1 >= wb + WS) continue;  // warp-uniform
        float2 gb[NB];
#pragma unroll
        for (int bd = 0; bd < NB - 1; ++bd) gb[bd] = bgs[bd][m];
        gb[NB - 1] = make_float2(im.gs, im.g0);
        const int i0 = wb + lane, u0 = i0 - im.fl + half - 1, k0 = i0 - im.D;
        const float kf0 = (float)k0;
#pragma unroll
        for (int s = 0; s < PER; ++s) {
          if ((unsigned)(u0 + 32 * s) < (unsigned)Tw) {  // sample in the image's window
            const float2 cs = tab[k0 + 32 * s + half];
            const float t = (kf0 + (float)(32 * s)) - im.e;
            const float w = cs.x * im.ce + cs.y * im.se;
            const float r = __fdividef(w * w, t);
#pragma unroll
            for (int bd = 0; bd < NB; ++bd) {
              if (NB > 1 && gb[bd].y == 0.f) continue;  // this band's gain is 0 in float: not added
              const float x = t == 0.f ? gb[bd].y : gb[bd].x * r;
              // Kahan: cmp carries the low part the running sum lost
              const float y = x - cmp[bd][s], tsum = acc[bd][s] + y;
              cmp[bd][s] = (tsum - acc[bd][s]) - y;
              acc[bd][s] = tsum;
            }
          }
        }
      }
      __syncthreads();
    }
    __syncthreads();  // wtot is rewritten by the next round
  }
#pragma unroll
  for (int s = 0; s < PER; ++s) {
    const int i = wb + lane + 32 * s;
    if (i < g.L) {
      float v[NB];
#pragma unroll
      for (int bd = 0; bd < NB; ++bd) v[bd] = (i & 1) ? 0.f - acc[bd][s] : acc[bd][s];
      g.out[((NB - 1) * rows + row) * g.L + i] = v[NB - 1];
#pragma unroll
      for (int bd = 0; bd < NB - 1; ++bd) g.out[(bd * rows + row) * g.L + i] = v[bd] - v[bd + 1];
    }
  }
}

__global__ void __launch_bounds__(NT) ism_kernel(const Geo g) { ism_tile<1, false>(g); }
__global__ void __launch_bounds__(NT) ism_dir_kernel(const Geo g) { ism_tile<1, true>(g); }

// one CTA per SM is enough to let ptxas keep every band's sums in registers (no spills up to NB = 8)
template <int NB>
__global__ void __launch_bounds__(NT, 1) ism_bands_kernel(const Geo g) { ism_tile<NB, false>(g); }
template <int NB>
__global__ void __launch_bounds__(NT, 1) ism_bands_dir_kernel(const Geo g) { ism_tile<NB, true>(g); }


constexpr int QK = 32;                // tanh-sinh: 2 QK + 1 points per dimension, steps of 3 / QK
constexpr int QM = 2 * QK + 1;
constexpr int QN = QM * QM;
constexpr double GROW = 1.1;          // envelope nodes n_k = tau (GROW^k - 1)
constexpr int NK = 72;                // nodes one tile spans: at most ln(TT + 1) / ln(GROW) + 3
constexpr uint64_t GAMMA = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // the SplitMix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ int node_of(double n, double tau, double lr) { return (int)floor(log1p(n / tau) / lr); }

// Adds the tail of every computed band to the rows ism_tile wrote: band k's envelope is E(n; beta_k) exp(-2 att_k n)
// (the air's 10^(-a_k (c n / fs) / 10), added to ln E at the sample, exactly), its noise xi(seed, c, n) is shared by the
// bands, so row KB - 1 gets v_{KB-1} and row k < KB - 1 gets v_k - v_{k+1}.  The bands are walked from the last one
// down, each with the node evaluation of the flat tail; with one band this is the flat tail.  DIR weights the point
// (z, phi) by M S = (ma[z] + mb[z] mc[phi]) (sa[z] + sb[z] sc[phi]): with u_x^2 = (1 - z^2) cos^2 phi,
// u_y^2 = (1 - z^2) sin^2 phi, u_z^2 = z^2, ma = p^2 + (1 - p)^2 v_z^2 z^2, mb = (1 - p)^2 (1 - z^2),
// mc = v_x^2 cos^2 phi + v_y^2 sin^2 phi (the microphone's pattern; sa, sb, sc the source's).
template <bool DIR>
__device__ __forceinline__ void tail_tile(const Geo& g) {
  __shared__ double qa[QM], qr[QM], qw[QM], pb[QM], pw[QM];  // z: lambda_z z, sqrt(1 - z^2), weight; azimuth
  __shared__ double dw[DIR ? 6 : 1][QM];                     // DIR: ma, mb, mc, sa, sb, sc
  __shared__ double nn[NK], nf[NK], nd[NK];                  // node, ln of the direction mean, its derivative
  __shared__ double part[WARPS][2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row = blockIdx.y, b = row / g.C, rows = gridDim.y;
  const int c = (int)(row % g.C), t0 = blockIdx.x * TT, half = g.Tw / 2;
  const double n_d = ceil(g.td[b] * g.fs), s_d = fmax(n_d - half, 0.0);  // the tail's first sample
  const int end = min(t0 + TT, g.L);
  if ((double)end <= s_d) return;
  const int start = (int)s_d;
  const double ks = g.fs / g.c;
  const double scale = g.c / (4.0 * M_PI * g.room[3 * b] * g.room[3 * b + 1] * g.room[3 * b + 2] * g.fs);
  const int first = max(t0, start);
  const double lr = log(GROW);
  if (DIR) {  // the patterns' tables; the first band with a tail synchronises before reading them
    for (int i = tid; i < 2 * QM; i += NT) {
      const int e = i / QM, t = i - e * QM;  // end: 0 the microphone, 1 the source
      const double* d = e ? g.src_dir : g.mic_dir;
      const double* pv = d ? d + 4 * (e ? b : row) : nullptr;
      const double p = pv ? pv[0] : 1.0, a = (1.0 - p) * (1.0 - p);
      const double vx = pv ? pv[1] : 0.0, vy = pv ? pv[2] : 0.0, vz = pv ? pv[3] : 0.0;
      const double h = 3.0 / QK, s = (t - QK) * h, x = 0.5 * (1.0 + tanh(0.5 * M_PI * sinh(s)));
      double sn, co;
      sincospi(0.5 * x, &sn, &co);
      dw[3 * e][t] = p * p + a * vz * vz * x * x;
      dw[3 * e + 1][t] = a * fmax(0.0, 1.0 - x * x);
      dw[3 * e + 2][t] = vx * vx * co * co + vy * vy * sn * sn;
    }
  }

  // this thread's samples first + tid + NT s: the Box-Muller radius and cosine of each
  const uint64_t key = mix64(mix64(g.seed[b]) + (uint64_t)c);
  double rad[PER], cosv[PER];
  float prev[PER];
#pragma unroll
  for (int s = 0; s < PER; ++s) {
    const int i = first + tid + NT * s;
    const uint64_t z = mix64(key + (uint64_t)i * GAMMA);
    const double u1 = ((double)(z >> 32) + 0.5) * 0x1p-32, u2 = (double)(z & 0xffffffffull) * 0x1p-32;
    double sn, co;
    sincospi(2.0 * u2, &sn, &co);
    rad[s] = sqrt(-2.0 * log(u1)), cosv[s] = co, prev[s] = 0.f;
  }

  for (int bd = g.KB - 1; bd >= 0; --bd) {
    double be[6];
    bool zero = false;
    for (int a = 0; a < 6; ++a) {
      be[a] = g.beta[(6 * b + a) * g.K + bd];
      zero = zero || be[a] == 0.0;  // E = 0
    }
    const double ea = g.air ? 2.0 * g.air[b * g.K + bd] * (M_LN10 / 20.0) / ks : 0.0;  // energy, per sample
    int k_lo = 0, k_hi = 1;
    double tau = 1.0;
    if (!zero) {
      const double lx = -(log(be[0]) + log(be[1])) / (g.room[3 * b] * ks);
      const double ly = -(log(be[2]) + log(be[3])) / (g.room[3 * b + 1] * ks);
      const double lz = -(log(be[4]) + log(be[5])) / (g.room[3 * b + 2] * ks);
      const double m = fmin(lx, fmin(ly, lz));  // sum lambda_a |u_a| >= m on the unit sphere
      tau = fmax(1.0, fmin(1.0 / (lx + ly + lz), (double)g.L));
      k_lo = node_of(first, tau, lr);
      k_hi = max(k_lo + 1, min(node_of(end - 1, tau, lr) + 1, k_lo + NK - 1));

      for (int i = tid; i < QM; i += NT) {
        const double h = 3.0 / QK, t = (i - QK) * h, a = 0.5 * M_PI * sinh(t), ch = cosh(a);
        const double x = 0.5 * (1.0 + tanh(a)), w = 0.25 * M_PI * h * cosh(t) / (ch * ch);
        double s, co;
        sincospi(0.5 * x, &s, &co);
        qa[i] = lz * x, qr[i] = sqrt(fmax(0.0, 1.0 - x * x)), qw[i] = w * (2.0 / M_PI);
        pb[i] = lx * co + ly * s, pw[i] = 0.5 * M_PI * w;
      }
      __syncthreads();
      for (int k = k_lo; k <= k_hi; ++k) {
        const double n = tau * expm1(k * lr);
        double s0 = 0.0, s1 = 0.0;
        for (int q = tid; q < QN; q += NT) {
          const int i = q / QM, j = q - i * QM;
          const double sg = qa[i] + qr[i] * pb[j] - m;
          double e = qw[i] * pw[j] * exp(-n * sg);
          if (DIR) e *= (dw[0][i] + dw[1][i] * dw[2][j]) * (dw[3][i] + dw[4][i] * dw[5][j]);
          s0 += e, s1 += e * sg;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, o);
          s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        }
        if (lane == 0) part[warp][0] = s0, part[warp][1] = s1;
        __syncthreads();
        if (tid == 0) {
          double S0 = 0.0, S1 = 0.0;
          for (int w = 0; w < WARPS; ++w) S0 += part[w][0], S1 += part[w][1];
          const bool ok = S0 > 0.0;  // else every term underflowed: E is 0 to double precision
          nn[k - k_lo] = n, nf[k - k_lo] = ok ? log(S0) - n * m : -1e300, nd[k - k_lo] = ok ? -m - S1 / S0 : 0.0;
        }
        __syncthreads();
      }
    }

#pragma unroll
    for (int s = 0; s < PER; ++s) {
      const int i = first + tid + NT * s;
      if (i >= end) break;
      float v = 0.f;
      if (!zero) {
        const int k = min(max(node_of(i, tau, lr), k_lo), k_hi - 1) - k_lo;
        const double h = nn[k + 1] - nn[k], t = (i - nn[k]) / h, t2 = t * t, t3 = t2 * t;
        const double f = (2 * t3 - 3 * t2 + 1) * nf[k] + (t3 - 2 * t2 + t) * h * nd[k] + (3 * t2 - 2 * t3) * nf[k + 1] +
                         (t3 - t2) * h * nd[k + 1];
        double amp = sqrt(scale * exp(f - ea * i));
        const double x = (i - n_d + half + 0.5) / g.Tw;
        if (x < 1.0) {
          double sn, co;
          sincospi(x, &sn, &co);
          amp *= sqrt(0.5 * (1.0 - co));
        }
        v = (float)(amp * rad[s] * cosv[s]);
      }
      float* o = g.out + (bd * rows + row) * (int64_t)g.L;
      if (bd == g.KB - 1) {
        if (!zero) o[i] += v;
      } else {
        o[i] += v - prev[s];
      }
      prev[s] = v;
    }
    __syncthreads();  // the next band rewrites the tables and the nodes
  }
}

__global__ void __launch_bounds__(NT) tail_kernel(const Geo g) { tail_tile<false>(g); }
__global__ void __launch_bounds__(NT) tail_dir_kernel(const Geo g) { tail_tile<true>(g); }

// y = r_last + conv_0 + conv_1 + ... (the crossovers' outputs, added in band order), one row per blockIdx.y.  The
// crossovers run on the FFT engine, whose rounding spreads over whole blocks, so the samples before the first one any
// band can reach are written as the exact zeros they are: every image is at least as far as the direct path d, so
// nothing reaches n < floor(d) - Tw/2 + 1 - half, nor, with a tail, n < n_d - Tw/2 - half; one sample of margin is
// kept for the rounding of d.
__global__ void __launch_bounds__(256) band_sum_kernel(const Geo g, int half, const float* __restrict__ conv,
                                                       int n_conv, float* __restrict__ y) {
  const int64_t row = blockIdx.y, b = row / g.C, rows = gridDim.y, n = rows * (int64_t)g.L;
  const double ks = g.fs / g.c;
  const double X = (g.src[3 * b] - g.mics[3 * row]) * ks, Y = (g.src[3 * b + 1] - g.mics[3 * row + 1]) * ks;
  const double Z = (g.src[3 * b + 2] - g.mics[3 * row + 2]) * ks;
  double z0 = floor(sqrt(X * X + Y * Y + Z * Z)) - g.Tw / 2 - half;
  if (g.td) z0 = fmin(z0, fmax(ceil(g.td[b] * g.fs) - g.Tw / 2, 0.0) - half - 1);
  const float* last = g.out + (int64_t)n_conv * n + row * (int64_t)g.L;
  float* o = y + row * (int64_t)g.L;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.L; i += gridDim.x * blockDim.x) {
    float v = 0.f;
    if ((double)i >= z0) {
      v = last[i];
      for (int k = 0; k < n_conv; ++k) v += conv[k * n + row * (int64_t)g.L + i];
    }
    o[i] = v;
  }
}

}  // namespace rir
}  // namespace b2a

using namespace b2a::rir;

static Geo geo(const double* room, const double* src, const double* mics, const double* beta, int C, int64_t L,
               double fs, double c, int max_order, float* out) {
  Geo g;
  g.room = room, g.src = src, g.mics = mics, g.beta = beta, g.td = nullptr, g.seed = nullptr, g.air = nullptr;
  g.mic_dir = nullptr, g.src_dir = nullptr;
  g.C = C, g.L = (int)L, g.K = 1, g.KB = 1, g.max_order = max_order, g.Tw = 2 * (int)floor(0.004 * fs + 0.5), g.fs = fs, g.c = c, g.out = out;
  return g;
}

// Bands whose lower crossover 125 2^(k - 1/2) Hz is below fs / 2 (band 0 always)
static int bands_kept(int K, double fs) {
  int kb = 1;
  while (kb < K && 125.0 * exp2(kb - 0.5) < 0.5 * fs) ++kb;
  return kb;
}

template <int NB>
static void launch_bands(const dim3& grid, const Geo& g, bool dir, void* stream) {
  if (dir)
    B2A_LAUNCH(ism_bands_dir_kernel<NB>, grid, dim3(NT), 0, stream, g);
  else
    B2A_LAUNCH(ism_bands_kernel<NB>, grid, dim3(NT), 0, stream, g);
}

extern "C" int b2a_rir_bands_kept(int K, double fs) {
  if (K < 1 || K > MAX_BANDS || !(fs > 0.0)) return 0;
  return bands_kept(K, fs);
}

extern "C" int b2a_rir_directional_f32(const double* room, const double* src, const double* mics, const double* beta,
                                       const double* air, const double* t_d, const uint64_t* seed,
                                       const double* mic_dir, const double* src_dir, int64_t B, int C, int K, int64_t L,
                                       double fs, double c, int max_order, float* out, void* stream) {
  B2A_REQUIRE(room && src && mics && beta && out, B2A_E_INVALID, "rir: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && L >= 1, B2A_E_INVALID, "rir: bad shape B=%lld C=%d L=%lld", (long long)B, C,
              (long long)L);
  B2A_REQUIRE(K >= 1 && K <= MAX_BANDS, B2A_E_INVALID, "rir: K=%d bands; 1 .. %d are supported", K, MAX_BANDS);
  B2A_REQUIRE(B * C * K <= 65535, B2A_E_INVALID, "rir: %lld rows (items x microphones x bands); at most 65535",
              (long long)(B * C * K));
  B2A_REQUIRE(L <= (1 << 30), B2A_E_INVALID, "rir: L=%lld; at most 2^30 samples", (long long)L);
  B2A_REQUIRE(fs >= 125.0 && fs <= 384000.0, B2A_E_INVALID, "rir: fs=%g; 125 .. 384000 Hz are supported", fs);
  B2A_REQUIRE(c > 0.0 && c < 1e30, B2A_E_INVALID, "rir: sound speed %g must be positive and finite", c);
  B2A_REQUIRE(max_order >= -1, B2A_E_INVALID, "rir: max_order=%d must be >= -1", max_order);
  B2A_REQUIRE(!t_d == !seed, B2A_E_INVALID, "rir: a diffuse tail needs both t_d and seed");
  B2A_REQUIRE(!t_d || max_order == -1, B2A_E_INVALID, "rir: max_order=%d with a diffuse tail", max_order);
  Geo g = geo(room, src, mics, beta, C, L, fs, c, max_order, out);
  g.air = air, g.td = t_d, g.seed = seed, g.K = K, g.KB = bands_kept(K, fs);
  g.mic_dir = mic_dir, g.src_dir = src_dir;
  const bool dir = mic_dir || src_dir;
  const dim3 grid((unsigned)((L + TT - 1) / TT), (unsigned)(B * C));
  switch (g.KB) {
    case 1:
      if (dir)
        B2A_LAUNCH(ism_dir_kernel, grid, dim3(NT), 0, stream, g);
      else
        B2A_LAUNCH(ism_kernel, grid, dim3(NT), 0, stream, g);
      break;
    case 2: launch_bands<2>(grid, g, dir, stream); break;
    case 3: launch_bands<3>(grid, g, dir, stream); break;
    case 4: launch_bands<4>(grid, g, dir, stream); break;
    case 5: launch_bands<5>(grid, g, dir, stream); break;
    case 6: launch_bands<6>(grid, g, dir, stream); break;
    case 7: launch_bands<7>(grid, g, dir, stream); break;
    default: launch_bands<8>(grid, g, dir, stream); break;
  }
  B2A_CUDA_OK(cudaGetLastError());
  if (t_d) {
    if (dir)
      B2A_LAUNCH(tail_dir_kernel, grid, dim3(NT), 0, stream, g);
    else
      B2A_LAUNCH(tail_kernel, grid, dim3(NT), 0, stream, g);
    B2A_CUDA_OK(cudaGetLastError());
  }
  return B2A_OK;
}

extern "C" int b2a_rir_f32(const double* room, const double* src, const double* mics, const double* beta,
                           const double* air, const double* t_d, const uint64_t* seed, int64_t B, int C, int K,
                           int64_t L, double fs, double c, int max_order, float* out, void* stream) {
  return b2a_rir_directional_f32(room, src, mics, beta, air, t_d, seed, nullptr, nullptr, B, C, K, L, fs, c, max_order,
                                 out, stream);
}

extern "C" int b2a_rir_band_sum_f32(const double* src, const double* mics, const double* t_d, int64_t B, int C,
                                    int64_t L, double fs, double c, int half, const float* bands, const float* conv,
                                    int n_conv, float* out, void* stream) {
  B2A_REQUIRE(src && mics && bands && conv && out, B2A_E_INVALID, "rir_band_sum: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && L >= 1 && B * C <= 65535 && L <= (1 << 30) && n_conv >= 1 && n_conv < MAX_BANDS &&
                  half >= 0,
              B2A_E_INVALID, "rir_band_sum: bad shape B=%lld C=%d L=%lld n_conv=%d half=%d", (long long)B, C,
              (long long)L, n_conv, half);
  B2A_REQUIRE(fs >= 125.0 && fs <= 384000.0 && c > 0.0 && c < 1e30, B2A_E_INVALID, "rir_band_sum: fs=%g c=%g", fs, c);
  Geo g = geo(nullptr, src, mics, nullptr, C, L, fs, c, -1, const_cast<float*>(bands));
  g.td = t_d;
  const int64_t bx = (L + 255) / 256;
  const dim3 grid((unsigned)(bx < 64 ? bx : 64), (unsigned)(B * C));
  B2A_LAUNCH(band_sum_kernel, grid, dim3(256), 0, stream, g, half, conv, n_conv, out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
