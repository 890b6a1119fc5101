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

struct Geo {
  const double *room, *src, *mics, *beta;
  int C, L, Tw, max_order;
  double fs, c;
  float* out;
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

__global__ void __launch_bounds__(NT) ism_kernel(const Geo g) {
  __shared__ float2 tab[TW_MAX + 1];
  __shared__ Img img[CAP];
  __shared__ int64_t wtot[WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row = blockIdx.y, b = row / g.C;
  const int t0 = blockIdx.x * TT, Tw = g.Tw, half = Tw / 2;
  const double ks = g.fs / g.c;  // samples per metre
  const double Lx = g.room[3 * b] * ks, Ly = g.room[3 * b + 1] * ks, Lz = g.room[3 * b + 2] * ks;
  const double sx = g.src[3 * b] * ks, sy = g.src[3 * b + 1] * ks, sz = g.src[3 * b + 2] * ks;
  const double rx = g.mics[3 * row] * ks, ry = g.mics[3 * row + 1] * ks, rz = g.mics[3 * row + 2] * ks;
  const double* be = g.beta + 6 * b;
  const double bx0 = be[0], bx1 = be[1], by0 = be[2], by1 = be[3], bz0 = be[4], bz1 = be[5];
  const double gscale = ks / (4.0 * M_PI);  // g = product of the betas * gscale / d

  for (int i = tid; i <= Tw; i += NT) {
    double s, c;
    sincospi((double)(i - half) / Tw, &s, &c);
    tab[i] = make_float2((float)c, (float)s);
  }
  // the shell: floor(d) in [dlo, dhi)
  const double dlo = (double)t0 - half;
  const double dhi = fmin((double)t0 + TT + half - 1, (double)g.L);
  const double reach = dhi * (1.0 + 1e-12) + 1e-6;  // lines with rho >= reach have no image in the shell
  int64_t Mx = (int64_t)ceil(dhi / (2 * Lx)) + 1, My = (int64_t)ceil(dhi / (2 * Ly)) + 1;
  if (g.max_order >= 0) {  // |2 mx - q| <= max_order
    Mx = min(Mx, (int64_t)(g.max_order / 2 + 1));
    My = min(My, (int64_t)(g.max_order / 2 + 1));
  }
  const int64_t ny = 2 * (2 * My + 1), n_lines = 2 * (2 * Mx + 1) * ny * 2;
  const int wb = t0 + warp * WS;  // the warp's first sample

  float acc[PER], cmp[PER];
#pragma unroll
  for (int s = 0; s < PER; ++s) acc[s] = 0.f, cmp[s] = 0.f;
  __syncthreads();

  for (int64_t l0 = 0; l0 < n_lines; l0 += NT) {
    // this thread's line and its mz runs [za, zb], [zc, zd]
    const int64_t line = l0 + tid;
    int64_t za = 0, zb = -1, zc = 0, zd = -1, mx = 0, my = 0;
    int q = 0, j = 0, k = 0;
    double X = 0, Y = 0, Zc = 0, pxy = 0;
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
        pxy = ipow(bx0, mx - q) * ipow(bx1, mx) * ipow(by0, my - j) * ipow(by1, my) * gscale;
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
        const double gd = pxy * ipow(bz0, mz - k) * ipow(bz1, mz) / d;
        Img im;
        im.fl = FAR;
        if (fl >= dlo && fl < dhi && (float)gd != 0.f) {
          const double D = d - fl > 0.5 ? fl + 1 : fl, e = d - D;
          const double sg = fmod(D, 2.0) != 0.0 ? -gd : gd;  // (-1)^D g
          double se, ce, sw, cw;
          sincospi(e, &se, &ce);
          sincospi(e / Tw, &sw, &cw);
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
        const int i0 = wb + lane, u0 = i0 - im.fl + half - 1, k0 = i0 - im.D;
        const float kf0 = (float)k0;
#pragma unroll
        for (int s = 0; s < PER; ++s) {
          if ((unsigned)(u0 + 32 * s) < (unsigned)Tw) {  // sample in the image's window
            const float2 cs = tab[k0 + 32 * s + half];
            const float t = (kf0 + (float)(32 * s)) - im.e;
            const float w = cs.x * im.ce + cs.y * im.se;
            const float x = t == 0.f ? im.g0 : im.gs * __fdividef(w * w, t);
            // Kahan: cmp carries the low part the running sum lost
            const float y = x - cmp[s], tsum = acc[s] + y;
            cmp[s] = (tsum - acc[s]) - y;
            acc[s] = tsum;
          }
        }
      }
      __syncthreads();
    }
    __syncthreads();  // wtot is rewritten by the next round
  }
  float* o = g.out + row * (int64_t)g.L;
#pragma unroll
  for (int s = 0; s < PER; ++s) {
    const int i = wb + lane + 32 * s;
    if (i < g.L) o[i] = (i & 1) ? 0.f - acc[s] : acc[s];
  }
}

}  // namespace rir
}  // namespace b2a

using namespace b2a::rir;

extern "C" int b2a_rir_ism_f32(const double* room, const double* src, const double* mics, const double* beta, int64_t B,
                               int C, int64_t L, double fs, double c, int max_order, float* out, void* stream) {
  B2A_REQUIRE(room && src && mics && beta && out, B2A_E_INVALID, "rir_ism: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && L >= 1, B2A_E_INVALID, "rir_ism: bad shape B=%lld C=%d L=%lld", (long long)B, C,
              (long long)L);
  B2A_REQUIRE(B * C <= 65535, B2A_E_INVALID, "rir_ism: %lld rows (items x microphones); at most 65535 per call",
              (long long)(B * C));
  B2A_REQUIRE(L <= (1 << 30), B2A_E_INVALID, "rir_ism: L=%lld; at most 2^30 samples", (long long)L);
  B2A_REQUIRE(fs >= 125.0 && fs <= 384000.0, B2A_E_INVALID, "rir_ism: fs=%g; 125 .. 384000 Hz are supported", fs);
  B2A_REQUIRE(c > 0.0 && c < 1e30, B2A_E_INVALID, "rir_ism: sound speed %g must be positive and finite", c);
  B2A_REQUIRE(max_order >= -1, B2A_E_INVALID, "rir_ism: max_order=%d must be >= -1", max_order);
  Geo g;
  g.room = room, g.src = src, g.mics = mics, g.beta = beta, g.C = C, g.L = (int)L, g.max_order = max_order;
  g.Tw = 2 * (int)floor(0.004 * fs + 0.5), g.fs = fs, g.c = c, g.out = out;
  const dim3 grid((unsigned)((L + TT - 1) / TT), (unsigned)(B * C));
  B2A_LAUNCH(ism_kernel, grid, dim3(NT), 0, stream, g);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
