// spectral_tc.cu -- the fused framing -> window -> real DFT -> |.| -> banded mel -> post-op kernel with the DFT's
// first (radix-128) stage on the Hopper tensor cores (wgmma.mma_async, fp16 operands in shared memory, fp32
// accumulators in registers).
//
// Same contract as spectral_warp_kernel<10,0> (spectral.cu): replaces torch.stft + abs + mel matmul + log of
// ref:audiotools/core/audio_signal.py:1195-1202,1355,1367 and ref:audiotools/metrics/spectral.py:187-190 for
// window_length 2048, and (optionally) the x*gain of EffectMixin.normalize (ref:audiotools/core/effects.py:219).
//
// Factorisation of the 2048-point real DFT, n = 16 a + b (a < 128, b < 16), k = c + 128 d (c < 128, d < 16):
//   X[c + 128 d] = sum_b W16^{bd} . W2048^{bc} . Y_b[c],   Y_b[c] = sum_a xw[16 a + b] W128^{ac}
// * Y_b[c] for c = 0..63 (the other half follows from xw being real) is ONE GEMM on the tensor cores:
//   D[128 rows x (16 groups x 16 frames)] = F[128 x 128] . XW[128 x 256].  Row R of F (16-row slab s = R / 16,
//   j = R % 16) is c = 8 s + j % 8, Re for j < 8 (64 cos) and Im for j >= 8 (-64 sin); the Im row of c = 0 (Im Y[0] = 0)
//   carries c = 64 instead (64 (-1)^a).  With this order the wgmma accumulator fragment of a thread holds Re AND Im of
//   one c for two consecutive frames of every group b.  Operands are fp16 with an exact two-term split of BOTH sides
//   (x = h1 + h2, F = F1 + F2; products h1 F1 + h2 F1 + h1 F2, fp32 accumulation): fp32 quality; the samples of a tile
//   are pre-scaled by a power of two so that max |x| lands in [512, 1024) and F by 64, which keeps both correction
//   terms out of the fp16 subnormals.  F1, F2 are the A operand (built once per CTA), the windowed frames the B
//   operand, both in the canonical no-swizzle K-major shared-memory layout.
// * Warpgroup g (of 4) computes rows 64 (g % 2) .. +64 for frames 8 (g / 2) .. +8 of all 16 groups; the groups are
//   staged in two halves of 8 (one 64 KB operand buffer), 24 wgmma m64n64k16 per half and warpgroup.
// * the second stage -- twiddle by W2048^{bc} and a 16-point complex DFT over b -- runs in registers straight from
//   the accumulators, one thread per (c, frame).  Outputs d >= 8 are the mirrored bins 2048 - k.  c = 0 / c = 64
//   (real inputs) pack the two frames of the thread into one complex DFT and separate them with the even/odd split.
// * |X| of the 16 frames of a tile goes to shared memory (on top of the dead B operand), the banded FP32 mel
//   projection + post-op + coalesced tile store are those of spectral.cu.
//
// Per 16-frame tile: 1 TMA-staged span (19 bulk copies, padded per 512 samples -> conflict-free strided reads).
#ifndef B2A_SIM
#include <cuda_fp16.h>
#endif

#include "b2a_common.h"
#include "fft_warp.cuh"
#include "spectral_internal.h"

namespace b2a {
namespace spectral {

namespace tc {

constexpr int NFFT = 2048;
constexpr int FR = 16;        // frames per tile = N of the MMA
constexpr int NG = 16;        // groups b
constexpr int KA = 128;       // a per group = K of a group's GEMM
constexpr int THREADS = 512;
constexpr int NWARP = THREADS / 32;
constexpr int XBS = 1156;     // floats per |X| slot (1025 + band over-read slack; 1156 % 32 == 4: frames interleave)
constexpr int BLK = 512;      // span padding granule (samples)
constexpr int BLKP = BLK + 4; // padded granule
constexpr int B_PART = 8 * 4096;  // bytes of one fp16 part (hi or lo) of one half (8 groups) of the B operand
constexpr int F_PART = 128 * 256;  // bytes of one fp16 part (F1 or F2) of the A operand

__host__ __device__ __forceinline__ int pad_idx(int i) { return i + 4 * (i >> 9); }

#ifdef B2A_SIM
static inline float h2f(uint16_t h) { _Float16 v; memcpy(&v, &h, 2); return (float)v; }
static inline uint16_t f2h(float f) { _Float16 v = (_Float16)f; uint16_t h; memcpy(&h, &v, 2); return h; }
#endif

__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
#ifdef B2A_SIM
  return (uint32_t)f2h(lo) | ((uint32_t)f2h(hi) << 16);
#else
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
#endif
}
__device__ __forceinline__ float f16lo_to_f32(uint32_t w) {
#ifdef B2A_SIM
  return h2f((uint16_t)(w & 0xffff));
#else
  return __half2float(__ushort_as_half((unsigned short)(w & 0xffff)));
#endif
}
__device__ __forceinline__ float f16hi_to_f32(uint32_t w) {
#ifdef B2A_SIM
  return h2f((uint16_t)(w >> 16));
#else
  return __half2float(__ushort_as_half((unsigned short)(w >> 16)));
#endif
}
// two-term fp16 split of a pair: hi = rn(v), lo = rn(v - hi)  (v - hi is exact in fp32)
__device__ __forceinline__ void split2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2(v0, v1);
  lo = pack_f16x2(v0 - f16lo_to_f32(hi), v1 - f16hi_to_f32(hi));
}

__device__ __forceinline__ void fence_async_smem() {
#ifndef B2A_SIM
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}

#ifndef B2A_SIM
// wgmma shared-memory matrix descriptor: canonical no-swizzle K-major layout of 8-row x 16-byte core matrices,
// LBO = bytes between the two core matrices along K, SBO = bytes between consecutive 8-row groups
__device__ __forceinline__ uint64_t smem_desc(const void* p, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  return (uint64_t)((a >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);  // base offset 0, layout type 0 = no swizzle
}
#endif
// Keeps the compiler from moving accesses of the accumulators across the wgmma fence / wait around them.
__device__ __forceinline__ void fence_acc(float (&d)[32]) {
#ifndef B2A_SIM
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
#else
  (void)d;
#endif
}
__device__ __forceinline__ void wgmma_fence() {
#ifndef B2A_SIM
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#endif
}
__device__ __forceinline__ void wgmma_commit() {
#ifndef B2A_SIM
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
#endif
}
__device__ __forceinline__ void wgmma_wait_all() {
#ifndef B2A_SIM
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#endif
}
// d[64 x 64] (+)= A[64 x 16] . B[64 x 16]^T for the calling warpgroup, fp16 in, fp32 accumulate.  A: 64 rows of F at
// a_smem (8-row groups 2048 B apart), B: 64 rows n = 8 i + r (group i, frame r) at b_smem (8-row groups 4096 B apart);
// both K-major, the two 8-wide K chunks 128 B apart.  Thread (warp w of the group, lane l) receives
// d[4 i + 2 h + e] = D[16 w + l / 4 + 8 h][8 i + 2 (l % 4) + e].  Under the CPU simulator each thread computes its
// own fragment from the same shared-memory bytes.
__device__ __forceinline__ void wgmma_64x64x16(float (&d)[32], const unsigned char* a_smem, const unsigned char* b_smem,
                                               int accumulate) {
#ifdef B2A_SIM
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  for (int i = 0; i < 8; ++i)
    for (int h = 0; h < 2; ++h)
      for (int e = 0; e < 2; ++e) {
        const int m = 16 * w + (l >> 2) + 8 * h, n = 8 * i + 2 * (l & 3) + e;
        float acc = accumulate ? d[4 * i + 2 * h + e] : 0.f;
        for (int k = 0; k < 16; ++k) {
          uint16_t ah, bh;
          memcpy(&ah, a_smem + (m >> 3) * 2048 + (k >> 3) * 128 + (m & 7) * 16 + (k & 7) * 2, 2);
          memcpy(&bh, b_smem + (n >> 3) * 4096 + (k >> 3) * 128 + (n & 7) * 16 + (k & 7) * 2, 2);
          acc += h2f(ah) * h2f(bh);
        }
        d[4 * i + 2 * h + e] = acc;
      }
#else
  const uint64_t da = smem_desc(a_smem, 128, 2048), db = smem_desc(b_smem, 128, 4096);
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(accumulate));
#endif
}
// arm `bar` with the byte count of the whole span, then one bulk copy per 512-sample granule (padded destination)
__device__ __forceinline__ void tma_span(float* sp, const float* src, int span, unsigned long long* bar) {
#ifdef B2A_SIM
  for (int i = 0; i < span; ++i) sp[pad_idx(i)] = src[i];
  (void)bar;
#else
  const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((unsigned)span * 4u) : "memory");
  for (int i = 0; i < span; i += BLK) {
    const unsigned bytes = (unsigned)min(BLK, span - i) * 4u;
    const unsigned d = (unsigned)__cvta_generic_to_shared(sp + pad_idx(i));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d),
                 "l"(src + i), "r"(bytes), "r"(b) : "memory");
  }
#endif
}

struct Smem {
  int off_b, off_f, off_span, off_win, off_tw, off_mel, off_mpk, off_mseg, off_red, total;
};
static Smem smem_layout(const Params& p) {
  Smem s;
  auto al = [](int v) { return (v + 127) & ~127; };
  int o = 0;
  s.off_b = o; o = al(o + max(2 * B_PART, FR * XBS * 4));   // B operand (hi, lo) of a half; later the |X| slots
  s.off_f = o; o = al(o + 2 * F_PART);                       // A operand F1, F2
  const int nblk = (p.span + BLK - 1) / BLK;
  s.off_span = o; o = al(o + nblk * BLKP * 4);
  s.off_win = o; o = al(o + NFFT * 4);
  s.off_tw = o; o = al(o + NG * 128 * 8);
  s.off_mel = o; o = al(o + p.n_mels * (FR + 1) * 4);
  s.off_mpk = o; o = al(o + p.mel_packed_len * 4);
  s.off_mseg = o; o = al(o + p.n_mels * 16);
  s.off_red = o; o = al(o + 256);
  s.total = o;
  return s;
}

struct KParams {
  Params p;
  Smem s;
};

__global__ void __launch_bounds__(THREADS, 1) spectral_tc_kernel(const B2A_GRID_CONSTANT KParams kp) {
  const Params& p = kp.p;
  B2A_DYN_SMEM(smem);
  unsigned char* bop = smem + kp.s.off_b;
  unsigned char* fop = smem + kp.s.off_f;
  float* xs = reinterpret_cast<float*>(smem + kp.s.off_b);  // |X| slots alias the B operand (dead after the MMAs)
  float* sp = reinterpret_cast<float*>(smem + kp.s.off_span);
  float* wsc = reinterpret_cast<float*>(smem + kp.s.off_win);
  float2* tw = reinterpret_cast<float2*>(smem + kp.s.off_tw);  // [b][row]
  float* melt = reinterpret_cast<float*>(smem + kp.s.off_mel);
  float* mpk = reinterpret_cast<float*>(smem + kp.s.off_mpk);
  int4* mseg = reinterpret_cast<int4*>(smem + kp.s.off_mseg);
  float* red = reinterpret_cast<float*>(smem + kp.s.off_red);

  __shared__ __align__(8) unsigned long long s_bar_tma;
  __shared__ int s_clamp;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rb = (warp >> 2) & 1, fh = warp >> 3;        // warpgroup: rows 64 rb .. +64, frames 8 fh .. +8
  const int c = 32 * rb + 8 * (warp & 3) + (lane >> 2);  // DFT-128 bin of this thread's accumulator rows
  const int f0 = 8 * fh + 2 * (lane & 3);                // ... and its two frames f0, f0 + 1
  const int hop = p.hop, F = NFFT / 2 + 1;
  const int total_tiles = p.rows * p.n_tiles;

  if (tid == 0) mbar_init(&s_bar_tma, 1);
  __syncthreads();

  // ---- first tile's span in flight while the tables are built
  int t = blockIdx.x;
  bool by_tma = false;
  auto stage = [&](int tt) -> bool {
    const int rw = tt / p.n_tiles, tile = tt - rw * p.n_tiles;
    const int ws = (tile * FR + p.drop_edge) * hop + p.origin;
    const float* xr = p.x + (size_t)rw * (size_t)p.T;
    const bool interior = (ws >= 0) && (ws + p.span <= p.T);
    if (interior && ((((uintptr_t)(xr + ws)) & 15) == 0) && ((p.span & 3) == 0)) {
      if (tid == 0) tma_span(sp, xr + ws, p.span, &s_bar_tma);
      return true;
    }
    for (int i = tid; i < p.span; i += THREADS) {
      const int u = src_index(ws + i, p.T, p.pad, p.right_pad, p.pad_mode, p.center);
      sp[pad_idx(i)] = (u >= 0) ? __ldg(xr + u) : 0.f;
    }
    return false;
  };
  if (t < total_tiles) by_tma = stage(t);
  unsigned par_tma = 0;

  // ---- DFT-128 matrix F (A operand, fp16 hi / lo parts): row R = (slab R / 16, j = R % 16) is bin cr = 8 slab + j % 8,
  //      64 cos(2 pi a cr / 128) for j < 8, -64 sin(..) for j >= 8; the Im row of cr = 0 is 64 (-1)^a (bin 64)
  for (int i = tid; i < 128 * 64; i += THREADS) {
    const int R = i >> 6, a0 = 2 * (i & 63);
    const int cr = 8 * (R >> 4) + (R & 7), im = (R >> 3) & 1;
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int a = a0 + e;
      float sn, cs;
      sincospif((float)((a * cr) & 127) * (1.0f / 64.0f), &sn, &cs);
      v[e] = 64.0f * (im ? -sn : cs);
      if (cr == 0 && im) v[e] = (a & 1) ? -64.0f : 64.0f;
    }
    uint32_t h, l;
    split2(v[0], v[1], h, l);
    const int off = (R >> 3) * 2048 + (a0 >> 3) * 128 + (R & 7) * 16 + (a0 & 7) * 2;
    *reinterpret_cast<uint32_t*>(fop + off) = h;
    *reinterpret_cast<uint32_t*>(fop + F_PART + off) = l;
  }
  // ---- second-stage twiddles W2048^{b c} at [b][2 c]; [b][1] = W2048^{64 b} (the c = 64 packed pair).  (The odd
  //      entries [b][2 c + 1] hold the conjugates and are not read.)
  for (int i = tid; i < NG * 128; i += THREADS) {
    const int b = i >> 7, r = i & 127;
    const int cc = (r == 1) ? 64 : (r >> 1);
    float sn, cs;
    sincospif((float)(b * cc) * (1.0f / 1024.0f), &sn, &cs);
    tw[i] = make_float2(cs, ((r & 1) && r != 1) ? sn : -sn);
  }
  // ---- banded mel weights (same packing as spectral_warp_kernel: rows grouped by (w = m % 8, step i))
  const bool packed = p.mel_packed_len > 0;
  if (packed) {
    for (int m = tid; m < p.n_mels; m += THREADS) {
      const int lo4 = __ldg(p.mel_lo + m) & ~3;
      int n4 = (((__ldg(p.mel_hi + m) + 3) & ~3) - lo4) >> 2;
      mseg[m] = make_int4(0, lo4, n4 < 0 ? 0 : n4, 0);
    }
    __syncthreads();
    if (tid == 0) {
      int run = 0, reach = 0;
      for (int w = 0; w < 8; ++w)
        for (int i = 0; 4 * (w + 8 * i) < p.n_mels; ++i) {
          int mx = 0;
          for (int j = 0; j < 4; ++j) { const int m = 4 * (w + 8 * i) + j; if (m < p.n_mels) mx = max(mx, mseg[m].z); }
          mx = (mx + 1) & ~1;
          for (int j = 0; j < 4; ++j) {
            const int m = 4 * (w + 8 * i) + j;
            if (m < p.n_mels) { mseg[m].x = run; mseg[m].w = mx; run += mx; reach = max(reach, mseg[m].y + 4 * mx); }
          }
        }
      s_clamp = reach > XBS;
    }
    __syncthreads();
    for (int m = warp; m < p.n_mels; m += NWARP) {
      const int4 sg = mseg[m];
      const float* wrow = p.mel_fb + (size_t)m * F;
      for (int i = lane; i < 4 * sg.w; i += 32) {
        const int k = sg.y + i;
        mpk[4 * sg.x + i] = (i < 4 * sg.z && k < F) ? __ldg(wrow + k) : 0.f;
      }
    }
  }
  fence_async_smem();  // generic-proxy writes of F -> visible to the tensor core (async proxy)
  __syncthreads();

#pragma unroll 1
  for (; t < total_tiles; t += gridDim.x) {
    const int rw = t / p.n_tiles, tile = t - rw * p.n_tiles;
    const int n0 = tile * FR;
    const int ws = (n0 + p.drop_edge) * hop + p.origin;
    const float g = p.gain ? __ldg(p.gain + rw / p.rows_per_gain) : 1.0f;
    if (by_tma) { mbar_wait(&s_bar_tma, par_tma); par_tma ^= 1u; }
    __syncthreads();

    // ---- (1) power-of-two scale of the tile: max |x| S in [512, 1024)
    float mx = 0.f;
    for (int j = tid; j < (p.span >> 2); j += THREADS) {
      const float4 v = *reinterpret_cast<const float4*>(sp + pad_idx(4 * j));
      mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
    }
    for (int i = (p.span & ~3) + tid; i < p.span; i += THREADS) mx = fmaxf(mx, fabsf(sp[pad_idx(i)]));
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < NWARP; ++w) mx = fmaxf(mx, red[w]);
    float S = 1.0f;
    {
      const int E = (int)((__float_as_uint(mx) >> 23) & 0xff);  // mx = m 2^(E-126), m in [0.5, 1)
      if (E >= 27 && E <= 230) S = __uint_as_float((uint32_t)(263 - E) << 23);  // 2^(10 - (E - 126))
    }
    const float inv_scale = 1.0f / (S * 64.0f);
    // ---- (2) window x S
    for (int i = tid * 4; i < NFFT; i += THREADS * 4) {
      float4 w = __ldg(reinterpret_cast<const float4*>(p.window + i));
      w.x *= S; w.y *= S; w.z *= S; w.w *= S;
      *reinterpret_cast<float4*>(wsc + i) = w;
    }
    __syncthreads();

    // ---- (3) + (4): windowed frames -> fp16 (hi, lo) B operand, in two halves of 8 groups (one operand buffer); each
    //      warpgroup multiplies its 64 rows of F with its 8 frames of the half's groups: 3 products x 8 k-steps of
    //      wgmma m64n64k16.  Unit u (64 per half) = (nh, ac, gq'): frames 8 nh + (lane & 7), a in [8 ac, +8),
    //      groups b = 4 (2 half + gq') + e.  Sample of (n, a, b) = span[n hop + 16 a + b].
    const bool blk_aligned = (hop & (BLK - 1)) == 0;  // every frame starts on a padding granule
    float acc[2][32];  // [half][4 i + 2 im + e]: Re (im = 0) / Im (im = 1) of bin c, group 8 half + i, frame f0 + e
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      {
        const int u = 4 * warp + (lane >> 3);
        const int nh = u >> 5, ac = (u >> 1) & 15, gq = 2 * half + (u & 1);
        const int n = 8 * nh + (lane & 7);
        const int o0 = 128 * ac + 4 * gq;
        const int i0 = n * hop + o0;
        // all 8 loads of a unit fall into one 512-sample granule when the frames start on granule boundaries
        const float* sbase = sp + (blk_aligned ? pad_idx(i0) : 0);
        uint32_t hw[4][4], lw[4][4];  // [e = b - 4 gq][pair of a]
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          float4 pr[2];
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            const int j = 2 * jp + e2;
            float4 xv;
            if (blk_aligned) {
              xv = *reinterpret_cast<const float4*>(sbase + 16 * j);
            } else if ((hop & 3) == 0) {
              xv = *reinterpret_cast<const float4*>(sp + pad_idx(i0 + 16 * j));
            } else {
              const int i = i0 + 16 * j;
              xv = make_float4(sp[pad_idx(i)], sp[pad_idx(i + 1)], sp[pad_idx(i + 2)], sp[pad_idx(i + 3)]);
            }
            const float4 wv = *reinterpret_cast<const float4*>(wsc + o0 + 16 * j);
            pr[e2] = make_float4(xv.x * wv.x, xv.y * wv.y, xv.z * wv.z, xv.w * wv.w);
          }
          split2(pr[0].x, pr[1].x, hw[0][jp], lw[0][jp]);
          split2(pr[0].y, pr[1].y, hw[1][jp], lw[1][jp]);
          split2(pr[0].z, pr[1].z, hw[2][jp], lw[2][jp]);
          split2(pr[0].w, pr[1].w, hw[3][jp], lw[3][jp]);
        }
        unsigned char* dst = bop + (4 * (gq - 2 * half)) * 4096 + nh * 2048 + ac * 128 + (lane & 7) * 16;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          *reinterpret_cast<int4*>(dst + e * 4096) = make_int4((int)hw[e][0], (int)hw[e][1], (int)hw[e][2], (int)hw[e][3]);
          *reinterpret_cast<int4*>(dst + B_PART + e * 4096) = make_int4((int)lw[e][0], (int)lw[e][1], (int)lw[e][2], (int)lw[e][3]);
        }
      }
      fence_async_smem();  // generic-proxy writes of the operand -> visible to the tensor core (async proxy)
      __syncthreads();
      fence_acc(acc[half]);
      wgmma_fence();
#pragma unroll
      for (int prod = 0; prod < 3; ++prod) {  // h1 F1, h2 F1, h1 F2
        const unsigned char* ap = fop + (prod == 2 ? F_PART : 0) + rb * 16384;
        const unsigned char* bp = bop + (prod == 1 ? B_PART : 0) + fh * 2048;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) wgmma_64x64x16(acc[half], ap + ks * 256, bp + ks * 256, (prod | ks) != 0);
      }
      wgmma_commit();
      if (half == 0) {  // the operand buffer is refilled with the second half: every warpgroup must be done reading it
        wgmma_wait_all();
        fence_acc(acc[0]);
        __syncthreads();
      }
    }
    // everybody streams the scaled waveform out while the tensor cores work on the second half
    if (p.y_out) {  // y = g x for the samples this tile owns ([n0 hop, (n0 + FR) hop), the last tile up to T)
      const int wt = tid, WT = THREADS;
      const int own_lo = n0 * hop;
      const int own_hi = (tile == p.n_tiles - 1) ? p.T : min(p.T, (n0 + FR) * hop);
      float* yr = p.y_out + (size_t)rw * (size_t)p.T;
      const int lo = max(own_lo, ws), hi = min(own_hi, ws + p.span);
      const bool vec = (((lo - ws) & 3) == 0) && ((((uintptr_t)(yr + lo)) & 15) == 0);
      if (vec) {
        const int n4 = (hi - lo) >> 2;
        for (int i = wt; i < n4; i += WT) {
          float4 v = *reinterpret_cast<const float4*>(sp + pad_idx(lo - ws + 4 * i));
          v.x *= g; v.y *= g; v.z *= g; v.w *= g;
          st_stream4(yr + lo + 4 * i, v);
        }
        for (int w = lo + 4 * n4 + wt; w < hi; w += WT) yr[w] = sp[pad_idx(w - ws)] * g;
      } else {
        for (int w = lo + wt; w < hi; w += WT) yr[w] = sp[pad_idx(w - ws)] * g;
      }
      const float* xr = p.x + (size_t)rw * (size_t)p.T;
      for (int w = max(own_lo, ws + p.span) + wt; w < own_hi; w += WT) yr[w] = __ldg(xr + w) * g;
    }
    __syncthreads();  // the span is dead: the next tile's samples stream in underneath the MMAs and the epilogue
    {
      const int tn = t + gridDim.x;
      by_tma = (tn < total_tiles) ? stage(tn) : false;
    }
    wgmma_wait_all();
    fence_acc(acc[1]);
    __syncthreads();  // the |X| slots below overwrite the operand buffer: every warpgroup's MMAs must be complete

    // ---- (5) second stage in registers: per thread two 16-point DFTs over b.  c != 0: one per frame (z = Re + i Im of
    //      bin c), 16 bins k = +-c + 128 d each.  c = 0: the accumulator's Re rows hold Y[0], its Im rows Y[64], both
    //      real: pass 0 packs Y[0] of frames f0 + i f1, pass 1 packs Y[64] likewise.  All 64 accumulators are moved
    //      into z first so that they are dead before the DFTs.
    {
      const bool c0 = (c == 0);
      float2 z[2][NG];
#pragma unroll
      for (int b = 0; b < NG; ++b) {
        const float* A = &acc[b >> 3][4 * (b & 7)];
        z[0][b] = make_float2(A[0], c0 ? A[1] : A[2]);
        z[1][b] = make_float2(c0 ? A[2] : A[1], A[3]);
      }
#pragma unroll
      for (int pass = 0; pass < 2; ++pass) {
        const int twi = c0 ? pass : 2 * c;
#pragma unroll
        for (int b = 1; b < NG; ++b) z[pass][b] = cmul(z[pass][b], tw[b * 128 + twi]);
        float2 o[NG];
        DFT<NG, 1>::run(z[pass], o);
        if (!c0) {
          float* xf = xs + (f0 + pass) * XBS;
          float* P1 = xf + c;  // d = 1..7  -> c + 128 d
          float* P2 = xf - c;  // d = 9..15 -> -c + 128 (16 - d)
          xf[c] = fast_sqrt(fmaf(o[0].x, o[0].x, o[0].y * o[0].y));
#pragma unroll
          for (int d = 1; d < 8; ++d) P1[128 * d] = fast_sqrt(fmaf(o[d].x, o[d].x, o[d].y * o[d].y));
          xf[1024 - c] = fast_sqrt(fmaf(o[8].x, o[8].x, o[8].y * o[8].y));
#pragma unroll
          for (int d = 9; d < 16; ++d) P2[128 * (16 - d)] = fast_sqrt(fmaf(o[d].x, o[d].x, o[d].y * o[d].y));
        } else {
          // Y = DFT(u + i v) of two real-input problems u = frame f0, v = frame f0 + 1:
          //   pass 0 (c = 0):  U[d] = (Y[d] + conj Y[16-d]) / 2, V[d] = (Y[d] - conj Y[16-d]) / 2i  -> bins 128 d, d = 0..8
          //   pass 1 (c = 64): partner index 15 - d, bins 64 + 128 d, d = 0..7
          float* xu = xs + f0 * XBS;
          float* xv = xs + (f0 + 1) * XBS;
          const int koff = pass ? 64 : 0;
#pragma unroll
          for (int d = 0; d < 9; ++d) {
            const float2 yd = o[d];
            const float2 yn = pass ? o[(15 - d) & 15] : o[(16 - d) & 15];
            const float2 U = make_float2(0.5f * (yd.x + yn.x), 0.5f * (yd.y - yn.y));
            const float2 V = make_float2(0.5f * (yd.y + yn.y), 0.5f * (yn.x - yd.x));
            if (d < 8 || !pass) {
              xu[koff + 128 * d] = sqrtf(fmaf(U.x, U.x, U.y * U.y));
              xv[koff + 128 * d] = sqrtf(fmaf(V.x, V.x, V.y * V.y));
            }
          }
        }
      }
    }
    if (tid < FR) {  // band rows read 4 wide: keep the three floats behind bin 1024 finite (x 0 weight)
      float* xf = xs + tid * XBS;
      xf[1025] = 0.f; xf[1026] = 0.f; xf[1027] = 0.f;
    }
    __syncthreads();

    // ---- (6) banded mel projection + post-op: warps 0-7 take frames 0-7, warps 8-15 frames 8-15
    {
      const int fl = lane & 7, jq = lane >> 3, w8 = warp & 7;
      const int f = 8 * (warp >> 3) + fl;
      const float lscale = p.post_power * 0.30102999566398120f;
      const float ga = fabsf(g) * inv_scale;  // |X| is stored in the tile's scaled units: undo S and the 64 of F here
      const float* xf = xs + f * XBS;
      if (packed) {
        const float4* mpk4 = reinterpret_cast<const float4*>(mpk);
        const int lim = XBS - 4;
        for (int mm = 4 * w8 + jq; mm < p.n_mels; mm += 32) {
          const int4 sg = mseg[mm];
          const float4* w4 = mpk4 + sg.x;
          float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
          if (!s_clamp) {
            const float4* v4 = reinterpret_cast<const float4*>(xf + sg.y);
            for (int it = 0; it < sg.w; it += 2) {
              const float4 wa = w4[it], wb = w4[it + 1], va = v4[it], vb = v4[it + 1];
              a0 = fmaf(wa.x, va.x, a0); a1 = fmaf(wa.y, va.y, a1);
              a2 = fmaf(wb.x, vb.x, a2); a3 = fmaf(wb.y, vb.y, a3);
              a0 = fmaf(wa.z, va.z, a0); a1 = fmaf(wa.w, va.w, a1);
              a2 = fmaf(wb.z, vb.z, a2); a3 = fmaf(wb.w, vb.w, a3);
            }
          } else {
            for (int it = 0; it < sg.w; ++it) {
              const float4 w = w4[it];
              const float4 v = *reinterpret_cast<const float4*>(xf + min(sg.y + 4 * it, lim));
              a0 = fmaf(w.x, v.x, a0); a1 = fmaf(w.y, v.y, a1);
              a0 = fmaf(w.z, v.z, a0); a1 = fmaf(w.w, v.w, a1);
            }
          }
          float acc = ((a0 + a1) + (a2 + a3)) * ga;
          if (p.post == B2A_POST_LOG10) acc = lscale * fast_log2(fmaxf(acc, p.post_eps));
          else if (p.post == B2A_POST_LN) acc = logf(acc + p.post_eps);
          melt[mm * (FR + 1) + f] = acc;
        }
      } else {
        for (int mm = 4 * w8 + jq; mm < p.n_mels; mm += 32) {
          float acc = mel_band(p.mel_fb, p.mel_lo, p.mel_hi, F, mm, xf) * ga;
          if (p.post == B2A_POST_LOG10) acc = lscale * fast_log2(fmaxf(acc, p.post_eps));
          else if (p.post == B2A_POST_LN) acc = logf(acc + p.post_eps);
          melt[mm * (FR + 1) + f] = acc;
        }
      }
    }
    __syncthreads();
    {
      const int nf = min(FR, p.n_frames - n0);
      float* o = p.mel_out + (size_t)rw * p.n_mels * p.n_frames + n0;
      for (int i = tid; i < p.n_mels * FR; i += THREADS) {
        const int m = i / FR, f = i - m * FR;
        if (f < nf) o[(size_t)m * p.n_frames + f] = melt[m * (FR + 1) + f];
      }
    }
    // (the barrier at the top of the next iteration orders these reads of melt / xs before they are rewritten)
  }

}

}  // namespace tc

// Opt-in: the FP32 warp kernel is the default; b2a_spectral_tc_enable(1) selects the tensor-core path.
static int g_tc_enabled = 0;

bool tc_supported(const Params& p) {
  if (!g_tc_enabled) return false;
  if (p.n_fft != tc::NFFT || !p.mel_out || p.stft_out) return false;
  if (p.hop < 1 || p.hop > 512) return false;
  if (!p.center || p.row_origin) return false;
  Params q = p;
  q.span = (tc::FR - 1) * q.hop + q.n_fft;
  tc::Smem s = tc::smem_layout(q);
  if (s.total > 227 * 1024 - 64) {
    q.mel_packed_len = 0;  // band table from global
    s = tc::smem_layout(q);
    if (s.total > 227 * 1024 - 64) return false;
  }
  return true;
}

int launch_tc(Params& p, void* stream) {
  p.span = (tc::FR - 1) * p.hop + p.n_fft;
  p.n_tiles = (p.n_frames + tc::FR - 1) / tc::FR;
  tc::KParams kp;
  kp.s = tc::smem_layout(p);
  if (kp.s.total > 227 * 1024 - 64) {
    p.mel_packed_len = 0;
    kp.s = tc::smem_layout(p);
  }
  B2A_REQUIRE(kp.s.total <= 227 * 1024 - 64, B2A_E_UNSUPPORTED, "spectral_tc: %d bytes of shared memory", kp.s.total);
  p.smem_bytes = kp.s.total;
  kp.p = p;
  const int64_t total = (int64_t)p.rows * p.n_tiles;
  B2A_REQUIRE(total < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spectral_tc: too many tiles");
  B2A_CUDA_OK(cudaFuncSetAttribute(tc::spectral_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kp.s.total));
  const int64_t cap = num_sms();
  const unsigned grid = (unsigned)(total < cap ? total : cap);
  B2A_LAUNCH(tc::spectral_tc_kernel, dim3(grid), dim3(tc::THREADS), (size_t)kp.s.total, stream, kp);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

}  // namespace spectral
}  // namespace b2a

extern "C" int b2a_spectral_uses_tensor_cores(int n_fft, int hop, int want_mel, int want_stft) {
  b2a::spectral::Params p;
  memset(&p, 0, sizeof(p));
  p.n_fft = n_fft; p.hop = hop; p.center = 1; p.n_mels = 128; p.mel_packed_len = 0;
  p.mel_out = want_mel ? reinterpret_cast<float*>(8) : nullptr;
  p.stft_out = want_stft ? reinterpret_cast<float2*>(8) : nullptr;
  return b2a::spectral::tc_supported(p) ? 1 : 0;
}

extern "C" int b2a_spectral_tc_enable(int on) {
  const int prev = b2a::spectral::g_tc_enabled;
  b2a::spectral::g_tc_enabled = on ? 1 : 0;
  return prev;
}
