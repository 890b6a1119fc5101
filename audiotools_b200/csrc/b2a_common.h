// b2a_common.h -- shared helpers of the sm_90a kernels behind include/b2a.h.
//
// The same sources compile two ways:
//   nvcc -gencode arch=compute_90a,code=sm_90a     -> libb2a.so (the product)
//   g++ -x c++ -DB2A_SIM -include tests/cusim/cusim.h -> test-only CPU execution of the
//     identical kernel bodies (tests/cusim); inline PTX is compiled out there.
#pragma once
#ifndef B2A_SIM
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b2a.h"

#define B2A_NUM_SMS 132  // H100 SXM; only a fallback when the device attribute cannot be read

// ---------------------------------------------------------------------------------------
// error plumbing (thread-local message, integer codes; nothing throws)
// ---------------------------------------------------------------------------------------
namespace b2a {
char* err_buf();
int fail(int code, const char* fmt, ...);
}  // namespace b2a

#define B2A_REQUIRE(cond, code, ...) \
  do {                               \
    if (!(cond)) return b2a::fail((code), __VA_ARGS__); \
  } while (0)

#define B2A_CUDA_OK(expr)                                                                   \
  do {                                                                                      \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      return b2a::fail(B2A_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                       __FILE__, __LINE__);                                                 \
  } while (0)

// ---------------------------------------------------------------------------------------
// launch + dynamic shared memory, CUDA vs sim
// B2A_LAUNCH is the only place a kernel is launched; each launch adds one to b2a_kernel_launches (b2a.h) in both
// builds, so the simulator counts exactly what the GPU build launches.
// ---------------------------------------------------------------------------------------
#ifdef B2A_SIM
#define B2A_GRID_CONSTANT
#else
#define B2A_GRID_CONSTANT __grid_constant__
#endif

#define B2A_COUNT_LAUNCH() __atomic_fetch_add(&b2a_kernel_launches, 1, __ATOMIC_RELAXED)

#ifdef B2A_SIM
#define B2A_LAUNCH(kernel, grid, block, smem, stream, ...)                 \
  do {                                                                     \
    B2A_COUNT_LAUNCH();                                                    \
    cusim::launch((grid), (block), (smem), [&] { kernel(__VA_ARGS__); }); \
  } while (0)
#define B2A_DYN_SMEM(name) unsigned char* name = cusim::ctx()->dyn_smem
#define B2A_BAR_SYNC(id, nthreads) cusim::named_bar((id), (nthreads))
#else
#define B2A_LAUNCH(kernel, grid, block, smem, stream, ...)                           \
  do {                                                                               \
    B2A_COUNT_LAUNCH();                                                              \
    kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);        \
  } while (0)
#define B2A_DYN_SMEM(name) extern __shared__ __align__(1024) unsigned char name[]
// named barrier over a sub-set of the CTA's warps (ids 1..15; 0 is __syncthreads)
#define B2A_BAR_SYNC(id, nthreads) asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
#endif

namespace b2a {

// SMs of the current device (cached per device ordinal; B2A_NUM_SMS when the attribute cannot be read)
int num_sms();

// shared-memory offsets are kept 16 B aligned (float4 / TMA access)
inline int align16(int v) { return (v + 15) & ~15; }

// Grid of a persistent 256-thread kernel: the CTAs resident at once with `smem` bytes of dynamic shared memory (at most
// `max_per_sm` per SM when > 0) on every SM, but no more than `work` items, each CTA looping over the rest.
template <class Kernel>
int persistent_grid(Kernel kern, int smem, int64_t work, int64_t* grid, int max_per_sm = 0) {
  int per_sm = 1;
  B2A_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, (size_t)smem));
  if (per_sm < 1) per_sm = 1;
  if (max_per_sm > 0 && per_sm > max_per_sm) per_sm = max_per_sm;
  const int64_t cap = (int64_t)num_sms() * per_sm;
  *grid = work < cap ? work : cap;
  return B2A_OK;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// order-preserving uint32 key of a float (radix selection): a < b as floats <=> ord_key(a) < ord_key(b), NaN aside
__device__ __forceinline__ unsigned ord_key(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_val(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Complex-pair helpers: fma / add / mul on (re, im) pairs, each half rounded exactly like the scalar instruction.
// Hopper has no packed FP32 instruction, so each is two scalar operations (the compiler pairs them freely).
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
// (the _rn intrinsics keep a separate multiply and add from being contracted into an fma)
__device__ __forceinline__ float2 add2(float2 a, float2 b) {
#ifdef B2A_SIM
  return make_float2(a.x + b.x, a.y + b.y);
#else
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#endif
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) {
#ifdef B2A_SIM
  return make_float2(a.x * b.x, a.y * b.y);
#else
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
#endif
}
__device__ __forceinline__ float2 neg2(float2 a) { return make_float2(-a.x, -a.y); }
__device__ __forceinline__ float2 bcast2(float v) { return make_float2(v, v); }

// ---------------------------------------------------------------------------------------
// TMA bulk copy (1-D, global -> shared) completing on an mbarrier: one elected thread arms the barrier with
// the byte count and issues ONE copy for a whole contiguous span (SASS: UBLKCP); the consumers spin on the
// barrier's phase parity.  16-byte aligned source, destination and size.  Under the CPU simulator the issuing
// thread copies synchronously and the wait is a no-op (a __syncthreads always follows it in the kernels).
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
#ifdef B2A_SIM
  *bar = 0;
  (void)count;
#else
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
#ifdef B2A_SIM
  memcpy(smem_dst, gmem_src, bytes);
  (void)bar;
#else
  const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  // order the CTA's earlier generic-proxy accesses of the destination (made visible to this thread by the
  // preceding barrier) before the async-proxy write
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d),
               "l"(gmem_src), "r"(bytes), "r"(b)
               : "memory");
#endif
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
#ifdef B2A_SIM
  (void)bar; (void)parity;
#else
  const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "B2A_MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra B2A_MBAR_DONE;\n"
      "bra B2A_MBAR_WAIT;\n"
      "B2A_MBAR_DONE:\n"
      "}\n" ::"r"(b),
      "r"(parity)
      : "memory");
#endif
}

// streaming (evict-first) 128-bit global accesses for data touched exactly once
__device__ __forceinline__ float4 ld_stream4(const float* p) {
#ifdef B2A_SIM
  return *reinterpret_cast<const float4*>(p);
#else
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
#endif
}
__device__ __forceinline__ void st_stream4(float* p, float4 v) {
#ifdef B2A_SIM
  *reinterpret_cast<float4*>(p) = v;
#else
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
#endif
}

}  // namespace b2a
