// pg_common.cuh — shared device/host helpers for the sm_90a kernels.
//
// Everything here is written against raw PTX (mbarrier, TMA, wgmma); no CUTLASS, no torch.
// Host side: error reporting for the C ABI and CUtensorMap construction through the
// driver entry point (no link-time dependency on libcuda).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pg_b200.h"

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ----------------------------------------------------------------------------------------------
// Host: error plumbing for the C ABI (thread-local message, returned by pg_last_error()).
// ----------------------------------------------------------------------------------------------
void pg_set_error(const char* fmt, ...);
int pg_check_launch(const char* what);  // cudaGetLastError() -> 0 / non-zero + message

#define PG_REQUIRE(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      pg_set_error(__VA_ARGS__);         \
      return 1;                          \
    }                                    \
  } while (0)

// Base-address check of the operands that kernels read or write with 16-byte vector accesses: a misaligned base (a column
// view starting mid-row) is refused with an error instead of faulting on the device.  NULL (an unused operand) passes.
static inline bool pg_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

#define PG_CUDA(call)                                                             \
  do {                                                                            \
    cudaError_t _e = (call);                                                      \
    if (_e != cudaSuccess) {                                                      \
      pg_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

// Builds a 2-D bf16 tensor map: global tensor [rows][cols] with row pitch `ld` elements, box
// [box_rows][box_cols], 128-byte swizzle (box_cols * 2 bytes must be <= 128).
int pg_make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                         uint64_t ld, uint32_t box_rows, uint32_t box_cols);
// Generic N-d bf16 map (dims innermost first), 128B swizzle.
int pg_make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes /* rank-1 entries */, const uint32_t* box,
                         int swizzle128);
int pg_make_tmap_nd(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);
int pg_make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                    uint32_t box_rows, uint32_t box_cols, int swizzle_bytes);
int pg_num_sms();
// Fixed-order reductions.  Kernels whose blocks (or split-K slices) each produce a partial sum write it to a slice of
// the library's device scratch buffer instead of adding it to the output with atomics; pg_sum_partials then adds the
// slices up in slice order, so every run computes bit-identical results.
// pg_scratch: the current device's buffer, at least `bytes` long (grown outside CUDA-graph capture only; a superseded
// buffer is kept, so captured graphs stay valid).  One buffer per device: reductions must be issued on one stream at a
// time (the library's kernels all run on the caller's current stream).
int pg_scratch(size_t bytes, cudaStream_t stream, float** out);
// out[m * ld_out + n] += sum over p = 0 .. nparts-1 of part[p * part_stride + m * N + n]   (m < M, n < N)
int pg_sum_partials(const float* part, int nparts, long long part_stride, int M, int N, int64_t ld_out, float* out,
                    cudaStream_t stream);

// ----------------------------------------------------------------------------------------------
// Device: PTX wrappers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (reported as a CUDA error) instead of a hung GPU.  The timeout path
// makes no function call (no printf): a call anywhere in a kernel serialises its wgmma pipeline.
#ifndef PG_MBAR_TIMEOUT_CYCLES
#define PG_MBAR_TIMEOUT_CYCLES (4000000000ll)
#endif
#ifndef PG_MBAR_SUSPEND_NS
#define PG_MBAR_SUSPEND_NS 20000
#endif
// Up to 256 try_waits in one tight PTX loop (3 instructions per wake-up).  PG_MBAR_SUSPEND_NS > 0 passes a
// suspend-time hint (the warp may be parked that long: cheap for the issue slots, slow to wake -- measured as ~1 k
// cycles per hand-off in the attention kernels); 0 uses try_wait's default (short) suspension; PG_MBAR_SPIN polls
// with test_wait and never suspends.
__device__ __forceinline__ bool mbar_wait_round(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
#if defined(PG_MBAR_SPIN)
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
      "mov.u32 n, 0;\n"
      "PG_WAIT_LOOP:\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "@p bra PG_WAIT_DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 4096;\n\t"
      "@p bra PG_WAIT_LOOP;\n\t"
      "setp.ne.u32 p, n, n;\n"
      "PG_WAIT_DONE:\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#elif PG_MBAR_SUSPEND_NS > 0
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
      "mov.u32 n, 0;\n"
      "PG_WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "@p bra PG_WAIT_DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 256;\n\t"
      "@p bra PG_WAIT_LOOP;\n\t"
      "setp.ne.u32 p, n, n;\n"
      "PG_WAIT_DONE:\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"((uint32_t)PG_MBAR_SUSPEND_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
      "mov.u32 n, 0;\n"
      "PG_WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "@p bra PG_WAIT_DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 1024;\n\t"
      "@p bra PG_WAIT_LOOP;\n\t"
      "setp.ne.u32 p, n, n;\n"
      "PG_WAIT_DONE:\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  while (!mbar_wait_round(bar, parity)) {  // the clock is only read every 256 wake-ups
    if (t0 == 0) {
      t0 = clock64();
    } else if (clock64() - t0 > PG_MBAR_TIMEOUT_CYCLES) {
      __trap();
    }
  }
}

// ---- named barriers (bar.sync waits for `count` threads, bar.arrive signals without waiting) ----
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// ---- per-warpgroup register budget (every warp of the warpgroup executes the same instruction) ----
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// Warp-converged TMA issue (`elect.sync` instead of `if (lane == 0)`: the tensor-map pointer,
// coordinates and barrier address stay in uniform registers instead of being re-broadcast in a loop for every copy).
__device__ __forceinline__ void mbar_arrive_expect_tx_w(uint64_t* bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_w(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_w(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_w(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2,
                                              int c3) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// Single-thread TMA issue (the GEMM epilogue: one thread of a warpgroup moves its staging buffers).
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0) {
  asm volatile("cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3}], [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// global <- shared; the boxes are clipped at the tensor map's dims.  The issuing thread tracks them as bulk groups.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// all of this thread's bulk groups have completed (their global writes included)
__device__ __forceinline__ void bulk_wait_group_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// ---- small math helpers ----
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// The bin (class) of an 8-bit input value under the image likelihoods (losses.categorical_nll,
// losses.logistic_mixture_nll): rint(clamp(x, 0, 1) * (K - 1)), exactly k for x = k / (K - 1) in fp32.
__device__ __forceinline__ int target_class(float x, int K) {
  return (int)rintf(fminf(fmaxf(x, 0.f), 1.f) * (float)(K - 1));
}

// Running max m and sum s of exp(l - m) over the values added, in the order added: a larger l rescales the sum once
// (s e^(m - l) + 1).
struct OnlineLse {
  float m = -INFINITY, s = 0.f;
  __device__ __forceinline__ void add(float l) {
    if (l > m) {
      s = s * expf(m - l) + 1.f;  // the first value: 0 * exp(-inf) + 1
      m = l;
    } else {
      s += expf(l - m);
    }
  }
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  bf162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  bf162 h = *reinterpret_cast<bf162*>(&u);
  return __bfloat1622float2(h);
}

// Activation ids (PG_ACT_*) come from include/pg_b200.h.

__device__ __forceinline__ float pg_tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float pg_exp2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// ELU for bf16 outputs (the GEMM epilogues): one MUFU; the cubic covers the cancellation range of e^x - 1
// (|rel err| < 2e-5 everywhere, far inside bf16's 2^-9)
__device__ __forceinline__ float pg_elu_fast(float x) {
  const float e = pg_exp2_fast(x * 1.4426950408889634f) - 1.f;
  const float p = x * fmaf(x, fmaf(x, 0.16666667f, 0.5f), 1.f);
  return x > 0.f ? x : (x > -0.0625f ? p : e);
}
// atanh(erf(x / sqrt 2)) ~= x (c0 + c1 x^2 + c2 x^4): least-squares fit on [-8, 8]
__device__ __forceinline__ float pg_gelu_q(float x) {
  x = fminf(fmaxf(x, -8.f), 8.f);  // the fit is monotone on [-8, 8]; tanh is saturated there (q(8) = 13.7)
  const float x2 = x * x;
  return x * fmaf(x2, fmaf(x2, -0.0003563930330798993f, 0.037032072878891306f), 0.7974856909542073f);
}

__device__ __forceinline__ float pg_act_fwd(int act, float x) {
  switch (act) {
    case PG_ACT_RELU: return fmaxf(x, 0.f);
    // erf-GELU through Phi(x) = 0.5 (1 + tanh(q(x))), q fitted: with an exact tanh |gelu err| < 2.8e-5; tanh.approx adds
    // its own error (2^-11 relative by the PTX ISA, i.e. up to 2^-12 |x tanh(q)|); on an H100 the total reached 3.2e-5
    // (tests/test_conv_path_kernels_gpu.py)
    case PG_ACT_GELU: {
      const float hx = 0.5f * x;
      return fmaf(hx, pg_tanh_fast(pg_gelu_q(x)), hx);
    }
    case PG_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case PG_ACT_TANH: return tanhf(x);
    default: return x;
  }
}
// GELU and its derivative from one tanh (the forward epilogue that also stores act'(pre), PG_ACT_STORE_DERIV)
__device__ __forceinline__ void pg_gelu_both(float x, float& g, float& d) {
  const float xc = fminf(fmaxf(x, -8.f), 8.f);
  const float x2 = xc * xc;
  const float q = xc * fmaf(x2, fmaf(x2, -0.0003563930330798993f, 0.037032072878891306f), 0.7974856909542073f);
  const float qp = fmaf(x2, fmaf(x2, -0.0017819651653994965f, 0.11109621863667392f), 0.7974856909542073f);
  const float t = pg_tanh_fast(q);
  const float hx = 0.5f * x;
  g = fmaf(hx, t, hx);
  d = fmaf(xc * qp, fmaf(-0.5f * t, t, 0.5f), fmaf(0.5f, t, 0.5f));
}
// derivative w.r.t. the pre-activation x
__device__ __forceinline__ float pg_act_bwd(int act, float x) {
  switch (act) {
    case PG_ACT_RELU: return x > 0.f ? 1.f : 0.f;
    case PG_ACT_GELU: {
      // d/dx [x Phi(x)] with Phi = 0.5 (1 + tanh q(x)):  Phi + x * 0.5 (1 - t^2) q'(x)  — one MUFU (tanh), the
      // Gaussian term comes from the derivative of the same fit (|err| < 1.2e-4 vs erf-GELU's derivative with an exact
      // tanh; tanh.approx's 2^-11 relative error adds up to |0.5 - x q'(x) t| |t| 2^-11).
      const float xc = fminf(fmaxf(x, -8.f), 8.f);
      const float x2 = xc * xc;
      const float q = xc * fmaf(x2, fmaf(x2, -0.0003563930330798993f, 0.037032072878891306f), 0.7974856909542073f);
      const float qp = fmaf(x2, fmaf(x2, -0.0017819651653994965f, 0.11109621863667392f), 0.7974856909542073f);
      const float t = pg_tanh_fast(q);
      return fmaf(xc * qp, fmaf(-0.5f * t, t, 0.5f), fmaf(0.5f, t, 0.5f));
    }
    case PG_ACT_ELU: return x > 0.f ? 1.f : __expf(x);
    case PG_ACT_TANH: {
      float t = tanhf(x);
      return 1.f - t * t;
    }
    case PG_ACT_GIVEN: return x;  // the operand already is the derivative
    case PG_ACT_RELU_OUT: return x > 0.f ? 1.f : 0.f;      // x = relu(pre)
    case PG_ACT_ELU_OUT: return x > 0.f ? 1.f : x + 1.f;   // x = elu(pre): elu'(pre) = e^pre = elu(pre) + 1 for pre <= 0
    default: return 1.f;
  }
}
#include "pg_wgmma.cuh"
#endif  // __CUDACC__
