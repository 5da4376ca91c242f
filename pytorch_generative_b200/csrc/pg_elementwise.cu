// pg_elementwise.cu — the HBM-bound kernels of the path: NCHWLayerNorm, GatedActivation, the recipe's
// BCE-with-logits loss, bias-gradient column sums and the NCHW <-> pixel-major converters used at the
// Module boundary.  All are pure streaming kernels: 16-byte vector accesses, one pass over the data,
// fp32 math, row statistics by warp shuffles.
#include "../../include/pg_b200.h"
#include <stdlib.h>

#include "pg_common.cuh"

namespace {

// ---- 8-element vector load/store helpers (fp32: 2x16B, bf16: 1x16B) ----
template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&v)[8]);
template <>
__device__ __forceinline__ void load8<float>(const float* p, float (&v)[8]) {
  const float4 a = __ldcs(reinterpret_cast<const float4*>(p)), b = __ldcs(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<bf16>(const bf16* p, float (&v)[8]) {
  const uint4 u = __ldcs(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&v)[8]);
template <>
__device__ __forceinline__ void store8<float>(float* p, const float (&v)[8]) {
  __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  __stcs(reinterpret_cast<float4*>(p) + 1, make_float4(v[4], v[5], v[6], v[7]));
}
template <>
__device__ __forceinline__ void store8<bf16>(bf16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                                            pack_bf16x2(v[6], v[7]));
}

// ---- scalar conversions (the element-by-element paths) ----
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ float from_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16(v); }

// ------------------------------------------------------------------------------------------------
// LayerNorm over the channel dim of a pixel-major [P, C] fp32 matrix (reference nn/convolution.py:69-75).
// Fast path: C = 128 * V, one warp per row, the row lives in registers (V float4 per lane).
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, int P,
              float eps, bf16* __restrict__ y_bf16, float* __restrict__ y_f32, float* __restrict__ mean_out,
              float* __restrict__ rstd_out) {
  constexpr int C = 128 * V;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int warp_global = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int num_warps = gridDim.x * warps_per_block;
  float4 g[V], b[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
    b[i] = __ldg(reinterpret_cast<const float4*>(beta) + i * 32 + lane);
  }
  for (int row = warp_global; row < P; row += num_warps) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * C);
    float4 v[V];
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = __ldcs(xr + i * 32 + lane);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + bb * bb) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float4 o;
      o.x = (v[i].x - mean) * rstd * g[i].x + b[i].x;
      o.y = (v[i].y - mean) * rstd * g[i].y + b[i].y;
      o.z = (v[i].z - mean) * rstd * g[i].z + b[i].z;
      o.w = (v[i].w - mean) * rstd * g[i].w + b[i].w;
      if (y_f32) __stcs(reinterpret_cast<float4*>(y_f32 + (size_t)row * C) + i * 32 + lane, o);
      if (y_bf16) {
        uint2 pk = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
        reinterpret_cast<uint2*>(y_bf16 + (size_t)row * C)[i * 32 + lane] = pk;
      }
    }
  }
}

// Generic C: one warp per row, three cached passes.  Rows have pitch ld >= C: the statistics cover the first C
// columns, and columns C..ld of the outputs are written as zeros (the padded channels of a 16-byte operand pitch).
__global__ void ln_fwd_generic_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, int P, int C, int ld, float eps,
                                      bf16* __restrict__ y_bf16, float* __restrict__ y_f32,
                                      float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= P) return;
  const float* xr = x + (size_t)row * ld;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = xr[c] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  for (int c = lane; c < C; c += 32) {
    const float o = (xr[c] - mean) * rstd * gamma[c] + beta[c];
    if (y_f32) y_f32[(size_t)row * ld + c] = o;
    if (y_bf16) y_bf16[(size_t)row * ld + c] = __float2bfloat16(o);
  }
  for (int c = C + lane; c < ld; c += 32) {
    if (y_f32) y_f32[(size_t)row * ld + c] = 0.f;
    if (y_bf16) y_bf16[(size_t)row * ld + c] = __float2bfloat16(0.f);
  }
}

// Backward.  Each warp walks rows with a grid stride and keeps its lanes' dgamma/dbeta partial sums in
// registers; at the end the warps add them into shared memory one after another, and the block writes its [3][C]
// partial to `part` (slice blockIdx.x, summed in block order by pg_sum_partials).
template <int V, bool DY_BF16>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const void* __restrict__ dy_, const float* __restrict__ x, const float* __restrict__ gamma,
              const float* __restrict__ mean_in, const float* __restrict__ rstd_in, int P,
              const float* __restrict__ dres0, const float* __restrict__ dres1, float* __restrict__ dx_f32,
              bf16* __restrict__ dx_bf16, float* __restrict__ part) {
  constexpr int C = 128 * V;
  __shared__ float red[3 * C];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  const int warp_global = blockIdx.x * warps_per_block + wib;
  const int num_warps = gridDim.x * warps_per_block;
  float4 g[V], dg[V], db[V], ds[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    ds[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int row = warp_global; row < P; row += num_warps) {
    const float mean = __ldg(mean_in + row);
    const float rstd = __ldg(rstd_in + row);
    float4 xh[V], gy[V], rsum[V];
    float s1 = 0.f, s2 = 0.f;
    // residual-gradient tiles are fetched up front so that every load of this row is in flight before the
    // (serial) warp reductions below
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const size_t off = (size_t)row * C / 4 + i * 32 + lane;
      rsum[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (dres0) rsum[i] = __ldcs(reinterpret_cast<const float4*>(dres0) + off);
      if (dres1) {
        const float4 r = __ldcs(reinterpret_cast<const float4*>(dres1) + off);
        rsum[i].x += r.x; rsum[i].y += r.y; rsum[i].z += r.z; rsum[i].w += r.w;
      }
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float4 xv = __ldcs(reinterpret_cast<const float4*>(x + (size_t)row * C) + i * 32 + lane);
      float4 d;
      if (DY_BF16) {
        const uint2 u = __ldcs(reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(dy_) + (size_t)row * C) +
                               i * 32 + lane);
        const float2 a = unpack_bf16x2(u.x), b2 = unpack_bf16x2(u.y);
        d = make_float4(a.x, a.y, b2.x, b2.y);
      } else {
        d = __ldcs(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(dy_) + (size_t)row * C) + i * 32 +
                   lane);
      }
      xh[i] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
      gy[i] = make_float4(d.x * g[i].x, d.y * g[i].y, d.z * g[i].z, d.w * g[i].w);
      dg[i].x += d.x * xh[i].x; dg[i].y += d.y * xh[i].y; dg[i].z += d.z * xh[i].z; dg[i].w += d.w * xh[i].w;
      db[i].x += d.x; db[i].y += d.y; db[i].z += d.z; db[i].w += d.w;
      s1 += (gy[i].x + gy[i].y) + (gy[i].z + gy[i].w);
      s2 += (gy[i].x * xh[i].x + gy[i].y * xh[i].y) + (gy[i].z * xh[i].z + gy[i].w * xh[i].w);
    }
    const float m1 = warp_sum(s1) * (1.f / C);
    const float m2 = warp_sum(s2) * (1.f / C);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float4 o;
      o.x = rstd * (gy[i].x - m1 - xh[i].x * m2);
      o.y = rstd * (gy[i].y - m1 - xh[i].y * m2);
      o.z = rstd * (gy[i].z - m1 - xh[i].z * m2);
      o.w = rstd * (gy[i].w - m1 - xh[i].w * m2);
      const size_t off = (size_t)row * C / 4 + i * 32 + lane;
      o.x += rsum[i].x; o.y += rsum[i].y; o.z += rsum[i].z; o.w += rsum[i].w;
      ds[i].x += o.x; ds[i].y += o.y; ds[i].z += o.z; ds[i].w += o.w;
      if (dx_f32) __stcs(reinterpret_cast<float4*>(dx_f32) + off, o);
      if (dx_bf16) reinterpret_cast<uint2*>(dx_bf16)[off] = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
    }
  }
  // Block reduction of the per-lane column partials (dgamma, dbeta, column sums of the emitted gradient = the
  // bias gradient of the layer that produced x), warp 0 first: a fixed summation order.
  if (part) {
    for (int w = 0; w < warps_per_block; ++w) {
      if (wib == w) {
#pragma unroll
        for (int i = 0; i < V; ++i) {
          const int c0 = (i * 32 + lane) * 4;
          const float4 v[3] = {dg[i], db[i], ds[i]};
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            float4* r = reinterpret_cast<float4*>(red + k * C + c0);
            if (w == 0) {
              *r = v[k];
            } else {
              float4 t = *r;
              t.x += v[k].x; t.y += v[k].y; t.z += v[k].z; t.w += v[k].w;
              *r = t;
            }
          }
        }
      }
      __syncthreads();
    }
    for (int c = threadIdx.x; c < 3 * C; c += blockDim.x) part[(size_t)blockIdx.x * 3 * C + c] = red[c];
  }
}

// Any channel count.  One warp per block walks rows with a grid stride; its lanes own disjoint columns of the
// block's shared [3][C] partial sums (dgamma, dbeta, column sums of the emitted gradient), which go to slice
// blockIdx.x of `part` (summed in block order by pg_sum_partials).  Rows have pitch ld >= C; columns C..ld of the
// emitted gradient are written as zeros.
template <bool DY_BF16>
__global__ void __launch_bounds__(32)
ln_bwd_generic_kernel(const void* __restrict__ dy_, const float* __restrict__ x, const float* __restrict__ gamma,
                      const float* __restrict__ mean_in, const float* __restrict__ rstd_in, int P, int C, int ld,
                      const float* __restrict__ dres0, const float* __restrict__ dres1, float* __restrict__ dx_f32,
                      bf16* __restrict__ dx_bf16, float* __restrict__ part) {
  extern __shared__ float ln_acc[];  // [3][C]
  if (blockDim.x != 32) __trap();    // the plain += below relies on one warp per block (lanes own disjoint columns)
  float* acc_g = ln_acc;
  float* acc_b = ln_acc + C;
  float* acc_s = ln_acc + 2 * C;
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) ln_acc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int num_warps = gridDim.x * warps_per_block;
  const bool want_cols = part != nullptr;
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < P; row += num_warps) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    const size_t base = (size_t)row * ld;
    auto ld_dy = [&](int c) -> float {
      return DY_BF16 ? __bfloat162float(reinterpret_cast<const bf16*>(dy_)[base + c])
                     : reinterpret_cast<const float*>(dy_)[base + c];
    };
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (x[base + c] - mean) * rstd;
      const float d = ld_dy(c);
      const float gy = d * gamma[c];
      s1 += gy;
      s2 += gy * xh;
      if (want_cols) {
        acc_g[c] += d * xh;
        acc_b[c] += d;
      }
    }
    const float m1 = warp_sum(s1) / C, m2 = warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) {
      const float xh = (x[base + c] - mean) * rstd;
      float o = rstd * (ld_dy(c) * gamma[c] - m1 - xh * m2);
      if (dres0) o += dres0[base + c];
      if (dres1) o += dres1[base + c];
      if (want_cols) acc_s[c] += o;
      if (dx_f32) dx_f32[base + c] = o;
      if (dx_bf16) dx_bf16[base + c] = __float2bfloat16(o);
    }
    for (int c = C + lane; c < ld; c += 32) {
      if (dx_f32) dx_f32[base + c] = 0.f;
      if (dx_bf16) dx_bf16[base + c] = __float2bfloat16(0.f);
    }
  }
  __syncthreads();
  if (part)
    for (int c = threadIdx.x; c < 3 * C; c += blockDim.x) part[(size_t)blockIdx.x * 3 * C + c] = ln_acc[c];
}

// ------------------------------------------------------------------------------------------------
// GatedActivation (reference nn/convolution.py:62-66).  8 channels per thread.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
// One-MUFU forms for bf16 outputs (tanh.approx: max relative error 2^-11, below the 2^-9 of the bf16 result):
// sigmoid(x) = 0.5 tanh(x / 2) + 0.5.  The fp32-in / fp32-out module path keeps the exact functions (1e-3 parity).
template <bool FAST>
__device__ __forceinline__ float gate_sigmoid(float x) {
  return FAST ? fmaf(0.5f, pg_tanh_fast(0.5f * x), 0.5f) : sigmoidf_(x);
}
template <bool FAST>
__device__ __forceinline__ float gate_act(int act, float x) {
  return (FAST && act == PG_ACT_TANH) ? pg_tanh_fast(x) : pg_act_fwd(act, x);
}

// V channels per thread: 8 (one 16-byte access per operand) when C % 8 == 0, else 1 (element by element: the
// halves of a row then start at any element).
template <int V, typename T>
__device__ __forceinline__ void loadv(const T* p, float (&v)[V]) {
  if constexpr (V == 8) {
    load8<T>(p, v);
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = to_f(p[i]);
  }
}
template <int V, typename T>
__device__ __forceinline__ void storev(T* p, const float (&v)[V]) {
  if constexpr (V == 8) {
    store8<T>(p, v);
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) p[i] = from_f<T>(v[i]);
  }
}

template <int V, typename TX, typename TY>
__global__ void gated_fwd_kernel(const TX* __restrict__ x, int P, int C, int act, TY* __restrict__ y,
                                 const float* __restrict__ res = nullptr) {
  const int cg = C / V;
  const long long total = (long long)P * cg;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / cg;
    const int c = (int)(idx % cg) * V;
    float f[V], g[V], o[V];
    loadv<V, TX>(x + row * 2 * C + c, f);
    loadv<V, TX>(x + row * 2 * C + C + c, g);
    constexpr bool FAST = sizeof(TX) == 2;  // bf16 pre-activations (the fused stacks)
#pragma unroll
    for (int i = 0; i < V; ++i) o[i] = gate_act<FAST>(act, f[i]) * gate_sigmoid<FAST>(g[i]);
    if (res) {  // residual stream fused: y = res + gate(x)
      float rr[V];
      loadv<V, float>(res + row * C + c, rr);
#pragma unroll
      for (int i = 0; i < V; ++i) o[i] += rr[i];
    }
    storev<V, TY>(y + row * C + c, o);
  }
}
template <int V, typename TX, typename TDY, typename TDX>
__global__ void gated_bwd_kernel(const TX* __restrict__ x, const TDY* __restrict__ dy, int P, int C, int act,
                                 TDX* __restrict__ dx) {
  const int cg = C / V;
  const long long total = (long long)P * cg;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / cg;
    const int c = (int)(idx % cg) * V;
    float f[V], g[V], d[V], df[V], dgt[V];
    loadv<V, TX>(x + row * 2 * C + c, f);
    loadv<V, TX>(x + row * 2 * C + C + c, g);
    loadv<V, TDY>(dy + row * C + c, d);
    constexpr bool FAST = sizeof(TX) == 2;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float s = gate_sigmoid<FAST>(g[i]);
      const float a = gate_act<FAST>(act, f[i]);
      const float da = (FAST && act == PG_ACT_TANH) ? fmaf(-a, a, 1.f) : pg_act_bwd(act, f[i]);
      df[i] = d[i] * s * da;
      dgt[i] = d[i] * a * s * (1.f - s);
    }
    storev<V, TDX>(dx + row * 2 * C + c, df);
    storev<V, TDX>(dx + row * 2 * C + C + c, dgt);
  }
}

// ------------------------------------------------------------------------------------------------
// BCE with logits, summed (reference image_gpt.py:158-162).  loss = max(l,0) - l*t + log1p(exp(-|l|)).
// ------------------------------------------------------------------------------------------------
// Each block writes its partial loss to part[blockIdx.x] (summed in block order by pg_sum_partials).
__global__ void bce_kernel(const float* __restrict__ logits, const float* __restrict__ target, long long numel,
                           float grad_scale, float* __restrict__ part, float* __restrict__ dlogits) {
  __shared__ float red[32];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel;
       i += (long long)gridDim.x * blockDim.x) {
    const float l = logits[i], t = target[i];
    acc += fmaxf(l, 0.f) - l * t + log1pf(expf(-fabsf(l)));
    if (dlogits) dlogits[i] = (1.f / (1.f + expf(-l)) - t) * grad_scale;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0 && part) part[blockIdx.x] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Column sums (bias gradients).  Fast path: each thread owns 8 consecutive columns (16-byte loads for bf16,
// 2x16 for fp32), a warp covers 256 columns of one row per step, 8 warps stride over the rows of the block's
// strip; partial sums meet in shared memory, and the block writes row blockIdx.y of `part` ([row strips][C], summed
// in strip order by pg_sum_partials).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const T* __restrict__ x, int64_t ld, int P, int C, int rows_per_block, float* __restrict__ out) {
  __shared__ float red[8][256 + 8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, P);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (col < C) {  // C % 8 == 0 on this path
    for (int r = r0 + w; r < r1; r += 8) {
      float v[8];
      load8<T>(x + (size_t)r * ld + col, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[w][lane * 8 + i] = acc[i];
  __syncthreads();
  const int c = threadIdx.x;  // 256 threads <-> 256 columns of the block
  if (blockIdx.x * 256 + c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][c];
    out[(size_t)blockIdx.y * C + blockIdx.x * 256 + c] = t;
  }
}

// Generic fallback: block = 32x8 threads over a strip of rows, coalesced along columns.
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ x, int64_t ld, int P, int C, int rows_per_block,
                              float* __restrict__ out) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, P);
  float acc = 0.f;
  if (col < C) {
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      if constexpr (sizeof(T) == 2) acc += __bfloat162float(reinterpret_cast<const bf16*>(x)[(size_t)r * ld + col]);
      else acc += reinterpret_cast<const float*>(x)[(size_t)r * ld + col];
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    out[(size_t)blockIdx.y * C + col] = t;
  }
}

// ------------------------------------------------------------------------------------------------
// NCHW fp32 <-> pixel-major converters (per image: [C, HW] <-> [HW, C] transposes through smem).
// ------------------------------------------------------------------------------------------------
template <typename TO>
__global__ void nchw_to_pm_kernel(const float* __restrict__ x, int C, int HW, TO* __restrict__ out, int64_t ld_out) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((size_t)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < C) {
      const float v = tile[threadIdx.x][i];
      if constexpr (sizeof(TO) == 2) out[((size_t)n * HW + p) * ld_out + c] = __float2bfloat16(v);
      else out[((size_t)n * HW + p) * ld_out + c] = v;
    }
  }
}
template <typename TI>
__global__ void pm_to_nchw_kernel(const TI* __restrict__ x, int64_t ld_x, int C, int HW, int act, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (p < HW && c < C) {
      if constexpr (sizeof(TI) == 2) v = __bfloat162float(x[((size_t)n * HW + p) * ld_x + c]);
      else v = x[((size_t)n * HW + p) * ld_x + c];
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) out[((size_t)n * C + c) * HW + p] = pg_act_fwd(act, tile[threadIdx.x][i]);
  }
}

// g[p, c] = dy[p, c] * act'(pre[p, c]) -> bf16 (gradient through an activation applied to a conv output)
__global__ void dact_mul_kernel(const bf16* __restrict__ dy, int64_t ld_dy, const float* __restrict__ pre, int64_t ld_pre,
                                int P, int C, int act, bf16* __restrict__ out, int64_t ld_out) {
  const long long total = (long long)P * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / C;
    const int c = (int)(idx % C);
    out[r * ld_out + c] = __float2bfloat16(__bfloat162float(dy[r * ld_dy + c]) * pg_act_bwd(act, pre[r * ld_pre + c]));
  }
}

__global__ void cast_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long numel) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel;
       i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(x[i]);
}

// out = bf16(act(x)) over a pitched [P, C] matrix, V = 8 elements (one 16-byte store) per thread, or V = 1 when C or
// a pitch does not allow 16-byte accesses.
template <int V, typename TI>
__global__ void __launch_bounds__(256)
act_cast_kernel(const TI* __restrict__ x, int64_t ld_x, int P, int C, int act, bf16* __restrict__ out, int64_t ld_out) {
  const int cvn = C / V;
  const long long total = (long long)P * cvn;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / cvn;
    const int c = (int)(idx % cvn) * V;
    if constexpr (V == 1) {
      const float v = to_f(x[row * ld_x + c]);
      out[row * ld_out + c] = __float2bfloat16(act != PG_ACT_NONE ? pg_act_fwd(act, v) : v);
      continue;
    } else {
      float v[8];
      if constexpr (sizeof(TI) == 4) {
        const float4 a = *reinterpret_cast<const float4*>(x + row * ld_x + c);
        const float4 b = *reinterpret_cast<const float4*>(x + row * ld_x + c + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
        const uint4 a = *reinterpret_cast<const uint4*>(x + row * ld_x + c);
        const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(w[i]);
          v[2 * i] = f.x;
          v[2 * i + 1] = f.y;
        }
      }
      if (act != PG_ACT_NONE) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = pg_act_fwd(act, v[i]);
      }
      *reinterpret_cast<uint4*>(out + row * ld_out + c) =
          make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
    }
  }
}

// out = bf16(dy * act'(pre)) where `ya` holds the ACTIVATED value act(pre) (relu / elu): one pass.
template <typename TDY>
__global__ void __launch_bounds__(256)
dact_out_kernel(const TDY* __restrict__ dy, const bf16* __restrict__ ya, long long numel8, int dact, bf16* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel8; i += (long long)gridDim.x * blockDim.x) {
    float d[8], a[8], o[8];
    load8<TDY>(dy + i * 8, d);
    load8<bf16>(ya + i * 8, a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = d[j] * pg_act_bwd(dact, a[j]);
    store8<bf16>(out + i * 8, o);
  }
}

int grid_for(long long work_items, int threads, int max_blocks_per_sm = 16) {
  long long b = (work_items + threads - 1) / threads;
  long long cap = (long long)pg_num_sms() * max_blocks_per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

extern "C" int pg_layernorm_fwd_ld(const float* x, const float* gamma, const float* beta, int P, int C, int ld,
                                   float eps, void* y_bf16, float* y_f32, float* mean, float* rstd, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && gamma && beta && (y_bf16 || y_f32), "pg_layernorm_fwd: null argument");
  PG_REQUIRE(P > 0 && C > 0, "pg_layernorm_fwd: empty problem");
  PG_REQUIRE(ld >= C, "pg_layernorm_fwd: pitch %d is narrower than C=%d", ld, C);
  const int threads = 256, wpb = threads / 32;
  const bool fast = ld == C && (C % 128 == 0) && C <= 1024;
  PG_REQUIRE(!fast || (pg_aligned16(x) && pg_aligned16(gamma) && pg_aligned16(beta) && pg_aligned16(y_bf16) &&
                       pg_aligned16(y_f32)),
             "pg_layernorm_fwd: x, gamma, beta, y_bf16 and y_f32 must be 16-byte aligned (C=%d takes the vector path)", C);
  if (fast) {
    const int blocks = grid_for((long long)P * 32, threads, 8);
    bf16* yb = reinterpret_cast<bf16*>(y_bf16);
    switch (C / 128) {
#define LN_CASE(V) \
  case V: ln_fwd_kernel<V><<<blocks, threads, 0, stream>>>(x, gamma, beta, P, eps, yb, y_f32, mean, rstd); break;
      LN_CASE(1) LN_CASE(2) LN_CASE(3) LN_CASE(4) LN_CASE(5) LN_CASE(6) LN_CASE(7) LN_CASE(8)
#undef LN_CASE
    }
  } else {
    ln_fwd_generic_kernel<<<(P + wpb - 1) / wpb, threads, 0, stream>>>(x, gamma, beta, P, C, ld, eps,
                                                                         reinterpret_cast<bf16*>(y_bf16), y_f32, mean, rstd);
  }
  return pg_check_launch("pg_layernorm_fwd");
}

extern "C" int pg_layernorm_fwd(const float* x, const float* gamma, const float* beta, int P, int C, float eps,
                                void* y_bf16, float* y_f32, float* mean, float* rstd, void* stream) {
  return pg_layernorm_fwd_ld(x, gamma, beta, P, C, C, eps, y_bf16, y_f32, mean, rstd, stream);
}

extern "C" int pg_layernorm_bwd_ld(const void* dy_bf16, const float* dy_f32, const float* x, const float* gamma,
                                   const float* mean, const float* rstd, int P, int C, int ld, const float* dres0,
                                   const float* dres1, float* dx_f32, void* dx_bf16, float* dgamma, float* dbeta,
                                   float* dx_colsum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE((dy_bf16 != nullptr) != (dy_f32 != nullptr), "pg_layernorm_bwd: exactly one of dy_bf16 / dy_f32");
  PG_REQUIRE(x && gamma && mean && rstd && (dx_f32 || dx_bf16), "pg_layernorm_bwd: null argument");
  PG_REQUIRE(ld >= C, "pg_layernorm_bwd: pitch %d is narrower than C=%d", ld, C);
  const int threads = 256, wpb = threads / 32;
  const bool fast = ld == C && (C % 128 == 0) && C <= 1024;
  PG_REQUIRE(!fast || (pg_aligned16(dy_bf16) && pg_aligned16(dy_f32) && pg_aligned16(x) && pg_aligned16(gamma) &&
                       pg_aligned16(dres0) && pg_aligned16(dres1) && pg_aligned16(dx_f32) && pg_aligned16(dx_bf16)),
             "pg_layernorm_bwd: dy, x, gamma, dres0, dres1, dx_f32 and dx_bf16 must be 16-byte aligned (C=%d takes the "
             "vector path)", C);
  bf16* dxb = reinterpret_cast<bf16*>(dx_bf16);
  const bool want_part = dgamma || dbeta || dx_colsum;
  // block partials [blocks][3][C] in the scratch buffer, summed in block order below
  const int blocks = fast ? grid_for((long long)P * 32, threads, 2)  // 128 registers: two resident blocks per SM
                          : grid_for((long long)P * 32, 32, 8);      // one warp per block (see ln_bwd_generic_kernel)
  float* part = nullptr;
  if (want_part && pg_scratch((size_t)blocks * 3 * C * sizeof(float), stream, &part)) return 1;
  if (fast) {
    switch (C / 128) {
#define LNB_CASE(V)                                                                                              \
  case V:                                                                                                        \
    if (dy_bf16)                                                                                                 \
      ln_bwd_kernel<V, true><<<blocks, threads, 0, stream>>>(dy_bf16, x, gamma, mean, rstd, P, dres0, dres1, dx_f32, \
                                                             dxb, part);                                         \
    else                                                                                                         \
      ln_bwd_kernel<V, false><<<blocks, threads, 0, stream>>>(dy_f32, x, gamma, mean, rstd, P, dres0, dres1, dx_f32, \
                                                              dxb, part);                                        \
    break;
      LNB_CASE(1) LNB_CASE(2) LNB_CASE(3) LNB_CASE(4) LNB_CASE(5) LNB_CASE(6) LNB_CASE(7) LNB_CASE(8)
#undef LNB_CASE
    }
  } else {
    PG_REQUIRE(C <= 4096, "pg_layernorm_bwd: more than 4096 channels");
    const size_t smem = 3 * (size_t)C * sizeof(float);
    if (dy_bf16)
      ln_bwd_generic_kernel<true><<<blocks, 32, smem, stream>>>(dy_bf16, x, gamma, mean, rstd, P, C, ld, dres0, dres1,
                                                              dx_f32, dxb, part);
    else
      ln_bwd_generic_kernel<false><<<blocks, 32, smem, stream>>>(dy_f32, x, gamma, mean, rstd, P, C, ld, dres0, dres1,
                                                               dx_f32, dxb, part);
  }
  if (pg_check_launch("pg_layernorm_bwd")) return 1;
  float* outs[3] = {dgamma, dbeta, dx_colsum};
  for (int k = 0; k < 3; ++k)
    if (outs[k] && pg_sum_partials(part + (size_t)k * C, blocks, 3LL * C, 1, C, C, outs[k], stream)) return 1;
  return 0;
}

extern "C" int pg_layernorm_bwd(const void* dy_bf16, const float* dy_f32, const float* x, const float* gamma,
                                const float* mean, const float* rstd, int P, int C, const float* dres0,
                                const float* dres1, float* dx_f32, void* dx_bf16, float* dgamma, float* dbeta,
                                float* dx_colsum, void* stream) {
  return pg_layernorm_bwd_ld(dy_bf16, dy_f32, x, gamma, mean, rstd, P, C, C, dres0, dres1, dx_f32, dx_bf16, dgamma, dbeta,
                             dx_colsum, stream);
}

template <int V>
static int gated_fwd_launch(const void* x, int x_is_f32, int P, int C, int act, void* y, int y_is_f32, int blocks,
                            int threads, cudaStream_t stream) {
  if (x_is_f32 && y_is_f32)
    gated_fwd_kernel<V, float, float><<<blocks, threads, 0, stream>>>((const float*)x, P, C, act, (float*)y);
  else if (x_is_f32 && !y_is_f32)
    gated_fwd_kernel<V, float, bf16><<<blocks, threads, 0, stream>>>((const float*)x, P, C, act, (bf16*)y);
  else if (!x_is_f32 && y_is_f32)
    gated_fwd_kernel<V, bf16, float><<<blocks, threads, 0, stream>>>((const bf16*)x, P, C, act, (float*)y);
  else
    gated_fwd_kernel<V, bf16, bf16><<<blocks, threads, 0, stream>>>((const bf16*)x, P, C, act, (bf16*)y);
  return pg_check_launch("pg_gated_act_fwd");
}

template <int V>
static int gated_bwd_launch(const void* x, int x_is_f32, const void* dy, int dy_is_f32, int P, int C, int act, void* dx,
                            int blocks, int threads, cudaStream_t stream) {
  if (!x_is_f32 && dy_is_f32)  // bf16 pre-activation, fp32 gradient of a residual stream
    gated_bwd_kernel<V, bf16, float, bf16><<<blocks, threads, 0, stream>>>((const bf16*)x, (const float*)dy, P, C, act,
                                                                          (bf16*)dx);
  else if (x_is_f32)
    gated_bwd_kernel<V, float, float, float><<<blocks, threads, 0, stream>>>((const float*)x, (const float*)dy, P, C, act,
                                                                             (float*)dx);
  else
    gated_bwd_kernel<V, bf16, bf16, bf16><<<blocks, threads, 0, stream>>>((const bf16*)x, (const bf16*)dy, P, C, act,
                                                                          (bf16*)dx);
  return pg_check_launch("pg_gated_act_bwd");
}

extern "C" int pg_gated_act_fwd(const void* x, int x_is_f32, int P, int C, int act, void* y, int y_is_f32,
                                void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && y && P > 0 && C > 0, "pg_gated_act_fwd: null/empty argument");
  const bool vec = C % 8 == 0;  // else the element-by-element path
  PG_REQUIRE(!vec || (pg_aligned16(x) && pg_aligned16(y)), "pg_gated_act_fwd: x and y must be 16-byte aligned");
  const int threads = 256;
  const int blocks = grid_for((long long)P * (vec ? C / 8 : C), threads);
  if (vec) return gated_fwd_launch<8>(x, x_is_f32, P, C, act, y, y_is_f32, blocks, threads, stream);
  return gated_fwd_launch<1>(x, x_is_f32, P, C, act, y, y_is_f32, blocks, threads, stream);
}

extern "C" int pg_gated_res_fwd(const void* x, int x_is_f32, const float* res, int P, int C, int act, float* y, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && res && y && P > 0 && C > 0, "pg_gated_res_fwd: null/empty argument");
  const bool vec = C % 8 == 0;  // else the element-by-element path
  PG_REQUIRE(!vec || (pg_aligned16(x) && pg_aligned16(res) && pg_aligned16(y)),
             "pg_gated_res_fwd: x, res and y must be 16-byte aligned");
  const int threads = 256;
  const int blocks = grid_for((long long)P * (vec ? C / 8 : C), threads);
  if (vec) {
    if (x_is_f32) gated_fwd_kernel<8, float, float><<<blocks, threads, 0, stream>>>((const float*)x, P, C, act, y, res);
    else gated_fwd_kernel<8, bf16, float><<<blocks, threads, 0, stream>>>((const bf16*)x, P, C, act, y, res);
  } else {
    if (x_is_f32) gated_fwd_kernel<1, float, float><<<blocks, threads, 0, stream>>>((const float*)x, P, C, act, y, res);
    else gated_fwd_kernel<1, bf16, float><<<blocks, threads, 0, stream>>>((const bf16*)x, P, C, act, y, res);
  }
  return pg_check_launch("pg_gated_res_fwd");
}

extern "C" int pg_dact_from_out(const void* dy, int dy_is_f32, const void* ya_bf16, int64_t numel, int act, void* out_bf16,
                                void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(dy && ya_bf16 && out_bf16 && numel > 0 && numel % 8 == 0, "pg_dact_from_out: null argument or numel %% 8 != 0");
  PG_REQUIRE(act == PG_ACT_RELU || act == PG_ACT_ELU, "pg_dact_from_out: relu / elu only");
  PG_REQUIRE(pg_aligned16(dy) && pg_aligned16(ya_bf16) && pg_aligned16(out_bf16),
             "pg_dact_from_out: dy, ya and out must be 16-byte aligned");
  const int dact = act == PG_ACT_RELU ? PG_ACT_RELU_OUT : PG_ACT_ELU_OUT;
  const int blocks = grid_for(numel / 8, 256);
  if (dy_is_f32) dact_out_kernel<float><<<blocks, 256, 0, stream>>>((const float*)dy, (const bf16*)ya_bf16, numel / 8, dact, (bf16*)out_bf16);
  else dact_out_kernel<bf16><<<blocks, 256, 0, stream>>>((const bf16*)dy, (const bf16*)ya_bf16, numel / 8, dact, (bf16*)out_bf16);
  return pg_check_launch("pg_dact_from_out");
}

extern "C" int pg_gated_act_bwd(const void* x, int x_is_f32, const void* dy, int dy_is_f32, int P, int C, int act,
                                void* dx, int dx_is_f32, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && dy && dx && P > 0 && C > 0, "pg_gated_act_bwd: null/empty argument");
  PG_REQUIRE(x_is_f32 == dx_is_f32 && (x_is_f32 == dy_is_f32 || (!x_is_f32 && dy_is_f32)),
             "pg_gated_act_bwd: dx has x's dtype; dy has x's dtype or is fp32 over a bf16 x");
  const bool vec = C % 8 == 0;  // else the element-by-element path
  PG_REQUIRE(!vec || (pg_aligned16(x) && pg_aligned16(dy) && pg_aligned16(dx)),
             "pg_gated_act_bwd: x, dy and dx must be 16-byte aligned");
  const int threads = 256;
  const int blocks = grid_for((long long)P * (vec ? C / 8 : C), threads);
  if (vec) return gated_bwd_launch<8>(x, x_is_f32, dy, dy_is_f32, P, C, act, dx, blocks, threads, stream);
  return gated_bwd_launch<1>(x, x_is_f32, dy, dy_is_f32, P, C, act, dx, blocks, threads, stream);
}

extern "C" int pg_bce_logits_fwd_bwd(const float* logits, const float* target, int64_t numel, float grad_scale,
                                     float* loss_sum, float* dlogits, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(logits && target && numel > 0, "pg_bce_logits_fwd_bwd: null/empty argument");
  const int threads = 256;
  const int blocks = grid_for(numel, threads, 4);
  float* part = nullptr;
  if (loss_sum && pg_scratch((size_t)blocks * sizeof(float), stream, &part)) return 1;
  bce_kernel<<<blocks, threads, 0, stream>>>(logits, target, numel, grad_scale, part, dlogits);
  if (pg_check_launch("pg_bce_logits_fwd_bwd")) return 1;
  return loss_sum ? pg_sum_partials(part, blocks, 1, 1, 1, 1, loss_sum, stream) : 0;
}

// Column sums through per-strip partials ([strips][C] in the scratch buffer), added to `out` in strip order.
template <typename T>
static int colsum_impl(const T* x, int64_t ld, int P, int C, float* out, int accumulate, cudaStream_t stream,
                       bool vec, const char* who) {
  if (!accumulate) PG_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * C, stream));
  const int rows_per_block = vec ? 256 : 512;
  const int strips = (P + rows_per_block - 1) / rows_per_block;
  float* part = nullptr;
  if (pg_scratch((size_t)strips * C * sizeof(float), stream, &part)) return 1;
  if (vec) {
    dim3 grid((C + 255) / 256, strips);
    colsum_vec_kernel<T><<<grid, 256, 0, stream>>>(x, ld, P, C, rows_per_block, part);
  } else {
    dim3 grid((C + 31) / 32, strips), block(32, 8);
    colsum_kernel<T><<<grid, block, 0, stream>>>(x, ld, P, C, rows_per_block, part);
  }
  if (pg_check_launch(who)) return 1;
  return pg_sum_partials(part, strips, C, 1, C, C, out, stream);
}

extern "C" int pg_colsum_bf16(const void* x, int64_t ld, int P, int C, float* out, int accumulate, void* stream_) {
  PG_REQUIRE(x && out && P > 0 && C > 0, "pg_colsum_bf16: null/empty argument");
  const bool vec = C % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  return colsum_impl<bf16>((const bf16*)x, ld, P, C, out, accumulate, reinterpret_cast<cudaStream_t>(stream_), vec,
                           "pg_colsum_bf16");
}
extern "C" int pg_colsum_f32(const float* x, int64_t ld, int P, int C, float* out, int accumulate, void* stream_) {
  PG_REQUIRE(x && out && P > 0 && C > 0, "pg_colsum_f32: null/empty argument");
  const bool vec = C % 8 == 0 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  return colsum_impl<float>(x, ld, P, C, out, accumulate, reinterpret_cast<cudaStream_t>(stream_), vec, "pg_colsum_f32");
}

extern "C" int pg_nchw_to_pm(const float* x_nchw, int N, int C, int HW, void* out, int out_is_f32, int64_t ld_out,
                             void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x_nchw && out && N > 0 && C > 0 && HW > 0, "pg_nchw_to_pm: null/empty argument");
  dim3 grid((HW + 31) / 32, (C + 31) / 32, N), block(32, 8);
  if (out_is_f32) nchw_to_pm_kernel<float><<<grid, block, 0, stream>>>(x_nchw, C, HW, (float*)out, ld_out);
  else nchw_to_pm_kernel<bf16><<<grid, block, 0, stream>>>(x_nchw, C, HW, (bf16*)out, ld_out);
  return pg_check_launch("pg_nchw_to_pm");
}
extern "C" int pg_pm_to_nchw(const void* x_pm, int x_is_f32, int64_t ld_x, int N, int C, int HW, int act,
                             float* out_nchw, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x_pm && out_nchw && N > 0 && C > 0 && HW > 0, "pg_pm_to_nchw: null/empty argument");
  dim3 grid((HW + 31) / 32, (C + 31) / 32, N), block(32, 8);
  if (x_is_f32) pm_to_nchw_kernel<float><<<grid, block, 0, stream>>>((const float*)x_pm, ld_x, C, HW, act, out_nchw);
  else pm_to_nchw_kernel<bf16><<<grid, block, 0, stream>>>((const bf16*)x_pm, ld_x, C, HW, act, out_nchw);
  return pg_check_launch("pg_pm_to_nchw");
}
extern "C" int pg_cast_f32_to_bf16(const float* x, void* y, int64_t numel, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && y && numel > 0, "pg_cast_f32_to_bf16: null/empty argument");
  cast_kernel<<<grid_for(numel, 256), 256, 0, stream>>>(x, (bf16*)y, numel);
  return pg_check_launch("pg_cast_f32_to_bf16");
}

extern "C" int pg_dact_mul(const void* dy_bf16, int64_t ld_dy, const float* pre_f32, int64_t ld_pre, int P, int C, int act,
                           void* out_bf16, int64_t ld_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(dy_bf16 && pre_f32 && out_bf16 && P > 0 && C > 0, "pg_dact_mul: null/empty argument");
  dact_mul_kernel<<<grid_for((long long)P * C, 256), 256, 0, stream>>>((const bf16*)dy_bf16, ld_dy, pre_f32, ld_pre, P, C, act,
                                                                      (bf16*)out_bf16, ld_out);
  return pg_check_launch("pg_dact_mul");
}

extern "C" int pg_act_cast_bf16(const void* x, int x_is_f32, int64_t ld_x, int P, int C, int act, void* out_bf16,
                                int64_t ld_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x && out_bf16 && P > 0 && C > 0, "pg_act_cast_bf16: null/empty argument");
  // the 16-byte path needs C and both pitches in whole 16-byte vectors; anything else goes element by element
  const bool vec = C % 8 == 0 && ld_x % (x_is_f32 ? 4 : 8) == 0 && ld_out % 8 == 0;
  PG_REQUIRE(!vec || (pg_aligned16(x) && pg_aligned16(out_bf16)), "pg_act_cast_bf16: x and out must be 16-byte aligned");
  const int grid = grid_for((long long)P * (vec ? C / 8 : C), 256);
  bf16* out = (bf16*)out_bf16;
  if (vec) {
    if (x_is_f32) act_cast_kernel<8, float><<<grid, 256, 0, stream>>>((const float*)x, ld_x, P, C, act, out, ld_out);
    else act_cast_kernel<8, bf16><<<grid, 256, 0, stream>>>((const bf16*)x, ld_x, P, C, act, out, ld_out);
  } else {
    if (x_is_f32) act_cast_kernel<1, float><<<grid, 256, 0, stream>>>((const float*)x, ld_x, P, C, act, out, ld_out);
    else act_cast_kernel<1, bf16><<<grid, 256, 0, stream>>>((const bf16*)x, ld_x, P, C, act, out, ld_out);
  }
  return pg_check_launch("pg_act_cast_bf16");
}
