// pg_optim.cu — the optimizer part of the training step (reference trainer.py:182-191: clip_grad_norm_ over all
// parameters, then torch.optim.Adam.step) as two multi-tensor kernels over every parameter of the model:
//   1. pg_grad_sqnorm   per-block partial sums of g^2 (fixed chunking -> the reduction order is deterministic)
//   2. pg_adam_step     every block re-reduces the partials (a few KB) to the global gradient norm, derives the clip
//                       coefficient min(1, max_norm / (norm + 1e-6)) exactly as torch.nn.utils.clip_grad_norm_ does, and
//                       applies torch's Adam update (no amsgrad, no weight decay) to its chunk:
//                           m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
//                           p -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps)
// One pass over g for the norm, one pass over (g, p, m, v) for the update: 2.4 GB of HBM traffic at the ImageGPT C5
// parameter count (75.7 M) instead of the ~6 GB of the foreach norm / mul / lerp / addcmul / sqrt / addcdiv chain.
// Tensors are described by device arrays of pointers; a chunk table maps every block to (tensor, offset).
#include "../../include/pg_b200.h"
#include "pg_common.cuh"

namespace {

constexpr int OPT_THREADS = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = 0.f;
  if (w == 0) {
    t = lane < OPT_THREADS / 32 ? red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  t = red[0];
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(OPT_THREADS)
grad_sqnorm_kernel(const float* const* __restrict__ grads, const int64_t* __restrict__ numel,
                   const int2* __restrict__ chunks, int chunk_elems, float* __restrict__ partials) {
  __shared__ float red[OPT_THREADS / 32];
  const int2 ck = chunks[blockIdx.x];  // (tensor, chunk index inside it)
  const float* g = grads[ck.x];
  const int64_t n = numel[ck.x];
  const int64_t lo = (int64_t)ck.y * chunk_elems;
  const int64_t hi = min(lo + (int64_t)chunk_elems, n);
  float s = 0.f;
  if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
    const int64_t lo4 = lo / 4, hi4 = hi / 4;  // lo is a multiple of chunk_elems (itself a multiple of 4)
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t i = lo4 + threadIdx.x; i < hi4; i += OPT_THREADS) {
      const float4 x = g4[i];
      s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    }
    for (int64_t i = hi4 * 4 + threadIdx.x; i < hi; i += OPT_THREADS) s += g[i] * g[i];
  } else {
    for (int64_t i = lo + threadIdx.x; i < hi; i += OPT_THREADS) s += g[i] * g[i];
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// fp32 -> bf16 copies of many tensors in one launch (the per-step refresh of the tensor-core weight operands)
__global__ void __launch_bounds__(OPT_THREADS)
cast_multi_kernel(const float* const* __restrict__ src, bf16* const* __restrict__ dst, const int64_t* __restrict__ numel,
                  const int2* __restrict__ chunks, int chunk_elems) {
  const int2 ck = chunks[blockIdx.x];
  const float* x = src[ck.x];
  bf16* y = dst[ck.x];
  const int64_t n = numel[ck.x];
  const int64_t lo = (int64_t)ck.y * chunk_elems;
  const int64_t hi = min(lo + (int64_t)chunk_elems, n);
  int64_t tail = lo;
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
    const int64_t lo8 = lo / 8, hi8 = hi / 8;
    for (int64_t i = lo8 + threadIdx.x; i < hi8; i += OPT_THREADS) {
      const float4 a = reinterpret_cast<const float4*>(x)[2 * i], b = reinterpret_cast<const float4*>(x)[2 * i + 1];
      reinterpret_cast<uint4*>(y)[i] =
          make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
    }
    tail = hi8 * 8;
  }
  for (int64_t i = tail + threadIdx.x; i < hi; i += OPT_THREADS) y[i] = __float2bfloat16(x[i]);
}

struct AdamArgs {
  float* const* params;
  float* const* grads;
  float* const* exp_avg;
  float* const* exp_avg_sq;
  const int64_t* numel;
  const int2* chunks;
  const float* partials;
  int n_chunks, chunk_elems;
  float max_norm, skip_above;  // skip_above <= 0: never skip
  float lr_over_bc1, rsqrt_bc2, beta1, beta2, omb1, omb2, eps;  // omb = 1 - beta, rounded from double like torch's scalars
  float* norm_out;  // [2]: total gradient norm, 1 if the update was applied else 0
};

__device__ __forceinline__ void adam_elem(float& p, float& g, float& m, float& v, const AdamArgs& a, float coef) {
  g *= coef;
  m = m + a.omb1 * (g - m);            // exp_avg.lerp_(grad, 1 - beta1)
  v = a.beta2 * v + a.omb2 * (g * g);  // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
  const float denom = sqrtf(v) * a.rsqrt_bc2 + a.eps;
  p -= a.lr_over_bc1 * (m / denom);
}

__global__ void __launch_bounds__(OPT_THREADS) adam_step_kernel(const AdamArgs a) {
  __shared__ float red[OPT_THREADS / 32];
  // global norm: every block sums the same partials in the same order
  float s = 0.f;
  for (int i = threadIdx.x; i < a.n_chunks; i += OPT_THREADS) s += a.partials[i];
  const float norm = sqrtf(block_sum(s, red));
  // the trainer's rule is `not (norm <= skip_grad_norm)`: a NaN norm skips the step too
  const bool skip = a.skip_above > 0.f && !(norm <= a.skip_above);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.norm_out[0] = norm;
    a.norm_out[1] = skip ? 0.f : 1.f;
  }
  if (skip) return;
  // torch.nn.utils.clip_grad_norm_: clamp(max_norm / (norm + 1e-6), max=1).  A NaN norm keeps a NaN coefficient, which
  // turns every gradient, moment and parameter into NaN as torch's multiply does.
  float coef = a.max_norm / (norm + 1e-6f);
  coef = coef > 1.f ? 1.f : coef;
  const bool write_g = !(coef >= 1.f);  // clipping scales .grad in place, visibly

  const int2 ck = a.chunks[blockIdx.x];
  float* p = a.params[ck.x];
  float* g = a.grads[ck.x];
  float* m = a.exp_avg[ck.x];
  float* v = a.exp_avg_sq[ck.x];
  const int64_t n = a.numel[ck.x];
  const int64_t lo = (int64_t)ck.y * a.chunk_elems;
  const int64_t hi = min(lo + (int64_t)a.chunk_elems, n);
  const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                     reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  int64_t tail = lo;
  if (vec) {
    const int64_t lo4 = lo / 4, hi4 = hi / 4;
    for (int64_t i = lo4 + threadIdx.x; i < hi4; i += OPT_THREADS) {
      float4 P = reinterpret_cast<float4*>(p)[i], G = reinterpret_cast<float4*>(g)[i];
      float4 M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
      adam_elem(P.x, G.x, M.x, V.x, a, coef);
      adam_elem(P.y, G.y, M.y, V.y, a, coef);
      adam_elem(P.z, G.z, M.z, V.z, a, coef);
      adam_elem(P.w, G.w, M.w, V.w, a, coef);
      reinterpret_cast<float4*>(p)[i] = P;
      reinterpret_cast<float4*>(m)[i] = M;
      reinterpret_cast<float4*>(v)[i] = V;
      if (write_g) reinterpret_cast<float4*>(g)[i] = G;
    }
    tail = hi4 * 4;
  }
  for (int64_t i = tail + threadIdx.x; i < hi; i += OPT_THREADS) {
    float P = p[i], G = g[i], M = m[i], V = v[i];
    adam_elem(P, G, M, V, a, coef);
    p[i] = P; m[i] = M; v[i] = V;
    if (write_g) g[i] = G;
  }
}

}  // namespace

extern "C" int pg_grad_sqnorm(const void* grad_ptrs, const int64_t* numel, const void* chunks, int n_chunks, int chunk_elems,
                              float* partials, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(grad_ptrs && numel && chunks && partials && n_chunks > 0, "pg_grad_sqnorm: null/empty argument");
  PG_REQUIRE(chunk_elems > 0 && chunk_elems % 4 == 0, "pg_grad_sqnorm: chunk_elems must be a positive multiple of 4");
  grad_sqnorm_kernel<<<n_chunks, OPT_THREADS, 0, stream>>>(reinterpret_cast<const float* const*>(grad_ptrs), numel,
                                                          reinterpret_cast<const int2*>(chunks), chunk_elems, partials);
  return pg_check_launch("pg_grad_sqnorm");
}

extern "C" int pg_adam_step(const void* param_ptrs, const void* grad_ptrs, const void* exp_avg_ptrs, const void* exp_avg_sq_ptrs,
                            const int64_t* numel, const void* chunks, int n_chunks, int chunk_elems, const float* partials,
                            float max_norm, float skip_above, double lr, double beta1d, double beta2d, double epsd, int step,
                            float* norm_out, void* stream_) {
  const float beta1 = (float)beta1d, beta2 = (float)beta2d, eps = (float)epsd;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(param_ptrs && grad_ptrs && exp_avg_ptrs && exp_avg_sq_ptrs && numel && chunks && partials && norm_out,
             "pg_adam_step: null argument");
  PG_REQUIRE(n_chunks > 0 && chunk_elems > 0 && chunk_elems % 4 == 0 && step >= 1, "pg_adam_step: bad chunking / step");
  AdamArgs a;
  a.params = reinterpret_cast<float* const*>(param_ptrs);
  a.grads = reinterpret_cast<float* const*>(grad_ptrs);
  a.exp_avg = reinterpret_cast<float* const*>(exp_avg_ptrs);
  a.exp_avg_sq = reinterpret_cast<float* const*>(exp_avg_sq_ptrs);
  a.numel = numel;
  a.chunks = reinterpret_cast<const int2*>(chunks);
  a.partials = partials;
  a.n_chunks = n_chunks;
  a.chunk_elems = chunk_elems;
  a.max_norm = max_norm;
  a.skip_above = skip_above;
  // host-side scalars in double, like torch's _single_tensor_adam
  const double bc1 = 1.0 - pow(beta1d, (double)step);
  const double bc2 = 1.0 - pow(beta2d, (double)step);
  a.lr_over_bc1 = (float)(lr / bc1);
  a.rsqrt_bc2 = (float)(1.0 / sqrt(bc2));
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps;
  a.omb1 = (float)(1.0 - (double)beta1d);
  a.omb2 = (float)(1.0 - (double)beta2d);
  a.norm_out = norm_out;
  adam_step_kernel<<<n_chunks, OPT_THREADS, 0, stream>>>(a);
  return pg_check_launch("pg_adam_step");
}

extern "C" int pg_cast_multi_bf16(const void* src_ptrs, const void* dst_ptrs, const int64_t* numel, const void* chunks,
                                  int n_chunks, int chunk_elems, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(src_ptrs && dst_ptrs && numel && chunks && n_chunks > 0, "pg_cast_multi_bf16: null/empty argument");
  PG_REQUIRE(chunk_elems > 0 && chunk_elems % 8 == 0, "pg_cast_multi_bf16: chunk_elems must be a positive multiple of 8");
  cast_multi_kernel<<<n_chunks, OPT_THREADS, 0, stream>>>(reinterpret_cast<const float* const*>(src_ptrs),
                                                         reinterpret_cast<bf16* const*>(dst_ptrs), numel,
                                                         reinterpret_cast<const int2*>(chunks), chunk_elems);
  return pg_check_launch("pg_cast_multi_bf16");
}
