// pg_categorical.cu — the 256-way (any K >= 2) categorical likelihood of 8-bit images: a fused cross-entropy forward and
// backward over NCHW logits, and the per-pixel categorical draw of the samplers.
//
// Layout (losses.py owns the convention): an image of C channels has K * C logit channels, class k of channel c is logit
// channel k * C + c, i.e. the NCHW logits viewed as [N, K, C, HW].  Target class of an input value x:
// rint(clamp(x, 0, 1) * (K - 1)).  Every sum over k runs in ascending k; the per-image sums are block partials added
// in block order by pg_sum_partials: no atomics, every run gives the same bits.
#include "pg_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int UNROLL = 8;  // logits loads issued together per thread (they are independent; the recurrence is not)

// Thread (n, i) with i = c * HW + p over blockIdx.x; logit k of it is at logits[(n K + k) C HW + i], so a warp's loads
// are consecutive addresses for every k.
__global__ void __launch_bounds__(THREADS)
categorical_xent_kernel(const float* __restrict__ logits, const float* __restrict__ x, int K, long long CHW, float grad_scale,
                        float* __restrict__ nll, float* __restrict__ part, int n_img, float* __restrict__ dlogits) {
  __shared__ float red[THREADS / 32];
  const int n = blockIdx.y;
  const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
  float loss = 0.f;
  if (i < CHW) {
    const float* lp = logits + (long long)n * K * CHW + i;
    const int t = target_class(x[(long long)n * CHW + i], K);
    OnlineLse acc;
    int k = 0;
    for (; k + UNROLL <= K; k += UNROLL) {
      float v[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) v[j] = lp[(long long)(k + j) * CHW];
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) acc.add(v[j]);
    }
    for (; k < K; ++k) acc.add(lp[(long long)k * CHW]);
    const float lt = lp[(long long)t * CHW];
    loss = logf(acc.s) + (acc.m - lt);
    if (nll) nll[(long long)n * CHW + i] = loss;
    if (dlogits) {
      float* dp = dlogits + (long long)n * K * CHW + i;
      const float inv_s = 1.f / acc.s;
      for (k = 0; k + UNROLL <= K; k += UNROLL) {
        float v[UNROLL];
#pragma unroll
        for (int j = 0; j < UNROLL; ++j) v[j] = lp[(long long)(k + j) * CHW];
#pragma unroll
        for (int j = 0; j < UNROLL; ++j)
          dp[(long long)(k + j) * CHW] = (expf(v[j] - acc.m) * inv_s - (k + j == t ? 1.f : 0.f)) * grad_scale;
      }
      for (; k < K; ++k)
        dp[(long long)k * CHW] = (expf(lp[(long long)k * CHW] - acc.m) * inv_s - (k == t ? 1.f : 0.f)) * grad_scale;
    }
  }
  if (!part) return;
  loss = warp_sum(loss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = loss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < THREADS / 32 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) part[(long long)blockIdx.x * n_img + n] = v;
  }
}

// Thread (r, c): class k of row r is logits[r ld + k C + c].  Draws the first k whose ascending cumulative sum of
// exp(l - max) reaches u * sum (the cumulative and the sum are the same additions, so some k always qualifies for u <= 1).
__global__ void __launch_bounds__(THREADS)
categorical_sample_kernel(const float* __restrict__ logits, long long ld, int rows, int K, int C, const float* __restrict__ u,
                          float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (idx >= (long long)rows * C) return;
  const long long r = idx / C;
  const int c = (int)(idx % C);
  const float* lp = logits + r * ld + c;
  float m = -INFINITY;
  for (int k = 0; k < K; ++k) m = fmaxf(m, lp[(long long)k * C]);
  float s = 0.f;
  for (int k = 0; k < K; ++k) s += expf(lp[(long long)k * C] - m);
  const float target = u[idx] * s;
  float cum = 0.f;
  int pick = K - 1;  // NaN logits: no comparison holds
  for (int k = 0; k < K; ++k) {
    cum += expf(lp[(long long)k * C] - m);
    if (cum >= target) {
      pick = k;
      break;
    }
  }
  out[idx] = (float)pick / (float)(K - 1);
}

}  // namespace

extern "C" int pg_categorical_xent_fwd_bwd(const float* logits, const float* x, int N, int K, int C, int64_t HW,
                                           float grad_scale, float* nll, float* image_nll, float* dlogits,
                                           void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(N >= 1 && K >= 2 && C >= 1 && HW >= 1, "pg_categorical_xent_fwd_bwd: bad shape (N %d, K %d, C %d, HW %lld)",
             N, K, C, (long long)HW);
  PG_REQUIRE(N <= 65535, "pg_categorical_xent_fwd_bwd: %d images (at most 65535 per call)", N);
  PG_REQUIRE(logits && x, "pg_categorical_xent_fwd_bwd: null argument");
  const long long CHW = (long long)C * HW;
  const long long blocks = (CHW + THREADS - 1) / THREADS;
  PG_REQUIRE(blocks < (1LL << 31), "pg_categorical_xent_fwd_bwd: %lld pixels per image is too many", CHW);
  float* part = nullptr;
  if (image_nll && pg_scratch((size_t)blocks * N * sizeof(float), stream, &part)) return 1;
  categorical_xent_kernel<<<dim3((unsigned)blocks, N), THREADS, 0, stream>>>(logits, x, K, CHW, grad_scale, nll, part, N,
                                                                             dlogits);
  if (pg_check_launch("pg_categorical_xent_fwd_bwd")) return 1;
  return image_nll ? pg_sum_partials(part, (int)blocks, N, 1, N, N, image_nll, stream) : 0;
}

extern "C" int pg_categorical_sample(const float* logits, int64_t ld, int rows, int K, int C, const float* u,
                                     float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(rows >= 0 && K >= 2 && C >= 1, "pg_categorical_sample: bad shape (rows %d, K %d, C %d)", rows, K, C);
  PG_REQUIRE(ld >= (int64_t)K * C, "pg_categorical_sample: pitch %lld narrower than K * C = %lld", (long long)ld,
             (long long)K * C);
  if (rows == 0) return 0;
  PG_REQUIRE(logits && u && out, "pg_categorical_sample: null argument");
  const long long total = (long long)rows * C;
  categorical_sample_kernel<<<(unsigned)((total + THREADS - 1) / THREADS), THREADS, 0, stream>>>(logits, ld, rows, K, C,
                                                                                                 u, out);
  return pg_check_launch("pg_categorical_sample");
}
