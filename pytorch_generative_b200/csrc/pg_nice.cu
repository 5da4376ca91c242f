// pg_nice.cu — NICE (reference models/flow/nice.py): the elementwise ends of the flow around the coupling GEMMs.  The
// flow's stream is two fp32 half buffers lo = x[:, :D/2] and hi = x[:, D/2:], each of pitch ld >= D - D/2 with zero pad
// columns, so that a coupling network reads one half as a GEMM operand and writes the other as a new buffer (see
// include/pg_b200.h).  These kernels split an [n, D] matrix into the halves, join them back with the diagonal scaling,
// give the scaling's gradients and evaluate the logistic prior.  Every sum runs in a fixed order and there are no atomics.
#include "pg_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int SPLIT_ROWS = 128;  // images per batch slice of the log-scale gradient (fewer slices for small batches)
constexpr int MAX_SPLITS = 32;

// Column q of the halves' joint index space [0, 2 ld): half = q / ld, column c = q % ld of that half, feature j of x.
struct HalfCol {
  int half, c, j;
  bool valid;
};
__device__ __forceinline__ HalfCol half_col(long long q, int D, long long ld) {
  const int h_lo = D / 2, h_hi = D - D / 2;
  HalfCol r;
  r.half = (int)(q / ld);
  r.c = (int)(q % ld);
  r.j = r.half ? h_lo + r.c : r.c;
  r.valid = r.c < (r.half ? h_hi : h_lo);
  return r;
}

__global__ void __launch_bounds__(THREADS) nice_split_kernel(const float* __restrict__ x, int n, int D,
                                                            const float* __restrict__ log_scale, float sign,
                                                            float* __restrict__ lo, float* __restrict__ hi, long long ld,
                                                            int bf16_half, bf16* __restrict__ out_bf16) {
  const long long total = (long long)n * 2 * ld;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long b = i / (2 * ld);
    const HalfCol h = half_col(i % (2 * ld), D, ld);
    float v = 0.f;
    if (h.valid) {
      v = x[b * D + h.j];
      if (log_scale) v = v * expf(sign * log_scale[h.j]);
    }
    (h.half ? hi : lo)[b * ld + h.c] = v;
    if (out_bf16 && h.half == bf16_half) out_bf16[b * ld + h.c] = __float2bfloat16_rn(v);
  }
}

// Thread (b, j) writes z[b, j]; thread 0 of block 0 also sums the log-scales in ascending j.
__global__ void __launch_bounds__(THREADS) nice_join_kernel(const float* __restrict__ lo, const float* __restrict__ hi,
                                                           long long ld, int n, int D, const float* __restrict__ log_scale,
                                                           float sign, float* __restrict__ z, float* __restrict__ log_det) {
  if (log_det && blockIdx.x == 0 && threadIdx.x == 0) {
    float acc = 0.f;
    for (int j = 0; j < D; ++j) acc += log_scale[j];
    *log_det = acc;
  }
  const int h_lo = D / 2;
  const long long total = (long long)n * D;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long b = i / D;
    const int j = (int)(i % D);
    float v = j < h_lo ? lo[b * ld + j] : hi[b * ld + j - h_lo];
    if (log_scale) v = v * expf(sign * log_scale[j]);
    z[i] = v;
  }
}

// CTA (column block, batch slice): thread = one column q of the halves' index space, walking the slice's images in
// index order.  d = dz * exp(s) goes to the halves (and the bf16 copy of one half); the slice's sum of dz * z over its
// images, one fmaf chain per column, goes to the scratch partials.  Slice 0 initialises d_log_scale to g_log_det.
__global__ void __launch_bounds__(THREADS) nice_scale_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ z,
                                                                const float* __restrict__ log_scale,
                                                                const float* __restrict__ g_log_det, int n, int D,
                                                                float* __restrict__ d_lo, float* __restrict__ d_hi,
                                                                long long ld, int bf16_half, bf16* __restrict__ dm,
                                                                int per_split, float* __restrict__ part,
                                                                float* __restrict__ d_log_scale) {
  const long long q = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (q >= 2 * ld) return;
  const HalfCol h = half_col(q, D, ld);
  const int slice = blockIdx.y;
  const int bs = slice * per_split, be = min(n, bs + per_split);
  float* d = h.half ? d_hi : d_lo;
  const bool want_bf16 = dm && h.half == bf16_half;
  if (!h.valid) {
    for (int b = bs; b < be; ++b) {
      d[(long long)b * ld + h.c] = 0.f;
      if (want_bf16) dm[(long long)b * ld + h.c] = __float2bfloat16_rn(0.f);
    }
    return;
  }
  const float e = expf(log_scale[h.j]);
  float acc = 0.f;
  for (int b = bs; b < be; ++b) {
    const float g = dz[(long long)b * D + h.j];
    const float v = g * e;
    d[(long long)b * ld + h.c] = v;
    if (want_bf16) dm[(long long)b * ld + h.c] = __float2bfloat16_rn(v);
    acc = fmaf(g, z[(long long)b * D + h.j], acc);
  }
  part[(long long)slice * D + h.j] = acc;
  if (slice == 0) d_log_scale[h.j] = g_log_det ? *g_log_det : 0.f;
}

// One CTA per image: each thread sums its columns j = t, t + 256, ... in ascending order, the warps combine their lanes
// with a fixed butterfly and warp 0 adds the 8 warp sums in warp order.
__global__ void __launch_bounds__(THREADS) logistic_prior_kernel(const float* __restrict__ z, int D, float grad_scale,
                                                                float* __restrict__ log_prob, float* __restrict__ dz) {
  __shared__ float warp_sums[THREADS / 32];
  const long long row = (long long)blockIdx.x * D;
  float acc = 0.f;
  for (int j = threadIdx.x; j < D; j += THREADS) {
    const float v = z[row + j];
    const float a = fabsf(v);
    acc += a + 2.f * log1pf(expf(-a));  // softplus(v) + softplus(-v)
    if (dz) dz[row + j] = grad_scale * tanhf(0.5f * v);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) s += warp_sums[w];
    log_prob[blockIdx.x] = -s;
  }
}

unsigned grid_for(long long total) {
  long long blocks = (total + THREADS - 1) / THREADS;
  const long long cap = (long long)pg_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks < 1 ? 1 : blocks);
}

}  // namespace

extern "C" int pg_nice_split(const float* x, int n, int D, const float* log_scale, float sign, float* lo, float* hi,
                             int64_t ld, int bf16_half, void* out_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D >= 1, "pg_nice_split: empty problem (n %d, D %d)", n, D);
  PG_REQUIRE(ld >= D - D / 2, "pg_nice_split: pitch %lld narrower than the half (%d)", (long long)ld, D - D / 2);
  PG_REQUIRE(!out_bf16 || bf16_half == 0 || bf16_half == 1, "pg_nice_split: bf16_half %d is not 0 or 1", bf16_half);
  if (n == 0) return 0;
  PG_REQUIRE(x && lo && hi, "pg_nice_split: null argument");
  nice_split_kernel<<<grid_for((long long)n * 2 * ld), THREADS, 0, stream>>>(x, n, D, log_scale, sign, lo, hi, ld,
                                                                             bf16_half, (bf16*)out_bf16);
  return pg_check_launch("pg_nice_split");
}

extern "C" int pg_nice_join(const float* lo, const float* hi, int64_t ld, int n, int D, const float* log_scale, float sign,
                            float* z, float* log_det, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D >= 1, "pg_nice_join: empty problem (n %d, D %d)", n, D);
  PG_REQUIRE(ld >= D - D / 2, "pg_nice_join: pitch %lld narrower than the half (%d)", (long long)ld, D - D / 2);
  PG_REQUIRE(!log_det || log_scale, "pg_nice_join: log_det needs log_scale");
  if (n == 0 && !log_det) return 0;
  PG_REQUIRE(n == 0 || (lo && hi && z), "pg_nice_join: null argument");
  nice_join_kernel<<<grid_for((long long)n * D), THREADS, 0, stream>>>(lo, hi, ld, n, D, log_scale, sign, z, log_det);
  return pg_check_launch("pg_nice_join");
}

extern "C" int pg_nice_scale_bwd(const float* dz, const float* z, const float* log_scale, const float* g_log_det, int n,
                                 int D, float* d_lo, float* d_hi, int64_t ld, int bf16_half, void* dm_bf16,
                                 float* d_log_scale, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D >= 1, "pg_nice_scale_bwd: empty problem (n %d, D %d)", n, D);
  PG_REQUIRE(ld >= D - D / 2, "pg_nice_scale_bwd: pitch %lld narrower than the half (%d)", (long long)ld, D - D / 2);
  PG_REQUIRE(!dm_bf16 || bf16_half == 0 || bf16_half == 1, "pg_nice_scale_bwd: bf16_half %d is not 0 or 1", bf16_half);
  PG_REQUIRE(log_scale && d_log_scale && (n == 0 || (dz && z && d_lo && d_hi)), "pg_nice_scale_bwd: null argument");
  // batch slices: decided by n alone, so every run of a shape adds the same partials in the same order (no images: one
  // empty slice, so d_log_scale = g_log_det)
  int splits = 1, per_split = 0;
  if (n > 0) {
    splits = (n + SPLIT_ROWS - 1) / SPLIT_ROWS;
    if (splits > MAX_SPLITS) splits = MAX_SPLITS;
    per_split = (n + splits - 1) / splits;
    splits = (n + per_split - 1) / per_split;
  }
  float* part = nullptr;
  if (pg_scratch((size_t)splits * D * sizeof(float), stream, &part)) return 1;
  const long long cols = (2 * ld + THREADS - 1) / THREADS;
  PG_REQUIRE(cols < (1LL << 31), "pg_nice_scale_bwd: pitch %lld is too large", (long long)ld);
  nice_scale_bwd_kernel<<<dim3((unsigned)cols, splits), THREADS, 0, stream>>>(
      dz, z, log_scale, g_log_det, n, D, d_lo, d_hi, ld, bf16_half, (bf16*)dm_bf16, per_split, part, d_log_scale);
  if (pg_check_launch("pg_nice_scale_bwd")) return 1;
  return pg_sum_partials(part, splits, D, 1, D, D, d_log_scale, stream);
}

extern "C" int pg_logistic_prior_fwd_bwd(const float* z, int n, int D, float grad_scale, float* log_prob, float* dz,
                                         void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D >= 1, "pg_logistic_prior_fwd_bwd: empty problem (n %d, D %d)", n, D);
  if (n == 0) return 0;
  PG_REQUIRE(z && log_prob, "pg_logistic_prior_fwd_bwd: null argument");
  logistic_prior_kernel<<<(unsigned)n, THREADS, 0, stream>>>(z, D, grad_scale, log_prob, dz);
  return pg_check_launch("pg_logistic_prior_fwd_bwd");
}
