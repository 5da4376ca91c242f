// pg_vae.cu — the Gaussian latent of VAE / BetaVAE (reference models/vae/vae.py `forward`, vaes.py
// `unit_gaussian_kl_div`, `sample_from_gaussian`): between the encoder's last convolution and the decoder's first one.
// The encoder output h is pixel-major fp32 [n*hw, ld_h]: columns [0, L) hold the mean and [L, 2L) log_std (the
// reference's torch.split along channels).  The noise eps comes in the reference's NCHW order [n, L, hw].  Each image's
// KL sum is one CTA: every thread adds its entries in ascending index order and the CTA's threads are combined by a
// fixed tree, so the result is the same on every run.  No atomics.  The roundings are the reference's: each product and
// sum is rounded on its own (no fused multiply-add), and exp is expf.
#include "pg_common.cuh"

namespace {

constexpr int THREADS = 256;

__global__ void __launch_bounds__(THREADS)
vae_latent_fwd_kernel(const float* __restrict__ h, long long ld_h, const float* __restrict__ eps, int L, int hw,
                      bf16* __restrict__ z, long long ld_z, float* __restrict__ kl) {
  const int b = blockIdx.x;
  const long long per_image = (long long)hw * ld_z;
  float acc = 0.f;
  for (long long e = threadIdx.x; e < per_image; e += THREADS) {
    const int pix = (int)(e / ld_z), c = (int)(e % ld_z);
    const long long row = (long long)b * hw + pix;
    float zv = 0.f;
    if (c < L) {
      const float m = h[row * ld_h + c], ls = h[row * ld_h + L + c];
      const float sd = expf(ls);
      zv = __fadd_rn(m, __fmul_rn(sd, eps[((long long)b * L + c) * hw + pix]));
      // -0.5 * (1 + 2 log_std - exp(log_std)^2 - mean^2)
      float t = __fadd_rn(1.f, __fmul_rn(2.f, ls));
      t = __fsub_rn(t, __fmul_rn(sd, sd));
      t = __fsub_rn(t, __fmul_rn(m, m));
      acc = __fadd_rn(acc, __fmul_rn(-0.5f, t));
    }
    z[row * ld_z + c] = __float2bfloat16(zv);
  }
  __shared__ float part[THREADS / 32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < THREADS / 32; ++w) s += part[w];
    kl[b] = s;
  }
}

// dmean = dz + g mean,  dlog_std = dz exp(log_std) eps + g (exp(log_std)^2 - 1),  zero in dh's pad columns.
__global__ void __launch_bounds__(THREADS)
vae_latent_bwd_kernel(const float* __restrict__ h, long long ld_h, const float* __restrict__ eps,
                      const bf16* __restrict__ dz, long long ld_dz, const float* __restrict__ g_kl, int n, int L, int hw,
                      bf16* __restrict__ dh, long long ld_dh) {
  const long long total = (long long)n * hw * ld_dh;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long row = i / ld_dh;
    const int c = (int)(i % ld_dh);
    float v = 0.f;
    if (c < 2 * L) {
      const int b = (int)(row / hw), pix = (int)(row % hw), j = c < L ? c : c - L;
      const float m = h[row * ld_h + j], ls = h[row * ld_h + L + j];
      const float d = __bfloat162float(dz[row * ld_dz + j]);
      const float g = g_kl ? g_kl[b] : 0.f;
      if (c < L) {
        v = d + g * m;
      } else {
        const float sd = expf(ls);
        v = d * sd * eps[((long long)b * L + j) * hw + pix] + g * (sd * sd - 1.f);
      }
    }
    dh[i] = __float2bfloat16(v);
  }
}

}  // namespace

extern "C" int pg_vae_latent_fwd(const float* h, int64_t ld_h, const float* eps, int n, int L, int hw, void* z,
                                 int64_t ld_z, float* kl, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(h && eps && z && kl, "pg_vae_latent_fwd: null argument");
  PG_REQUIRE(n >= 0 && L >= 1 && hw >= 1, "pg_vae_latent_fwd: n = %d, L = %d, hw = %d", n, L, hw);
  PG_REQUIRE(ld_h >= 2 * L && ld_z >= L && ld_z % 8 == 0,
             "pg_vae_latent_fwd: pitches ld_h = %lld (>= 2L) and ld_z = %lld (>= L, a multiple of 8) for L = %d",
             (long long)ld_h, (long long)ld_z, L);
  PG_REQUIRE(pg_aligned16(z), "pg_vae_latent_fwd: z must be 16-byte aligned");
  if (n == 0) return 0;
  vae_latent_fwd_kernel<<<n, THREADS, 0, stream>>>(h, ld_h, eps, L, hw, (bf16*)z, ld_z, kl);
  return pg_check_launch("pg_vae_latent_fwd");
}

extern "C" int pg_vae_latent_bwd(const float* h, int64_t ld_h, const float* eps, const void* dz, int64_t ld_dz,
                                 const float* g_kl, int n, int L, int hw, void* dh, int64_t ld_dh, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(h && eps && dz && dh, "pg_vae_latent_bwd: null argument");
  PG_REQUIRE(n >= 0 && L >= 1 && hw >= 1, "pg_vae_latent_bwd: n = %d, L = %d, hw = %d", n, L, hw);
  PG_REQUIRE(ld_h >= 2 * L && ld_dz >= L && ld_dh >= 2 * L && ld_dh % 8 == 0,
             "pg_vae_latent_bwd: pitches ld_h = %lld, ld_dz = %lld, ld_dh = %lld (a multiple of 8) for L = %d",
             (long long)ld_h, (long long)ld_dz, (long long)ld_dh, L);
  PG_REQUIRE(pg_aligned16(dh), "pg_vae_latent_bwd: dh must be 16-byte aligned");
  const long long total = (long long)n * hw * ld_dh;
  if (total == 0) return 0;
  long long blocks = (total + THREADS - 1) / THREADS;
  const long long cap = (long long)pg_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  vae_latent_bwd_kernel<<<(unsigned)blocks, THREADS, 0, stream>>>(h, ld_h, eps, (const bf16*)dz, ld_dz, g_kl, n, L, hw,
                                                                  (bf16*)dh, ld_dh);
  return pg_check_launch("pg_vae_latent_bwd");
}
