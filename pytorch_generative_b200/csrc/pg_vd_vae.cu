// pg_vd_vae.cu — the elementwise stages of VeryDeepVAE (reference models/vae/vd_vae.py) between its convolutions:
// GELU operands with their stored derivative, the two-Gaussian latent of a TopDownBlock, 2x2 average pooling and the
// decoder's bias + nearest-neighbour unpooling.  Streams are pixel-major fp32 [n*h*w, ld >= C].  Every reduction runs
// in a fixed order (one thread or one CTA owns each sum), no kernel uses atomics, and every access is scalar, so no
// operand needs an aligned base.
#include "pg_common.cuh"

namespace {

constexpr int THREADS = 256;

unsigned grid_for(long long total) {
  long long blocks = (total + THREADS - 1) / THREADS;
  const long long cap = (long long)pg_num_sms() * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

__global__ void __launch_bounds__(THREADS)
gelu_cast_kernel(const float* __restrict__ x, long long ld_x, int P, int C, int width, bf16* __restrict__ g,
                 bf16* __restrict__ d, long long ld_out) {
  const long long total = (long long)P * width;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long r = i / width;
    const int c = (int)(i % width);
    float gv = 0.f, dv = 0.f;
    if (c < C) pg_gelu_both(x[r * ld_x + c], gv, dv);
    g[r * ld_out + c] = __float2bfloat16(gv);
    d[r * ld_out + c] = __float2bfloat16(dv);
  }
}

// One CTA per image.  KL(q || p) = -0.5 + (t - s) + (e^{2s} + (m_q - m_p)^2) / (2 e^{2t}), s = q_log_std,
// t = p_log_std, rounded operation by operation in the reference's order (vaes.py gaussian_kl_div).
__global__ void __launch_bounds__(THREADS)
vd_latent_fwd_kernel(const float* __restrict__ prior, long long ld_prior, const float* __restrict__ post,
                     long long ld_post, const float* __restrict__ x, long long ld_x, const float* __restrict__ eps, int L,
                     int C, int hw, bf16* __restrict__ z, long long ld_z, float* __restrict__ s, long long ld_s,
                     const float* __restrict__ kl_in, float* __restrict__ kl_out) {
  const int b = blockIdx.x;
  const long long row0 = (long long)b * hw;
  float acc = 0.f;
  for (long long e = threadIdx.x; e < (long long)hw * ld_z; e += THREADS) {
    const int pix = (int)(e / ld_z), c = (int)(e % ld_z);
    const long long row = row0 + pix;
    float zv = 0.f;
    if (c < L) {
      const float pm = prior[row * ld_prior + c], pt = prior[row * ld_prior + L + c];
      const float ep = eps[((long long)b * L + c) * hw + pix];
      if (post) {
        const float qm = post[row * ld_post + c], qs = post[row * ld_post + L + c];
        zv = __fadd_rn(qm, __fmul_rn(expf(qs), ep));
        const float dm = __fsub_rn(qm, pm);
        const float md = __fmul_rn(dm, dm);
        const float es = expf(qs), et = expf(pt);
        const float pv = __fmul_rn(es, es), qv = __fmul_rn(2.f, __fmul_rn(et, et));
        const float k = __fadd_rn(__fadd_rn(-0.5f, __fsub_rn(pt, qs)), __fdiv_rn(__fadd_rn(pv, md), qv));
        acc = __fadd_rn(acc, k);
      } else {
        zv = __fadd_rn(pm, __fmul_rn(expf(pt), ep));
      }
    }
    z[row * ld_z + c] = __float2bfloat16(zv);
  }
  for (long long e = threadIdx.x; e < (long long)hw * C; e += THREADS) {
    const long long row = row0 + e / C;
    const int c = (int)(e % C);
    s[row * ld_s + c] = __fadd_rn(x[row * ld_x + c], prior[row * ld_prior + 2 * L + c]);
  }
  if (!post) return;
  __shared__ float part[THREADS / 32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < THREADS / 32; ++w) t += part[w];
    kl_out[b] = kl_in ? __fadd_rn(kl_in[b], t) : t;
  }
}

// dprior = [dm_p | dt | bf16(dsum) | 0], dpost = [dm_q | ds | 0]; with d = m_q - m_p and v = e^{2t}:
//   dm_q = dz + g d / v,  ds = dz e^s eps + g (e^{2s} / v - 1),  dm_p = -g d / v,  dt = g (1 - (e^{2s} + d^2) / v).
// Sampling from the prior (post == NULL): dm_p = dz, dt = dz e^t eps.
__global__ void __launch_bounds__(THREADS)
vd_latent_bwd_kernel(const float* __restrict__ prior, long long ld_prior, const float* __restrict__ post,
                     long long ld_post, const float* __restrict__ eps, const bf16* __restrict__ dz, long long ld_dz,
                     const float* __restrict__ g_kl, const float* __restrict__ dsum, long long ld_dsum, int n, int L,
                     int C, int hw, bf16* __restrict__ dprior, long long ld_dprior, bf16* __restrict__ dpost,
                     long long ld_dpost) {
  const long long rows = (long long)n * hw;
  const int width = (int)(ld_dprior > ld_dpost ? ld_dprior : ld_dpost);
  const long long total = rows * width;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long row = i / width;
    const int c = (int)(i % width);
    const int b = (int)(row / hw), pix = (int)(row % hw);
    float vp = 0.f, vq = 0.f;
    if (c < 2 * L) {
      const int j = c < L ? c : c - L;
      const float dzv = dz ? __bfloat162float(dz[row * ld_dz + j]) : 0.f;
      const float ep = eps[((long long)b * L + j) * hw + pix];
      const float pm = prior[row * ld_prior + j], pt = prior[row * ld_prior + L + j];
      if (post) {
        const float g = g_kl ? g_kl[b] : 0.f;
        const float qm = post[row * ld_post + j], qs = post[row * ld_post + L + j];
        const float d = qm - pm, v = expf(2.f * pt), e2s = expf(2.f * qs);
        if (c < L) {
          vq = dzv + g * d / v;
          vp = -g * d / v;
        } else {
          vq = dzv * expf(qs) * ep + g * (e2s / v - 1.f);
          vp = g * (1.f - (e2s + d * d) / v);
        }
      } else {
        vp = c < L ? dzv : dzv * expf(pt) * ep;
      }
    } else if (c < 2 * L + C) {
      vp = dsum[row * ld_dsum + c - 2 * L];
    }
    if (c < ld_dprior) dprior[row * ld_dprior + c] = __float2bfloat16(vp);
    if (dpost && c < ld_dpost) dpost[row * ld_dpost + c] = __float2bfloat16(vq);
  }
}

// y = the mean of each 2x2 window ((x00 + x01) + x10) + x11) / 4, as nn.AvgPool2d(2, 2): odd last rows / columns are
// dropped.
__global__ void __launch_bounds__(THREADS)
avg_pool2_fwd_kernel(const float* __restrict__ x, long long ld_x, int n, int h, int w, int C, float* __restrict__ y,
                     long long ld_y) {
  const int ho = h / 2, wo = w / 2;
  const long long total = (long long)n * ho * wo * C;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int j = (int)(r % wo), t = (int)(r / wo), ii = t % ho, b = t / ho;
    const long long r00 = ((long long)b * h + 2 * ii) * w + 2 * j;
    float v = __fadd_rn(x[r00 * ld_x + c], x[(r00 + 1) * ld_x + c]);
    v = __fadd_rn(v, x[(r00 + w) * ld_x + c]);
    v = __fadd_rn(v, x[(r00 + w + 1) * ld_x + c]);
    y[r * ld_y + c] = __fdiv_rn(v, 4.f);
  }
}

__global__ void __launch_bounds__(THREADS)
avg_pool2_bwd_kernel(const float* __restrict__ dy, long long ld_dy, int n, int h, int w, int C, float* __restrict__ dx,
                     long long ld_dx) {
  const int ho = h / 2, wo = w / 2;
  const long long total = (long long)n * h * w * C;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int j = (int)(r % w), t = (int)(r / w), ii = t % h, b = t / h;
    float v = 0.f;
    if (ii / 2 < ho && j / 2 < wo) v = __fdiv_rn(dy[(((long long)b * ho + ii / 2) * wo + j / 2) * ld_dy + c], 4.f);
    dx[r * ld_dx + c] = v;
  }
}

// y[b, I, J] = x[b, I / f, J / f] + bias[:, I / f, J / f] (x == NULL: 0 + bias), bias NCHW [1, C, s, s].
__global__ void __launch_bounds__(THREADS)
bias_unpool_fwd_kernel(const float* __restrict__ x, long long ld_x, const float* __restrict__ bias, int n, int s, int C,
                       int f, float* __restrict__ y, long long ld_y) {
  const int S = s * f;
  const long long total = (long long)n * S * S * C;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int J = (int)(r % S), t = (int)(r / S), I = t % S, b = t / S;
    const int si = I / f, sj = J / f;
    const float xv = x ? x[(((long long)b * s + si) * s + sj) * ld_x + c] : 0.f;
    y[r * ld_y + c] = __fadd_rn(xv, bias[((long long)c * s + si) * s + sj]);
  }
}

// One thread per (i, j, c) of the small image: for each image in ascending order, the sum of its f x f children in
// raster order is dx (when wanted) and is added to dbias.
__global__ void __launch_bounds__(THREADS)
bias_unpool_bwd_kernel(const float* __restrict__ dy, long long ld_dy, int n, int s, int C, int f, float* __restrict__ dx,
                       long long ld_dx, float* __restrict__ dbias) {
  const int S = s * f;
  const long long total = (long long)s * s * C;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int c = (int)(i % C);
    const int r = (int)(i / C), sj = r % s, si = r / s;
    float acc = 0.f;
    for (int b = 0; b < n; ++b) {
      float v = 0.f;
      for (int a = 0; a < f; ++a)
        for (int e = 0; e < f; ++e) v = __fadd_rn(v, dy[(((long long)b * S + si * f + a) * S + sj * f + e) * ld_dy + c]);
      if (dx) dx[(((long long)b * s + si) * s + sj) * ld_dx + c] = v;
      acc = __fadd_rn(acc, v);
    }
    dbias[((long long)c * s + si) * s + sj] = acc;
  }
}

}  // namespace

extern "C" int pg_gelu_cast(const float* x, int64_t ld_x, int P, int C, int width, void* g, void* d, int64_t ld_out,
                            void* stream_) {
  PG_REQUIRE(x && g && d, "pg_gelu_cast: null argument");
  PG_REQUIRE(P >= 0 && C >= 0 && width >= C && ld_x >= C && ld_out >= width,
             "pg_gelu_cast: P = %d, C = %d, width = %d (>= C), ld_x = %lld (>= C), ld_out = %lld (>= width)", P, C,
             width, (long long)ld_x, (long long)ld_out);
  const long long total = (long long)P * width;
  if (total == 0) return 0;
  gelu_cast_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      x, ld_x, P, C, width, (bf16*)g, (bf16*)d, ld_out);
  return pg_check_launch("pg_gelu_cast");
}

extern "C" int pg_vd_latent_fwd(const float* prior, int64_t ld_prior, const float* post, int64_t ld_post,
                                const float* x, int64_t ld_x, const float* eps, int n, int L, int C, int hw, void* z,
                                int64_t ld_z, float* s, int64_t ld_s, const float* kl_in, float* kl_out,
                                void* stream_) {
  PG_REQUIRE(prior && x && eps && z && s && (!post || kl_out), "pg_vd_latent_fwd: null argument");
  PG_REQUIRE(n >= 0 && L >= 1 && C >= 1 && hw >= 1, "pg_vd_latent_fwd: n = %d, L = %d, C = %d, hw = %d", n, L, C, hw);
  PG_REQUIRE(ld_prior >= 2 * L + C && (!post || ld_post >= 2 * L) && ld_x >= C && ld_s >= C && ld_z >= L,
             "pg_vd_latent_fwd: pitches ld_prior = %lld (>= 2L + C), ld_post = %lld (>= 2L), ld_x = %lld, ld_s = %lld "
             "(>= C), ld_z = %lld (>= L) for L = %d, C = %d", (long long)ld_prior, (long long)ld_post, (long long)ld_x,
             (long long)ld_s, (long long)ld_z, L, C);
  if (n == 0) return 0;
  vd_latent_fwd_kernel<<<n, THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      prior, ld_prior, post, ld_post, x, ld_x, eps, L, C, hw, (bf16*)z, ld_z, s, ld_s, kl_in, kl_out);
  return pg_check_launch("pg_vd_latent_fwd");
}

extern "C" int pg_vd_latent_bwd(const float* prior, int64_t ld_prior, const float* post, int64_t ld_post,
                                const float* eps, const void* dz, int64_t ld_dz, const float* g_kl, const float* dsum,
                                int64_t ld_dsum, int n, int L, int C, int hw, void* dprior, int64_t ld_dprior,
                                void* dpost, int64_t ld_dpost, void* stream_) {
  PG_REQUIRE(prior && eps && dsum && dprior && (!post == !dpost), "pg_vd_latent_bwd: null argument");
  PG_REQUIRE(n >= 0 && L >= 1 && C >= 1 && hw >= 1, "pg_vd_latent_bwd: n = %d, L = %d, C = %d, hw = %d", n, L, C, hw);
  PG_REQUIRE(ld_prior >= 2 * L + C && (!post || ld_post >= 2 * L) && (!dz || ld_dz >= L) && ld_dsum >= C &&
                 ld_dprior >= 2 * L + C && (!dpost || ld_dpost >= 2 * L),
             "pg_vd_latent_bwd: pitches ld_prior = %lld, ld_post = %lld, ld_dz = %lld, ld_dsum = %lld, ld_dprior = %lld, "
             "ld_dpost = %lld for L = %d, C = %d", (long long)ld_prior, (long long)ld_post, (long long)ld_dz,
             (long long)ld_dsum, (long long)ld_dprior, (long long)ld_dpost, L, C);
  const long long total = (long long)n * hw * (ld_dprior > ld_dpost ? ld_dprior : ld_dpost);
  if (total == 0) return 0;
  vd_latent_bwd_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      prior, ld_prior, post, ld_post, eps, (const bf16*)dz, ld_dz, g_kl, dsum, ld_dsum, n, L, C, hw, (bf16*)dprior,
      ld_dprior, (bf16*)dpost, dpost ? ld_dpost : 0);
  return pg_check_launch("pg_vd_latent_bwd");
}

extern "C" int pg_avg_pool2_fwd(const float* x, int64_t ld_x, int n, int h, int w, int C, float* y, int64_t ld_y,
                                void* stream_) {
  PG_REQUIRE(x && y, "pg_avg_pool2_fwd: null argument");
  PG_REQUIRE(n >= 0 && h >= 2 && w >= 2 && C >= 1 && ld_x >= C && ld_y >= C,
             "pg_avg_pool2_fwd: n = %d, h = %d, w = %d (>= 2), C = %d, ld_x = %lld, ld_y = %lld (>= C)", n, h, w, C,
             (long long)ld_x, (long long)ld_y);
  const long long total = (long long)n * (h / 2) * (w / 2) * C;
  if (total == 0) return 0;
  avg_pool2_fwd_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(x, ld_x, n, h, w, C,
                                                                                               y, ld_y);
  return pg_check_launch("pg_avg_pool2_fwd");
}

extern "C" int pg_avg_pool2_bwd(const float* dy, int64_t ld_dy, int n, int h, int w, int C, float* dx, int64_t ld_dx,
                                void* stream_) {
  PG_REQUIRE(dy && dx, "pg_avg_pool2_bwd: null argument");
  PG_REQUIRE(n >= 0 && h >= 2 && w >= 2 && C >= 1 && ld_dy >= C && ld_dx >= C,
             "pg_avg_pool2_bwd: n = %d, h = %d, w = %d (>= 2), C = %d, ld_dy = %lld, ld_dx = %lld (>= C)", n, h, w, C,
             (long long)ld_dy, (long long)ld_dx);
  const long long total = (long long)n * h * w * C;
  if (total == 0) return 0;
  avg_pool2_bwd_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(dy, ld_dy, n, h, w, C,
                                                                                               dx, ld_dx);
  return pg_check_launch("pg_avg_pool2_bwd");
}

extern "C" int pg_bias_unpool_fwd(const float* x, int64_t ld_x, const float* bias, int n, int s, int C, int f, float* y,
                                  int64_t ld_y, void* stream_) {
  PG_REQUIRE(bias && y, "pg_bias_unpool_fwd: null argument");
  PG_REQUIRE(n >= 0 && s >= 1 && C >= 1 && (f == 1 || f == 2) && (!x || ld_x >= C) && ld_y >= C,
             "pg_bias_unpool_fwd: n = %d, s = %d, C = %d, f = %d (1 or 2), ld_x = %lld, ld_y = %lld (>= C)", n, s, C, f,
             (long long)ld_x, (long long)ld_y);
  const long long total = (long long)n * s * s * f * f * C;
  if (total == 0) return 0;
  bias_unpool_fwd_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(x, ld_x, bias, n, s,
                                                                                                 C, f, y, ld_y);
  return pg_check_launch("pg_bias_unpool_fwd");
}

extern "C" int pg_bias_unpool_bwd(const float* dy, int64_t ld_dy, int n, int s, int C, int f, float* dx, int64_t ld_dx,
                                  float* dbias, void* stream_) {
  PG_REQUIRE(dy && dbias, "pg_bias_unpool_bwd: null argument");
  PG_REQUIRE(n >= 0 && s >= 1 && C >= 1 && (f == 1 || f == 2) && ld_dy >= C && (!dx || ld_dx >= C),
             "pg_bias_unpool_bwd: n = %d, s = %d, C = %d, f = %d (1 or 2), ld_dy = %lld, ld_dx = %lld (>= C)", n, s, C,
             f, (long long)ld_dy, (long long)ld_dx);
  const long long total = (long long)s * s * C;
  bias_unpool_bwd_kernel<<<grid_for(total), THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(dy, ld_dy, n, s, C,
                                                                                                 f, dx, ld_dx, dbias);
  return pg_check_launch("pg_bias_unpool_bwd");
}
