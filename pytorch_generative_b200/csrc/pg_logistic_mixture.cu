// pg_logistic_mixture.cu — the discretised logistic mixture likelihood of 8-bit images (PixelCNN++'s DMOL): a fused
// NLL forward and backward over NCHW parameters, and the per-pixel mixture draw of the samplers.
//
// Layout (losses.py owns the convention): an image of C channels has M * G parameter channels, G = (C + 1)(C + 2) / 2,
// T = C (C - 1) / 2, viewed as [N, M * G, HW]:
//   mixture logit pi_m at channel m, mean mu_{m,c} at M + m C + c, raw log-scale ls_{m,c} at M + M C + m C + c, raw
//   coupling coefficient r_{m,t} at M + 2 M C + m T + t, t = c (c - 1) / 2 + j for j < c.
// Bin of x: k = target_class(x, K), centre x' = 2k / (K - 1) - 1, half-width h = 1 / (K - 1).  Per component and
// channel: log_s = max(ls, -7), mu' = mu + sum_{j<c} tanh(r) x'_j, inv = exp(-log_s), a = inv (x' - mu' + h),
// b = inv (x' - mu' - h), D = inv 2h (= a - b), and the exact log-mass of the bin:
//   bin 0: -softplus(-a);  bin K - 1: -softplus(b);  otherwise -softplus(-a) - softplus(b) + log(-expm1(-D)).
// Per-pixel NLL = logsumexp_m(pi) - logsumexp_m(pi_m + sum_c lp_{m,c}).  Components are walked in ascending m, channels
// in ascending c; the per-image sums are block partials added in block order by pg_sum_partials: no atomics, every
// run gives the same bits.
#include "pg_common.cuh"

namespace {

constexpr int THREADS = 128;  // one thread per (image, pixel); 64 x 1024 pixels fill 512 blocks

// x'_k = 2k h - 1 with h = fl(1 / (K - 1)): within 3 u of 2k / (K - 1) - 1, and no division in the loops.
__device__ __forceinline__ float bin_centre(int k, float h) { return fmaf((float)(2 * k), h, -1.f); }

__device__ __forceinline__ float softplus(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }

// The divisions below have divisors in [1, 4] (or, in d_log_mass, in [2^-100, 2^126] or past it, where the quotient is
// below 2^-36 and 0 is within the bound): __fdividef's range, where it is within 2 ulp.  IEEE division would add an
// out-of-line slow path whose register saves spill.

// 1 / (1 + e^-z) without overflow, and relatively accurate in both tails.
__device__ __forceinline__ float sigmoid(float z) {
  if (z >= 0.f) return __fdividef(1.f, 1.f + expf(-z));
  const float e = expf(z);
  return __fdividef(e, 1.f + e);
}

// 1 - tanh(r)^2 as sech(r)^2 = 4 e / (1 + e)^2 with e = exp(-2|r|): relatively accurate where tanh(r) rounds to +-1.
__device__ __forceinline__ float sech2(float r) {
  const float e = expf(-2.f * fabsf(r));
  const float d = 1.f + e;
  return __fdividef(4.f * e, d * d);
}

// D / expm1(D), the derivative of log(-expm1(-D)) by log D, for D > 0; 1 where D is too small for __fdividef.
__device__ __forceinline__ float d_log_mass(float D) { return D < 0x1p-100f ? 1.f : __fdividef(D, expm1f(D)); }

// One component's term for one channel: the bin's log-mass lp and its derivatives by mu' (dmu) and by log_s (dls).
struct Bin {
  float lp, dmu, dls;
};

__device__ __forceinline__ Bin bin_terms(float xc, float mup, float log_s, float h2, float h, bool lo, bool hi,
                                         bool grads) {
  const float inv = expf(-log_s);
  const float d = xc - mup;
  const float a = inv * (d + h), b = inv * (d - h);
  Bin t;
  if (lo && hi) {
    const float D = inv * h2;
    t.lp = (-softplus(-a) - softplus(b)) + logf(-expm1f(-D));
    if (grads) {
      const float sa = sigmoid(-a), sb = sigmoid(b);
      t.dmu = -inv * (sa - sb);
      t.dls = (-a * sa + b * sb) - d_log_mass(D);
    }
  } else if (hi) {  // bin 0: everything below its upper edge
    t.lp = -softplus(-a);
    if (grads) {
      const float sa = sigmoid(-a);
      t.dmu = -inv * sa;
      t.dls = -a * sa;
    }
  } else {  // bin K - 1: everything above its lower edge
    t.lp = -softplus(b);
    if (grads) {
      const float sb = sigmoid(b);
      t.dmu = inv * sb;
      t.dls = b * sb;
    }
  }
  return t;
}

// Bin centres of one pixel's channels: in registers when C is a template constant, re-read from x otherwise.
template <int CT>
struct Centres {
  float v[CT];
  __device__ __forceinline__ float operator()(int j) const { return v[j]; }
};
template <>
struct Centres<0> {
  const float* x;
  long long HW;
  int K;
  float h;
  __device__ __forceinline__ float operator()(int j) const { return bin_centre(target_class(x[j * HW], K), h); }
};

// Thread (n, p): parameter channel q of it is at preds[(n M G + q) HW + p], so a warp's loads are consecutive addresses
// for every q.  Pass 1 reads the parameters for the NLL; pass 2 reads them again for d loss / d preds.
template <int CT>
__global__ void __launch_bounds__(THREADS)
logistic_mixture_kernel(const float* __restrict__ preds, const float* __restrict__ x, int M, int Cr, int K, long long HW,
                        float grad_scale, float* __restrict__ nll, float* __restrict__ part, int n_img,
                        float* __restrict__ dpreds) {
  __shared__ float red[THREADS / 32];
  const int C = CT > 0 ? CT : Cr;
  const int T = C * (C - 1) / 2;
  const int n = blockIdx.y;
  const long long p = (long long)blockIdx.x * THREADS + threadIdx.x;
  float loss = 0.f;
  if (p < HW) {
    const long long G = (long long)(C + 1) * (C + 2) / 2;
    const float* P = preds + (long long)n * M * G * HW + p;
    const float* xp = x + (long long)n * C * HW + p;
    const float* pmu = P + (long long)M * HW;
    const float* pls = pmu + (long long)M * C * HW;
    const float* pr = pls + (long long)M * C * HW;
    const float h = 1.f / (float)(K - 1), h2 = 2.f / (float)(K - 1);
    Centres<CT> xc;
    unsigned lo_mask = 0, hi_mask = 0;  // channel c's bin is not bin 0 / not bin K - 1 (generic C: recomputed)
    if constexpr (CT > 0) {
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        const int k = target_class(xp[c * HW], K);
        xc.v[c] = bin_centre(k, h);
        lo_mask |= (k > 0 ? 1u : 0u) << c;
        hi_mask |= (k < K - 1 ? 1u : 0u) << c;
      }
    } else {
      xc.x = xp;
      xc.HW = HW;
      xc.K = K;
      xc.h = h;
    }
    // bit 0: channel c's bin is not bin 0; bit 1: it is not bin K - 1
    auto edges = [&](int c) -> unsigned {
      if constexpr (CT > 0) {
        return ((lo_mask >> c) & 1u) | (((hi_mask >> c) & 1u) << 1);
      } else {
        const int k = target_class(xp[c * HW], K);
        return (k > 0 ? 1u : 0u) | (k < K - 1 ? 2u : 0u);
      }
    };
    // mu' of component m, channel c: mu plus the coupling to the earlier channels' bin centres, j ascending.
    auto coupled_mean = [&](int m, int c) {
      float mup = pmu[(long long)(m * C + c) * HW];
      const float* r = pr + (long long)(m * T + c * (c - 1) / 2) * HW;
#pragma unroll
      for (int j = 0; j < (CT > 0 ? CT - 1 : C - 1); ++j) {
        if (j >= c) break;
        mup = fmaf(tanhf(r[j * HW]), xc(j), mup);
      }
      return mup;
    };
    // sum_c lp_{m,c}, c ascending
    auto component_logp = [&](int m) {
      float L = 0.f;
#pragma unroll
      for (int c = 0; c < (CT > 0 ? CT : C); ++c) {
        const unsigned e = edges(c);
        const float log_s = fmaxf(pls[(long long)(m * C + c) * HW], -7.f);
        L += bin_terms(xc(c), coupled_mean(m, c), log_s, h2, h, e & 1u, e & 2u, false).lp;
      }
      return L;
    };

    OnlineLse lse_pi, lse_z;
    for (int m = 0; m < M; ++m) {
      const float pi = P[(long long)m * HW];
      lse_pi.add(pi);
      lse_z.add(pi + component_logp(m));
    }
    loss = (lse_pi.m - lse_z.m) + (logf(lse_pi.s) - logf(lse_z.s));
    if (nll) nll[(long long)n * HW + p] = loss;

    if (dpreds) {
      float* dP = dpreds + (long long)n * M * G * HW + p;
      float* dmu = dP + (long long)M * HW;
      float* dls = dmu + (long long)M * C * HW;
      float* dr = dls + (long long)M * C * HW;
      const float inv_s_pi = 1.f / lse_pi.s, inv_s_z = 1.f / lse_z.s;
      for (int m = 0; m < M; ++m) {
        const float pi = P[(long long)m * HW];
        const float soft = expf(pi - lse_pi.m) * inv_s_pi;               // softmax(pi)_m
        const float w = expf((pi + component_logp(m)) - lse_z.m) * inv_s_z;  // responsibility of component m
        dP[(long long)m * HW] = (soft - w) * grad_scale;
        const float ws = w * grad_scale;
#pragma unroll
        for (int c = 0; c < (CT > 0 ? CT : C); ++c) {
          const unsigned e = edges(c);
          const long long q = (long long)(m * C + c) * HW;
          const float ls = pls[q];
          const Bin t = bin_terms(xc(c), coupled_mean(m, c), fmaxf(ls, -7.f), h2, h, e & 1u, e & 2u, true);
          const float gmu = -(ws * t.dmu);
          dmu[q] = gmu;
          dls[q] = ls >= -7.f ? -(ws * t.dls) : 0.f;
          const long long rq = (long long)(m * T + c * (c - 1) / 2) * HW;
#pragma unroll
          for (int j = 0; j < (CT > 0 ? CT - 1 : C - 1); ++j) {
            if (j >= c) break;
            dr[rq + j * HW] = gmu * sech2(pr[rq + j * HW]) * xc(j);
          }
        }
      }
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

// Thread r: parameter q of row r is preds[r ld + q].  The component is the first m whose ascending cumulative sum of
// exp(pi - max) reaches u[r, 0] * sum (pg_categorical_sample's rule); then, for c ascending, the continuous draw
// v = mu' + exp(log_s) (log u - log1p(-u)) with u = u[r, 1 + c], coupled to the bin centres already drawn, is rounded to
// its bin: k = rint(clamp((v + 1) / 2, 0, 1) (K - 1)), out[r, c] = k / (K - 1).  Each bin then has exactly the mass the
// loss gives it: the tails beyond the end bins' outer edges round to the end bins.
__global__ void __launch_bounds__(THREADS)
logistic_mixture_sample_kernel(const float* __restrict__ preds, long long ld, int rows, int M, int C, int K,
                               const float* __restrict__ u, float* __restrict__ out) {
  const long long r = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (r >= rows) return;
  const float* P = preds + r * ld;
  const float* ur = u + r * (1 + C);
  float* o = out + r * C;
  float mx = -INFINITY;
  for (int m = 0; m < M; ++m) mx = fmaxf(mx, P[m]);
  float s = 0.f;
  for (int m = 0; m < M; ++m) s += expf(P[m] - mx);
  const float target = ur[0] * s;
  float cum = 0.f;
  int pick = M - 1;  // NaN logits: no comparison holds
  for (int m = 0; m < M; ++m) {
    cum += expf(P[m] - mx);
    if (cum >= target) {
      pick = m;
      break;
    }
  }
  const int T = C * (C - 1) / 2;
  const float* mu = P + M + pick * C;
  const float* ls = P + M + M * C + pick * C;
  const float* rr = P + M + 2 * M * C + pick * T;
  const float h = 1.f / (float)(K - 1);
  for (int c = 0; c < C; ++c) {
    float mup = mu[c];
    for (int j = 0; j < c; ++j)
      mup = fmaf(tanhf(rr[c * (c - 1) / 2 + j]), bin_centre(target_class(o[j], K), h), mup);
    const float uc = ur[1 + c];
    const float v = mup + expf(fmaxf(ls[c], -7.f)) * (logf(uc) - log1pf(-uc));
    const int k = target_class(0.5f * (v + 1.f), K);
    o[c] = (float)k / (float)(K - 1);
  }
}

template <int CT>
void launch_loss(dim3 grid, cudaStream_t stream, const float* preds, const float* x, int M, int C, int K, long long HW,
                 float grad_scale, float* nll, float* part, int N, float* dpreds) {
  logistic_mixture_kernel<CT><<<grid, THREADS, 0, stream>>>(preds, x, M, C, K, HW, grad_scale, nll, part, N, dpreds);
}

}  // namespace

extern "C" int pg_logistic_mixture_fwd_bwd(const float* preds, const float* x, int N, int M, int C, int K, int64_t HW,
                                           float grad_scale, float* nll, float* image_nll, float* dpreds,
                                           void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(N >= 1 && M >= 1 && C >= 1 && K >= 2 && HW >= 1,
             "pg_logistic_mixture_fwd_bwd: bad shape (N %d, M %d, C %d, K %d, HW %lld)", N, M, C, K, (long long)HW);
  PG_REQUIRE(N <= 65535, "pg_logistic_mixture_fwd_bwd: %d images (at most 65535 per call)", N);
  PG_REQUIRE(K <= (1 << 23), "pg_logistic_mixture_fwd_bwd: %d bins (at most 2^23)", K);
  PG_REQUIRE(preds && x, "pg_logistic_mixture_fwd_bwd: null argument");
  const long long blocks = (HW + THREADS - 1) / THREADS;
  PG_REQUIRE(blocks < (1LL << 31), "pg_logistic_mixture_fwd_bwd: %lld pixels per image is too many", (long long)HW);
  float* part = nullptr;
  if (image_nll && pg_scratch((size_t)blocks * N * sizeof(float), stream, &part)) return 1;
  const dim3 grid((unsigned)blocks, N);
  if (C == 1)
    launch_loss<1>(grid, stream, preds, x, M, C, K, HW, grad_scale, nll, part, N, dpreds);
  else if (C == 3)
    launch_loss<3>(grid, stream, preds, x, M, C, K, HW, grad_scale, nll, part, N, dpreds);
  else
    launch_loss<0>(grid, stream, preds, x, M, C, K, HW, grad_scale, nll, part, N, dpreds);
  if (pg_check_launch("pg_logistic_mixture_fwd_bwd")) return 1;
  return image_nll ? pg_sum_partials(part, (int)blocks, N, 1, N, N, image_nll, stream) : 0;
}

extern "C" int pg_logistic_mixture_sample(const float* preds, int64_t ld, int rows, int M, int C, int K, const float* u,
                                          float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(rows >= 0 && M >= 1 && C >= 1 && K >= 2, "pg_logistic_mixture_sample: bad shape (rows %d, M %d, C %d, K %d)",
             rows, M, C, K);
  PG_REQUIRE(K <= (1 << 23), "pg_logistic_mixture_sample: %d bins (at most 2^23)", K);
  const long long G = (long long)(C + 1) * (C + 2) / 2;
  PG_REQUIRE(ld >= (int64_t)M * G, "pg_logistic_mixture_sample: pitch %lld narrower than M * G = %lld", (long long)ld,
             (long long)M * G);
  if (rows == 0) return 0;
  PG_REQUIRE(preds && u && out, "pg_logistic_mixture_sample: null argument");
  logistic_mixture_sample_kernel<<<(unsigned)((rows + THREADS - 1) / THREADS), THREADS, 0, stream>>>(preds, ld, rows, M, C,
                                                                                                    K, u, out);
  return pg_check_launch("pg_logistic_mixture_sample");
}
