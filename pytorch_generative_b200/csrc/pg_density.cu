// pg_density.cu — KernelDensityEstimator and the mixture models (reference models/kde.py, models/mixture_models.py).
// Every kernel here pairs a query row (a test point, or a batch row) with a codebook row (a training point, or a mixture
// component), reduces over the D features in fp32 on the CUDA cores and then takes a logsumexp or a count over the
// codebook rows.  The [N, M, D] broadcast of the reference is never formed: a CTA owns a 64 x 64 tile of pairs, streams
// D through shared memory in chunks of 32 and keeps one 4 x 4 register block of pair sums per thread.  Splits (over the
// codebook rows, over D or over the batch) write partials to the library scratch, which later launches add in split
// order.  Grids depend on the shape and the SM count only and there are no atomics: every run is bit-identical.
#include <math.h>
#include <string.h>

#include "pg_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int TR = 64;         // query rows per tile
constexpr int TC = 64;         // codebook rows per tile
constexpr int DK = 32;         // features per shared-memory chunk
constexpr int PITCH = 68;      // row pitch of a staged chunk: float4-aligned, 68 / 4 odd
constexpr int MAX_SPLITS = 32;    // codebook splits of the KDE forward and the Parzen count ([splits, N] partials)
constexpr int BWD_SPLITS = 8;     // codebook splits of the KDE backward ([splits, N, D] partials)
constexpr int FEATURE_SPLITS = 8; // feature splits of the mixture forward
constexpr float NEG_INF = -INFINITY;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float at(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// dst[c][r] = src[(row0 + r) * D + d0 + c] for r < 64, c < DK (zero outside [rows) x [d_end)): a chunk of 64 rows, transposed so
// that a thread reads four consecutive rows of one feature as a float4.
__device__ __forceinline__ void stage_rows(float (*dst)[PITCH], const float* __restrict__ src, int rows, int row0, int D,
                                           int d0, int d_end) {
#pragma unroll
  for (int q = 0; q < TR * DK / THREADS; ++q) {
    const int e = threadIdx.x + q * THREADS;
    const int r = e / DK, c = e % DK;
    const int gr = row0 + r, gd = d0 + c;
    dst[c][r] = (gr < rows && gd < d_end) ? src[(long long)gr * D + gd] : 0.f;
  }
}

// Online logsumexp state: m the running maximum, l the sum of exp(s - m).  -inf terms contribute nothing.
__device__ __forceinline__ void lse_push(float& m, float& l, float s) {
  if (s > m) {
    l = (m == NEG_INF ? 0.f : l * expf(m - s)) + 1.f;
    m = s;
  } else if (s > NEG_INF) {
    l += expf(s - m);
  }
}
// (m, l) <- (m, l) + (m2, l2); the sum of the two rescaled terms is commutative, so both lanes of a butterfly agree.
__device__ __forceinline__ void lse_merge(float& m, float& l, float m2, float l2) {
  const float mx = fmaxf(m, m2);
  if (mx == NEG_INF) return;
  const float a = m == NEG_INF ? 0.f : l * expf(m - mx);
  const float b = m2 == NEG_INF ? 0.f : l2 * expf(m2 - mx);
  m = mx;
  l = a + b;
}

// Sum of (x - t)^2 over all D for the thread's 4 x 4 block of pairs (rows ty*4 + i of the query tile, columns tx*4 + j
// of the codebook tile), one fmaf chain per pair in ascending feature order.
__device__ __forceinline__ void pair_sqdist(float (*xs)[PITCH], float (*ts)[PITCH], const float* __restrict__ x, int N,
                                            int n0, const float* __restrict__ t, int M, int m0, int D, float acc[4][4]) {
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int d0 = 0; d0 < D; d0 += DK) {
    __syncthreads();
    stage_rows(xs, x, N, n0, D, d0, D);
    stage_rows(ts, t, M, m0, D, d0, D);
    __syncthreads();
#pragma unroll 8
    for (int d = 0; d < DK; ++d) {
      const float4 xv = ld4(&xs[d][ty * 4]), tv = ld4(&ts[d][tx * 4]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float df = at(xv, i) - at(tv, j);
          acc[i][j] = fmaf(df, df, acc[i][j]);
        }
    }
  }
}

// Splits of the codebook rows: up to `cap` splits of whole tiles.  Decided by M alone, so a query row's result does not
// depend on the batch it came in (a sub-batch gives the same bits); many query tiles simply make more CTAs.
void codebook_splits(int M, int cap, int* splits, int* tiles_per_split) {
  const int m_tiles = (M + TC - 1) / TC;
  const int s = m_tiles < cap ? m_tiles : cap;
  *tiles_per_split = (m_tiles + s - 1) / s;
  *splits = (m_tiles + *tiles_per_split - 1) / *tiles_per_split;
}

// ---- Gaussian KDE --------------------------------------------------------------------------------------------------
// CTA (query tile, split): s_nm = scale * |x_n - t_m|^2 with scale = -0.5 / h^2; per query row the online (max, sum) over
// the split's training rows.  Each thread keeps its own state for its 4 rows over its columns; the 16 threads of a row
// merge theirs by a fixed butterfly.  part[(split * N + n) * 2 + {0, 1}] = (max, sum).
__global__ void __launch_bounds__(THREADS) kde_gauss_fwd_kernel(const float* __restrict__ x, int N,
                                                               const float* __restrict__ t, int M, int D, float scale,
                                                               int tiles_per_split, float* __restrict__ part) {
  __shared__ __align__(16) float xs[DK][PITCH];
  __shared__ __align__(16) float ts[DK][PITCH];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int n0 = blockIdx.x * TR, split = blockIdx.y;
  const int m_begin = split * tiles_per_split * TC, m_end = min(M, m_begin + tiles_per_split * TC);
  float mx[4], sm[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) mx[i] = NEG_INF, sm[i] = 0.f;
  for (int m0 = m_begin; m0 < m_end; m0 += TC) {
    float acc[4][4];
    pair_sqdist(xs, ts, x, N, n0, t, M, m0, D, acc);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (m0 + tx * 4 + j < m_end)
#pragma unroll
        for (int i = 0; i < 4; ++i) lse_push(mx[i], sm[i], scale * acc[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, mx[i], off), l2 = __shfl_xor_sync(0xffffffffu, sm[i], off);
      lse_merge(mx[i], sm[i], m2, l2);
    }
    const int n = n0 + ty * 4 + i;
    if (tx == 0 && n < N) {
      part[((long long)split * N + n) * 2] = mx[i];
      part[((long long)split * N + n) * 2 + 1] = sm[i];
    }
  }
}

// Per query row: the splits' (max, sum) merged in split order, each sum rescaled by exp(m_s - max).
__global__ void __launch_bounds__(THREADS) kde_lse_merge_kernel(const float* __restrict__ part, int splits, int N, float Z,
                                                               float* __restrict__ lse, float* __restrict__ out) {
  for (int n = blockIdx.x * THREADS + threadIdx.x; n < N; n += gridDim.x * THREADS) {
    float m = NEG_INF;
    for (int s = 0; s < splits; ++s) m = fmaxf(m, part[((long long)s * N + n) * 2]);
    float l = 0.f;
    if (m > NEG_INF)
      for (int s = 0; s < splits; ++s) {
        const float ms = part[((long long)s * N + n) * 2];
        if (ms > NEG_INF) l += part[((long long)s * N + n) * 2 + 1] * expf(ms - m);
      }
    const float v = m > NEG_INF ? m + logf(l) : NEG_INF;
    if (lse) lse[n] = v;
    out[n] = v - Z;
  }
}

// CTA (query tile, split): for each training tile, the pair sums over all of D first (as the forward), then
// w_nm = c_n exp(s_nm - lse_n) with c_n = -g_n / h^2 into shared memory, then the training tile's D-chunks again:
// part[split][n][d] (+)= sum_m w_nm (x_nd - t_md), one fmaf chain per output in ascending m.
__global__ void __launch_bounds__(THREADS) kde_gauss_bwd_kernel(const float* __restrict__ x, int N,
                                                               const float* __restrict__ t, int M, int D, float scale,
                                                               float neg_inv_h2, const float* __restrict__ lse,
                                                               const float* __restrict__ g, int tiles_per_split,
                                                               float* __restrict__ part) {
  __shared__ __align__(16) float xs[DK][PITCH];
  __shared__ __align__(16) float ts[DK][PITCH];
  __shared__ __align__(16) float ws[TC][PITCH];  // ws[m][n]
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int n0 = blockIdx.x * TR, split = blockIdx.y;
  const int m_begin = split * tiles_per_split * TC, m_end = min(M, m_begin + tiles_per_split * TC);
  float c[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + ty * 4 + i;
    c[i] = n < N ? g[n] * neg_inv_h2 : 0.f;
    l[i] = n < N ? lse[n] : 0.f;
  }
  float* out = part + (long long)split * N * D;
  // phase-2 mapping: rows ty * 4 + i, features tx and tx + 16 of each chunk
  for (int m0 = m_begin; m0 < m_end; m0 += TC) {
    float acc[4][4];
    pair_sqdist(xs, ts, x, N, n0, t, M, m0, D, acc);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) w[i] = (m0 + tx * 4 + j < m_end && c[i] != 0.f) ? c[i] * expf(scale * acc[i][j] - l[i]) : 0.f;
      *reinterpret_cast<float4*>(&ws[tx * 4 + j][ty * 4]) = make_float4(w[0], w[1], w[2], w[3]);
    }
    const bool first = m0 == m_begin;
    for (int d0 = 0; d0 < D; d0 += DK) {
      __syncthreads();
      stage_rows(xs, x, N, n0, D, d0, D);
      stage_rows(ts, t, M, m0, D, d0, D);
      __syncthreads();
      float o[4][2];
      float xv[4][2];
#pragma unroll
      for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i][e] = 0.f, xv[i][e] = xs[tx + 16 * e][ty * 4 + i];
#pragma unroll 8
      for (int m = 0; m < TC; ++m) {
        const float4 wv = ld4(&ws[m][ty * 4]);
        const float t0 = ts[tx][m], t1 = ts[tx + 16][m];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          o[i][0] = fmaf(at(wv, i), xv[i][0] - t0, o[i][0]);
          o[i][1] = fmaf(at(wv, i), xv[i][1] - t1, o[i][1]);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= N) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int d = d0 + tx + 16 * e;
          if (d < D) {
            float* p = out + (long long)n * D + d;
            *p = first ? o[i][e] : *p + o[i][e];
          }
        }
      }
    }
  }
}

// ---- Parzen window -------------------------------------------------------------------------------------------------
// CTA (query tile, split): per pair, whether every |x_d - t_d| <= a_max (a_max: the largest fp32 whose IEEE quotient by h
// rounds to <= 0.5, so the test equals fl(|x_d - t_d| / h) <= 0.5; NaN is outside); per query row the count of inside
// pairs over the split's training rows, as an exact float in part[split * N + n].
__global__ void __launch_bounds__(THREADS) kde_parzen_kernel(const float* __restrict__ x, int N,
                                                            const float* __restrict__ t, int M, int D, float a_max,
                                                            int tiles_per_split, float* __restrict__ part) {
  __shared__ __align__(16) float xs[DK][PITCH];
  __shared__ __align__(16) float ts[DK][PITCH];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int n0 = blockIdx.x * TR, split = blockIdx.y;
  const int m_begin = split * tiles_per_split * TC, m_end = min(M, m_begin + tiles_per_split * TC);
  int count[4] = {0, 0, 0, 0};
  for (int m0 = m_begin; m0 < m_end; m0 += TC) {
    unsigned outside = 0;  // bit 4 i + j: pair (i, j) has a feature outside the window
    for (int d0 = 0; d0 < D; d0 += DK) {
      __syncthreads();
      stage_rows(xs, x, N, n0, D, d0, D);
      stage_rows(ts, t, M, m0, D, d0, D);
      __syncthreads();
#pragma unroll 8
      for (int d = 0; d < DK; ++d) {
        const float4 xv = ld4(&xs[d][ty * 4]), tv = ld4(&ts[d][tx * 4]);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (!(fabsf(at(xv, i) - at(tv, j)) <= a_max)) outside |= 1u << (4 * i + j);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (m0 + tx * 4 + j < m_end)
#pragma unroll
        for (int i = 0; i < 4; ++i) count[i] += !((outside >> (4 * i + j)) & 1u);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) count[i] += __shfl_xor_sync(0xffffffffu, count[i], off);
    const int n = n0 + ty * 4 + i;
    if (tx == 0 && n < N) part[(long long)split * N + n] = (float)count[i];
  }
}

// count = the splits' counts added in split order (exact integers); out = log(count) - log(M) - D log(h) in fp64.
__global__ void __launch_bounds__(THREADS) kde_parzen_merge_kernel(const float* __restrict__ part, int splits, int N,
                                                                  double log_norm, int* __restrict__ count,
                                                                  float* __restrict__ out) {
  for (int n = blockIdx.x * THREADS + threadIdx.x; n < N; n += gridDim.x * THREADS) {
    float c = 0.f;
    for (int s = 0; s < splits; ++s) c += part[(long long)s * N + n];
    if (count) count[n] = (int)c;
    if (out) out[n] = (float)(log((double)c) - log_norm);
  }
}

// ---- mixture models ------------------------------------------------------------------------------------------------
// Staging of a component chunk for the forward: for features d0 .. d0 + DK of components k0 .. k0 + 63,
//   Gaussian:  p0 = mean, p1 = exp(log_std), p2 = -log_std - 0.5 log(2 pi)
//   Bernoulli: p0 = logits, p1 = max(l, 0) + log1p(exp(-|l|))  (the stable BCE without its -l x term), p2 unused
// with terms of zero outside [K, D) (mean 0, std 1, z 0; logits 0, p1 0).
template <int KIND>
__device__ __forceinline__ void stage_components(float (*p0)[PITCH], float (*p1)[PITCH], float (*p2)[PITCH],
                                                 const float* __restrict__ a, const float* __restrict__ b, int K, int k0,
                                                 int D, int d0, int d_end, float half_log_2pi) {
#pragma unroll
  for (int q = 0; q < TC * DK / THREADS; ++q) {
    const int e = threadIdx.x + q * THREADS;
    const int r = e / DK, c = e % DK;
    const int k = k0 + r, d = d0 + c;
    const bool ok = k < K && d < d_end;
    const long long i = (long long)k * D + d;
    if (KIND == PG_MIXTURE_GAUSSIAN) {
      const float ls = ok ? b[i] : 0.f;
      p0[c][r] = ok ? a[i] : 0.f;
      p1[c][r] = expf(ls);
      p2[c][r] = ok ? -ls - half_log_2pi : 0.f;
    } else {
      const float l = ok ? a[i] : 0.f;
      p0[c][r] = l;
      p1[c][r] = ok ? fmaxf(l, 0.f) + log1pf(expf(-fabsf(l))) : 0.f;
    }
  }
}

// CTA (batch tile, component tile, feature split): part[(split * N + n) * K + k] = sum over the split's features of
// term(x_nd; k, d), one chain per pair in ascending d.  Gaussian term: z - 0.5 ((x - mean) / std)^2 with the IEEE
// division; Bernoulli term: l x - (max(l, 0) + log1p(exp(-|l|))).
template <int KIND>
__global__ void __launch_bounds__(THREADS) mixture_fwd_kernel(const float* __restrict__ x, int N, int D, int K,
                                                             const float* __restrict__ pa, const float* __restrict__ pb,
                                                             float half_log_2pi, int d_per_split,
                                                             float* __restrict__ part) {
  __shared__ __align__(16) float xs[DK][PITCH];
  __shared__ __align__(16) float p0[DK][PITCH];
  __shared__ __align__(16) float p1[DK][PITCH];
  __shared__ __align__(16) float p2[KIND == PG_MIXTURE_GAUSSIAN ? DK : 1][PITCH];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int n0 = blockIdx.x * TR, k0 = blockIdx.y * TC, split = blockIdx.z;
  const int d_begin = split * d_per_split, d_end = min(D, d_begin + d_per_split);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int d0 = d_begin; d0 < d_end; d0 += DK) {
    __syncthreads();
    stage_rows(xs, x, N, n0, D, d0, d_end);  // features beyond the split read as zero, and their terms are zero
    stage_components<KIND>(p0, p1, p2, pa, pb, K, k0, D, d0, d_end, half_log_2pi);
    __syncthreads();
#pragma unroll 4
    for (int d = 0; d < DK; ++d) {
      const float4 xv = ld4(&xs[d][ty * 4]);
      const float4 av = ld4(&p0[d][tx * 4]), bv = ld4(&p1[d][tx * 4]);
      if (KIND == PG_MIXTURE_GAUSSIAN) {
        const float4 zv = ld4(&p2[d][tx * 4]);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float q = __fdiv_rn(at(xv, i) - at(av, j), at(bv, j));
            acc[i][j] += at(zv, j) - 0.5f * (q * q);
          }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += fmaf(at(av, j), at(xv, i), -at(bv, j));
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + ty * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx * 4 + j;
      if (k < K) part[((long long)split * N + n) * K + k] = acc[i][j];
    }
  }
}

// log_softmax of the mixture logits into lsm (shared, K entries), computed the same way by every CTA: max, then the sum
// of exp(l - max) in ascending k, then l - max - log(sum).
__device__ void mixture_log_softmax(const float* __restrict__ logits, int K, float* lsm, float* sh2) {
  if (threadIdx.x == 0) {
    float mx = NEG_INF;
    for (int k = 0; k < K; ++k) mx = fmaxf(mx, logits[k]);
    float s = 0.f;
    for (int k = 0; k < K; ++k) s += expf(logits[k] - mx);
    sh2[0] = mx;
    sh2[1] = logf(s);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += THREADS) lsm[k] = logits[k] - sh2[0] - sh2[1];
  __syncthreads();
}

// One warp per batch row: a_nk = log_softmax_k + the feature splits' sums in split order; out_n = logsumexp_k a_nk (lane
// l keeps the online state of k = l, l + 32, ..., the lanes merge by a fixed butterfly).
__global__ void __launch_bounds__(THREADS) mixture_lse_kernel(const float* __restrict__ part, int splits, int N, int K,
                                                             const float* __restrict__ logits, float* __restrict__ a,
                                                             float* __restrict__ out) {
  extern __shared__ float lsm[];
  __shared__ float sh2[2];
  mixture_log_softmax(logits, K, lsm, sh2);
  const int lane = threadIdx.x % 32, warps = gridDim.x * (THREADS / 32);
  for (int n = blockIdx.x * (THREADS / 32) + threadIdx.x / 32; n < N; n += warps) {
    float m = NEG_INF, l = 0.f;
    for (int k = lane; k < K; k += 32) {
      float s = 0.f;
      for (int sp = 0; sp < splits; ++sp) s += part[((long long)sp * N + n) * K + k];
      const float v = lsm[k] + s;
      a[(long long)n * K + k] = v;
      lse_push(m, l, v);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
      lse_merge(m, l, m2, l2);
    }
    if (lane == 0) out[n] = m > NEG_INF ? m + logf(l) : NEG_INF;
  }
}

constexpr int NC = 32;  // batch rows (backward) or components (input gradient) per shared-memory chunk

// CTA (component tile, feature tile, batch slice): thread = components ty * 4 + i, features tx * 4 + j.  With
// gr_nk = g_n exp(a_nk - out_n), the slice's sums over its rows in ascending n:
//   Gaussian:  part[k D + d] = sum gr (x - mean) / std^2,  part[K D + k D + d] = sum gr (((x - mean) / std)^2 - 1)
//   Bernoulli: part[k D + d] = sum gr (x - sigmoid(l))
// and, from the CTAs of feature tile 0, part[P K D + k] = sum gr_nk - softmax_k sum g_n (P = 2 or 1 tensors).
template <int KIND>
__global__ void __launch_bounds__(THREADS, 2) mixture_grad_kernel(const float* __restrict__ x, int N, int D, int K,
                                                              const float* __restrict__ pa, const float* __restrict__ pb,
                                                              const float* __restrict__ logits,
                                                              const float* __restrict__ a, const float* __restrict__ out,
                                                              const float* __restrict__ g, int n_per_split,
                                                              long long part_stride, float* __restrict__ part) {
  __shared__ __align__(16) float xs[NC][PITCH];  // xs[n][d]
  __shared__ __align__(16) float gs[NC][PITCH];  // gs[n][k]
  __shared__ float gn[NC];
  __shared__ float sh2[2];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int k0 = blockIdx.x * TC, d0 = blockIdx.y * TC, split = blockIdx.z;
  const int n_begin = split * n_per_split, n_end = min(N, n_begin + n_per_split);
  const bool mix = blockIdx.y == 0;
  constexpr int P = KIND == PG_MIXTURE_GAUSSIAN ? 2 : 1;
  float u[4][4], v[4][4], acc0[4][4], acc1[4][4];  // Gaussian: u = mean, v = 1 / std; Bernoulli: u = sigmoid(l)
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + ty * 4 + i, d = d0 + tx * 4 + j;
      const bool ok = k < K && d < D;
      if (KIND == PG_MIXTURE_GAUSSIAN) {
        u[i][j] = ok ? pa[(long long)k * D + d] : 0.f;
        v[i][j] = ok ? 1.f / expf(pb[(long long)k * D + d]) : 0.f;
      } else {
        u[i][j] = ok ? 1.f / (1.f + expf(-pa[(long long)k * D + d])) : 0.f;
        v[i][j] = 0.f;
      }
      acc0[i][j] = acc1[i][j] = 0.f;
    }
  float kacc = 0.f, gacc = 0.f;  // thread t < 64: sum of gr over the slice for component k0 + t, and of g
  for (int nc = n_begin; nc < n_end; nc += NC) {
    __syncthreads();
#pragma unroll
    for (int q = 0; q < NC * TC / THREADS; ++q) {
      const int e = threadIdx.x + q * THREADS;
      const int r = e / TC, c = e % TC;
      const int n = nc + r, d = d0 + c, k = k0 + c;
      const bool okn = n < n_end;
      xs[r][c] = (okn && d < D) ? x[(long long)n * D + d] : 0.f;
      gs[r][c] = (okn && k < K) ? g[n] * expf(a[(long long)n * K + k] - out[n]) : 0.f;
    }
    if (threadIdx.x < NC) gn[threadIdx.x] = nc + threadIdx.x < n_end ? g[nc + threadIdx.x] : 0.f;
    __syncthreads();
    if (mix && threadIdx.x < TC) {
      for (int r = 0; r < NC; ++r) kacc += gs[r][threadIdx.x], gacc += gn[r];
    }
#pragma unroll 4
    for (int r = 0; r < NC; ++r) {
      const float4 xv = ld4(&xs[r][tx * 4]), gv = ld4(&gs[r][ty * 4]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (KIND == PG_MIXTURE_GAUSSIAN) {
            const float q = (at(xv, j) - u[i][j]) * v[i][j];
            acc0[i][j] = fmaf(at(gv, i), q * v[i][j], acc0[i][j]);
            acc1[i][j] = fmaf(at(gv, i), fmaf(q, q, -1.f), acc1[i][j]);
          } else {
            acc0[i][j] = fmaf(at(gv, i), at(xv, j) - u[i][j], acc0[i][j]);
          }
        }
    }
  }
  float* dst = part + (long long)split * part_stride;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + ty * 4 + i, d = d0 + tx * 4 + j;
      if (k < K && d < D) {
        dst[(long long)k * D + d] = acc0[i][j];
        if (P == 2) dst[(long long)K * D + (long long)k * D + d] = acc1[i][j];
      }
    }
  if (mix) {
    __syncthreads();
    if (threadIdx.x == 0) {  // the softmax's max and log-sum, as mixture_log_softmax computes them
      float mx = NEG_INF;
      for (int k = 0; k < K; ++k) mx = fmaxf(mx, logits[k]);
      float s = 0.f;
      for (int k = 0; k < K; ++k) s += expf(logits[k] - mx);
      sh2[0] = mx;
      sh2[1] = logf(s);
    }
    __syncthreads();
    const int k = k0 + threadIdx.x;
    if (threadIdx.x < TC && k < K)
      dst[(long long)P * K * D + k] = kacc - expf(logits[k] - sh2[0] - sh2[1]) * gacc;
  }
}

// CTA (batch tile, feature tile): dx_nd = sum over k (ascending) of gr_nk * (mean - x) / std^2 (Gaussian) or gr_nk * l
// (Bernoulli); written, not added.
template <int KIND>
__global__ void __launch_bounds__(THREADS) mixture_dx_kernel(const float* __restrict__ x, int N, int D, int K,
                                                            const float* __restrict__ pa, const float* __restrict__ pb,
                                                            const float* __restrict__ a, const float* __restrict__ out,
                                                            const float* __restrict__ g, float* __restrict__ dx) {
  __shared__ __align__(16) float gs[NC][PITCH];  // gs[k][n]
  __shared__ __align__(16) float p0[NC][PITCH];  // p0[k][d]: mean or logits
  __shared__ __align__(16) float p1[KIND == PG_MIXTURE_GAUSSIAN ? NC : 1][PITCH];  // 1 / std^2
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int n0 = blockIdx.x * TR, d0 = blockIdx.y * TC;
  float xv[4][4], acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + ty * 4 + i, d = d0 + tx * 4 + j;
      xv[i][j] = (n < N && d < D) ? x[(long long)n * D + d] : 0.f;
      acc[i][j] = 0.f;
    }
  for (int kc = 0; kc < K; kc += NC) {
    __syncthreads();
#pragma unroll
    for (int q = 0; q < NC * TR / THREADS; ++q) {
      const int e = threadIdx.x + q * THREADS;
      const int r = e / NC, c = e % NC;  // gs: row n0 + r, component kc + c
      const int n = n0 + r, k = kc + c;
      gs[c][r] = (n < N && k < K) ? g[n] * expf(a[(long long)n * K + k] - out[n]) : 0.f;
      const int rk = e / TC, cd = e % TC;  // p0 / p1: component kc + rk, feature d0 + cd
      const int k2 = kc + rk, d = d0 + cd;
      const bool ok = k2 < K && d < D;
      p0[rk][cd] = ok ? pa[(long long)k2 * D + d] : 0.f;
      if (KIND == PG_MIXTURE_GAUSSIAN) {
        const float s = ok ? expf(pb[(long long)k2 * D + d]) : 1.f;
        p1[rk][cd] = 1.f / (s * s);
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < NC; ++k) {
      const float4 gv = ld4(&gs[k][ty * 4]), mv = ld4(&p0[k][tx * 4]);
      if (KIND == PG_MIXTURE_GAUSSIAN) {
        const float4 iv = ld4(&p1[k][tx * 4]);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(at(gv, i), (at(mv, j) - xv[i][j]) * at(iv, j), acc[i][j]);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(at(gv, i), at(mv, j), acc[i][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + ty * 4 + i, d = d0 + tx * 4 + j;
      if (n < N && d < D) dx[(long long)n * D + d] = acc[i][j];
    }
}

unsigned row_grid(long long rows, int per_block) {
  long long blocks = (rows + per_block - 1) / per_block;
  const long long cap = (long long)pg_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks < 1 ? 1 : blocks);
}

// The largest fp32 a >= 0 with fl(a / h) <= 0.5 in IEEE division (round to nearest even).  The quotient is monotone in
// a, so a binary search over the bit patterns of [0, inf] finds it; -1 when no a qualifies.
float parzen_threshold(float h) {
  uint32_t lo = 0, hi = 0x7f800000u;  // the predicate holds at lo = +0 (0 / h = 0) for every h > 0
  auto inside = [h](uint32_t bits) {
    float a;
    memcpy(&a, &bits, sizeof a);
    volatile float q = a / h;
    return q <= 0.5f;
  };
  if (!inside(lo)) return -1.f;
  while (lo < hi) {  // invariant: inside(lo), and everything above hi is outside
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (inside(mid)) lo = mid;
    else hi = mid - 1;
  }
  float a;
  memcpy(&a, &lo, sizeof a);
  return a;
}

int check_rows(const char* who, const float* x, int N, const float* t, int M, int D) {
  PG_REQUIRE(N >= 0 && M >= 1 && D >= 1, "%s: empty problem (N %d, M %d, D %d)", who, N, M, D);
  PG_REQUIRE(N == 0 || (x && t), "%s: null argument", who);
  return 0;
}

}  // namespace

extern "C" int pg_kde_gauss_fwd(const float* x, int N, const float* t, int M, int D, float bandwidth, float Z, float* lse,
                                float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (check_rows("pg_kde_gauss_fwd", x, N, t, M, D)) return 1;
  PG_REQUIRE(bandwidth > 0.f, "pg_kde_gauss_fwd: bandwidth %g is not positive", (double)bandwidth);
  if (N == 0) return 0;
  PG_REQUIRE(out, "pg_kde_gauss_fwd: null output");
  int splits, tps;
  codebook_splits(M, MAX_SPLITS, &splits, &tps);
  float* part = nullptr;
  if (pg_scratch((size_t)splits * N * 2 * sizeof(float), stream, &part)) return 1;
  const float scale = -0.5f / (bandwidth * bandwidth);
  kde_gauss_fwd_kernel<<<dim3((N + TR - 1) / TR, splits), THREADS, 0, stream>>>(x, N, t, M, D, scale, tps, part);
  if (pg_check_launch("pg_kde_gauss_fwd")) return 1;
  kde_lse_merge_kernel<<<row_grid(N, THREADS), THREADS, 0, stream>>>(part, splits, N, Z, lse, out);
  return pg_check_launch("pg_kde_gauss_fwd");
}

extern "C" int pg_kde_gauss_bwd(const float* x, int N, const float* t, int M, int D, float bandwidth, const float* lse,
                                const float* g, float* dx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (check_rows("pg_kde_gauss_bwd", x, N, t, M, D)) return 1;
  PG_REQUIRE(bandwidth > 0.f, "pg_kde_gauss_bwd: bandwidth %g is not positive", (double)bandwidth);
  if (N == 0) return 0;
  PG_REQUIRE(lse && g && dx, "pg_kde_gauss_bwd: null argument");
  int splits, tps;
  codebook_splits(M, BWD_SPLITS, &splits, &tps);
  float* part = nullptr;
  if (pg_scratch((size_t)splits * N * D * sizeof(float), stream, &part)) return 1;
  const float h2 = bandwidth * bandwidth;
  kde_gauss_bwd_kernel<<<dim3((N + TR - 1) / TR, splits), THREADS, 0, stream>>>(x, N, t, M, D, -0.5f / h2, -1.f / h2,
                                                                                 lse, g, tps, part);
  if (pg_check_launch("pg_kde_gauss_bwd")) return 1;
  return pg_sum_partials(part, splits, (long long)N * D, N, D, D, dx, stream);
}

extern "C" int pg_kde_parzen_count(const float* x, int N, const float* t, int M, int D, double bandwidth, int* count,
                                   float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (check_rows("pg_kde_parzen_count", x, N, t, M, D)) return 1;
  PG_REQUIRE(bandwidth > 0.0 && (float)bandwidth > 0.f, "pg_kde_parzen_count: bandwidth %g is not positive", bandwidth);
  PG_REQUIRE(M < (1 << 24), "pg_kde_parzen_count: %d training rows (counts are exact below 2^24)", M);
  if (N == 0) return 0;
  PG_REQUIRE(count || out, "pg_kde_parzen_count: no output");
  int splits, tps;
  codebook_splits(M, MAX_SPLITS, &splits, &tps);
  float* part = nullptr;
  if (pg_scratch((size_t)splits * N * sizeof(float), stream, &part)) return 1;
  kde_parzen_kernel<<<dim3((N + TR - 1) / TR, splits), THREADS, 0, stream>>>(x, N, t, M, D,
                                                                              parzen_threshold((float)bandwidth), tps, part);
  if (pg_check_launch("pg_kde_parzen_count")) return 1;
  const double log_norm = log((double)M) + (double)D * log(bandwidth);
  kde_parzen_merge_kernel<<<row_grid(N, THREADS), THREADS, 0, stream>>>(part, splits, N, log_norm, count, out);
  return pg_check_launch("pg_kde_parzen_count");
}

extern "C" int pg_mixture_fwd(int kind, const float* x, int N, int D, int K, const float* mixture_logits, const float* p0,
                              const float* p1, float* a, float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(kind == PG_MIXTURE_GAUSSIAN || kind == PG_MIXTURE_BERNOULLI, "pg_mixture_fwd: unknown kind %d", kind);
  PG_REQUIRE(N >= 0 && D >= 1 && K >= 1, "pg_mixture_fwd: empty problem (N %d, D %d, K %d)", N, D, K);
  PG_REQUIRE(K <= 8192, "pg_mixture_fwd: %d components (at most 8192)", K);
  if (N == 0) return 0;
  PG_REQUIRE(x && mixture_logits && p0 && (kind == PG_MIXTURE_BERNOULLI || p1) && a && out,
             "pg_mixture_fwd: null argument");
  // feature splits decided by D alone (a sub-batch gives the same bits)
  const int n_tiles = (N + TR - 1) / TR, k_tiles = (K + TC - 1) / TC, d_chunks = (D + DK - 1) / DK;
  const int s = d_chunks < FEATURE_SPLITS ? d_chunks : FEATURE_SPLITS;
  const int chunks_per_split = (d_chunks + s - 1) / s;
  const int splits = (d_chunks + chunks_per_split - 1) / chunks_per_split;
  float* part = nullptr;
  if (pg_scratch((size_t)splits * N * K * sizeof(float), stream, &part)) return 1;
  const float half_log_2pi = 0.5f * logf((float)6.283185307179586);
  const dim3 grid(n_tiles, k_tiles, splits);
  if (kind == PG_MIXTURE_GAUSSIAN)
    mixture_fwd_kernel<PG_MIXTURE_GAUSSIAN><<<grid, THREADS, 0, stream>>>(x, N, D, K, p0, p1, half_log_2pi,
                                                                           chunks_per_split * DK, part);
  else
    mixture_fwd_kernel<PG_MIXTURE_BERNOULLI><<<grid, THREADS, 0, stream>>>(x, N, D, K, p0, p1, half_log_2pi,
                                                                            chunks_per_split * DK, part);
  if (pg_check_launch("pg_mixture_fwd")) return 1;
  mixture_lse_kernel<<<row_grid(N, THREADS / 32), THREADS, K * sizeof(float), stream>>>(part, splits, N, K,
                                                                                        mixture_logits, a, out);
  return pg_check_launch("pg_mixture_fwd");
}

extern "C" int pg_mixture_bwd(int kind, const float* x, int N, int D, int K, const float* mixture_logits, const float* p0,
                              const float* p1, const float* a, const float* out, const float* g, float* dparams,
                              float* dx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(kind == PG_MIXTURE_GAUSSIAN || kind == PG_MIXTURE_BERNOULLI, "pg_mixture_bwd: unknown kind %d", kind);
  PG_REQUIRE(N >= 0 && D >= 1 && K >= 1, "pg_mixture_bwd: empty problem (N %d, D %d, K %d)", N, D, K);
  if (N == 0) return 0;
  PG_REQUIRE(x && mixture_logits && p0 && (kind == PG_MIXTURE_BERNOULLI || p1) && a && out && g && dparams,
             "pg_mixture_bwd: null argument");
  const int P = kind == PG_MIXTURE_GAUSSIAN ? 2 : 1;
  const long long total = (long long)P * K * D + K;
  PG_REQUIRE(total < (1LL << 31), "pg_mixture_bwd: %lld gradient entries", total);
  const int k_tiles = (K + TC - 1) / TC, d_tiles = (D + TC - 1) / TC, n_chunks = (N + NC - 1) / NC;
  int s = (2 * pg_num_sms() + k_tiles * d_tiles - 1) / (k_tiles * d_tiles);
  s = s < 1 ? 1 : s > MAX_SPLITS ? MAX_SPLITS : s;
  s = s > n_chunks ? n_chunks : s;
  const int chunks_per_split = (n_chunks + s - 1) / s;
  const int splits = (n_chunks + chunks_per_split - 1) / chunks_per_split;
  float* part = nullptr;
  if (pg_scratch((size_t)splits * total * sizeof(float), stream, &part)) return 1;
  const dim3 grid(k_tiles, d_tiles, splits);
  if (kind == PG_MIXTURE_GAUSSIAN)
    mixture_grad_kernel<PG_MIXTURE_GAUSSIAN><<<grid, THREADS, 0, stream>>>(x, N, D, K, p0, p1, mixture_logits, a, out, g,
                                                                            chunks_per_split * NC, total, part);
  else
    mixture_grad_kernel<PG_MIXTURE_BERNOULLI><<<grid, THREADS, 0, stream>>>(x, N, D, K, p0, p1, mixture_logits, a, out,
                                                                             g, chunks_per_split * NC, total, part);
  if (pg_check_launch("pg_mixture_bwd")) return 1;
  if (pg_sum_partials(part, splits, total, 1, (int)total, total, dparams, stream)) return 1;
  if (!dx) return 0;
  const dim3 gx((N + TR - 1) / TR, d_tiles);
  if (kind == PG_MIXTURE_GAUSSIAN)
    mixture_dx_kernel<PG_MIXTURE_GAUSSIAN><<<gx, THREADS, 0, stream>>>(x, N, D, K, p0, p1, a, out, g, dx);
  else
    mixture_dx_kernel<PG_MIXTURE_BERNOULLI><<<gx, THREADS, 0, stream>>>(x, N, D, K, p0, p1, a, out, g, dx);
  return pg_check_launch("pg_mixture_bwd");
}
