// pg_gp.cu — the dense fp64 linear algebra of GaussianProcess (reference models/gaussian_process.py): a GEMM on the FP64
// tensor cores (mma.sync m16n8k16 .f64), a blocked right-looking Cholesky with a semi-definite pivot rule, and blocked
// triangular solves.  Matrices are row-major fp64 with 64-bit offsets.  Every sum runs in a fixed order (one thread or
// one MMA chain owns it, the k-order of the GEMM depends on k alone), no kernel uses atomics and nothing synchronises
// with the host, so repeat runs give the same bits and every launch can be captured in a CUDA graph.
#include "pg_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------------------------
// GEMM: C = alpha op(A) op(B) + beta C.  64 x 64 C tiles, 4 warps of 32 x 32 (2 x 4 m16n8k16 tiles), k in steps of
// 16: each step is one MMA per accumulator tile, so an element's sum runs over k in ascending 16-chunks whatever its
// tile.  Operands are staged through shared memory as [mn][k] (row pitch 20: the fragment loads of a half-warp hit 16
// distinct banks); the next k-step is held in registers while the current one runs.
// ------------------------------------------------------------------------------------------------------------------
constexpr int GBM = 64, GBN = 64, GBK = 16, GPAD = GBK + 4, GTHREADS = 128;

__device__ __forceinline__ void mma_f64_16x8x16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, "
      "{%4, %5, %6, %7, %8, %9, %10, %11}, {%12, %13, %14, %15}, {%0, %1, %2, %3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// Element (mn, kk) of an operand tile sits at p[mn * s_mn + kk * s_k] with one of the strides 1; the 1024 elements of
// a 64 x 16 tile are spread over 128 threads along the unit-stride axis, so global reads coalesce.
struct TileLoader {
  const double* p;
  long long s_mn, s_k;
  int extent_mn, extent_k;
  bool k_fast;

  // Thread t's q-th element: (mn, kk) = (t / 16 + 8 q, t % 16) when k is the unit-stride axis, else
  // (t % 64, t / 64 + 2 q); one pointer and one step per thread.
  __device__ __forceinline__ void load(double (&r)[8], int mn0, int k0) const {
    const int mn = mn0 + (k_fast ? threadIdx.x / GBK : threadIdx.x % GBM);
    const int kk = k0 + (k_fast ? threadIdx.x % GBK : threadIdx.x / GBM);
    const double* q0 = p + (long long)mn * s_mn + (long long)kk * s_k;
    const long long step = k_fast ? 8 * s_mn : 2 * s_k;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const bool in = k_fast ? (mn + 8 * q < extent_mn && kk < extent_k) : (mn < extent_mn && kk + 2 * q < extent_k);
      r[q] = in ? q0[q * step] : 0.0;
    }
  }
  __device__ __forceinline__ void store(double (*s)[GPAD], const double (&r)[8]) const {
    const int mn = k_fast ? threadIdx.x / GBK : threadIdx.x % GBM;
    const int kk = k_fast ? threadIdx.x % GBK : threadIdx.x / GBM;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (k_fast) s[mn + 8 * q][kk] = r[q];
      else s[mn][kk + 2 * q] = r[q];
    }
  }
};

__global__ void __launch_bounds__(GTHREADS)
gemm_f64_kernel(TileLoader la, TileLoader lb, int m, int n, int k, double alpha, double beta, double* __restrict__ C,
                long long ldc, int lower_only) {
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  if (lower_only && n0 > m0 + GBM - 1) return;  // the whole tile lies above the diagonal
  __shared__ double As[GBM][GPAD];
  __shared__ double Bs[GBN][GPAD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;

  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

  double ra[8], rb[8];
  if (k > 0) {
    la.load(ra, m0, 0);
    lb.load(rb, n0, 0);
  }
  for (int k0 = 0; k0 < k; k0 += GBK) {
    __syncthreads();
    la.store(As, ra);
    lb.store(Bs, rb);
    __syncthreads();
    if (k0 + GBK < k) {
      la.load(ra, m0, k0 + GBK);
      lb.load(rb, n0, k0 + GBK);
    }
    double bfr[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int v = 0; v < 4; ++v) bfr[j][v] = Bs[wn + j * 8 + g][t + 4 * v];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      double af[8];
#pragma unroll
      for (int v = 0; v < 8; ++v) af[v] = As[wm + i * 16 + g + 8 * (v & 1)][t + 4 * (v >> 1)];
#pragma unroll
      for (int j = 0; j < 4; ++j) mma_f64_16x8x16(acc[i][j], af, bfr[j]);
    }
  }

#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = m0 + wm + i * 16 + g + 8 * (e >> 1);
        const int c = n0 + wn + j * 8 + 2 * t + (e & 1);
        if (r >= m || c >= n || (lower_only && c > r)) continue;
        double* dst = C + (long long)r * ldc + c;
        const double ab = alpha == 0.0 ? 0.0 : alpha * acc[i][j][e];
        *dst = beta == 0.0 ? ab : ab + beta * *dst;  // beta == 0 never reads C (it may hold NaN)
      }
}

// ------------------------------------------------------------------------------------------------------------------
// Cholesky and triangular solves: NB x NB diagonal blocks.
// ------------------------------------------------------------------------------------------------------------------
constexpr int NB = 64;
constexpr int DTHREADS = 256;

// A[i][i] += noise, A[i][j] = 0 for j > i; *dropped = 0.
__global__ void __launch_bounds__(DTHREADS)
potrf_prep_kernel(double* __restrict__ A, int n, long long lda, double noise, int* __restrict__ dropped) {
  const long long total = (long long)n * n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *dropped = 0;
  for (long long e = (long long)blockIdx.x * DTHREADS + threadIdx.x; e < total; e += (long long)gridDim.x * DTHREADS) {
    const long long i = e / n, j = e % n;
    if (j > i) A[i * lda + j] = 0.0;
    else if (j == i) A[i * lda + j] += noise;
  }
}

// One CTA factors the diagonal block at (j0, j0) in place, column by column (right-looking, rank-1 updates in
// ascending pivot order).  The first block also computes the pivot tolerance tau = n 2^-52 max_i A_ii into tau[0].
// A pivot d with isfinite(d) && d <= tau is dropped: its column of L is zeroed and *dropped counts it.
__global__ void __launch_bounds__(DTHREADS)
potrf_diag_kernel(double* __restrict__ A, int n, long long lda, int j0, double* __restrict__ tau,
                  int* __restrict__ dropped) {
  __shared__ double S[NB][NB + 1];
  __shared__ double red[DTHREADS];
  __shared__ double s_tau;
  __shared__ int s_drop;
  const int b = min(NB, n - j0);
  if (j0 == 0) {
    double mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += DTHREADS) mx = fmax(mx, A[(long long)i * lda + i]);
    red[threadIdx.x] = mx;
    __syncthreads();
    for (int s = DTHREADS / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      s_tau = (double)n * 0x1p-52 * red[0];
      *tau = s_tau;
    }
  } else if (threadIdx.x == 0) {
    s_tau = *tau;
  }
  for (int e = threadIdx.x; e < b * b; e += DTHREADS) {
    const int i = e / b, j = e % b;
    S[i][j] = j <= i ? A[(long long)(j0 + i) * lda + j0 + j] : 0.0;
  }
  if (threadIdx.x == 0) s_drop = 0;
  __syncthreads();
  const double tol = s_tau;
  for (int kk = 0; kk < b; ++kk) {
    if (threadIdx.x == 0) {
      const double d = S[kk][kk];
      if (isfinite(d) && d <= tol) {
        S[kk][kk] = 0.0;
        ++s_drop;
      } else {
        S[kk][kk] = sqrt(d);
      }
    }
    __syncthreads();
    const double piv = S[kk][kk];
    for (int i = kk + 1 + threadIdx.x; i < b; i += DTHREADS) S[i][kk] = piv == 0.0 ? 0.0 : S[i][kk] / piv;
    __syncthreads();
    const int w = b - kk - 1;
    for (int e = threadIdx.x; e < w * w; e += DTHREADS) {
      const int i = kk + 1 + e / w, j = kk + 1 + e % w;
      if (j <= i) S[i][j] -= S[i][kk] * S[j][kk];
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < b * b; e += DTHREADS) {
    const int i = e / b, j = e % b;
    if (j <= i) A[(long long)(j0 + i) * lda + j0 + j] = S[i][j];
  }
  if (threadIdx.x == 0) *dropped += s_drop;
}

// Triangular solve of one diagonal block: L_d X = B_d (forward) or L_d^T X = B_d (backward), L_d the b x b lower block
// at L (pitch ldl), element (i, c) of B_d at B[i s_i + c s_c].  A CTA owns 32 columns c; thread (c, g) holds rows
// g, g + 8, ... of its column in registers.  Row r's solution is published through shared memory and every later row
// subtracts its term, so each element's sum runs in pivot order, independent of the other columns.  A zero diagonal
// entry gives x_r = 0.  The same kernel is the Cholesky panel: rows of A below the diagonal block solve x L11^T = a,
// i.e. L11 x^T = a^T, with the panel rows as the columns (s_i = 1, s_c = lda).
constexpr int TCOLS = 32, TGROUPS = 8, TROWS = NB / TGROUPS;

__global__ void __launch_bounds__(TCOLS * TGROUPS)
tri_solve_kernel(const double* __restrict__ L, long long ldl, int b, double* __restrict__ B, long long s_i,
                 long long s_c, int ncols, int transpose) {
  __shared__ double Ls[NB][NB];
  __shared__ double xs[NB][TCOLS];
  const int tid = threadIdx.y * TCOLS + threadIdx.x;
  for (int e = tid; e < b * b; e += TCOLS * TGROUPS) {
    const int i = e / b, j = e % b;
    Ls[i][j] = j <= i ? L[(long long)i * ldl + j] : 0.0;
  }
  const int c = blockIdx.x * TCOLS + threadIdx.x, g = threadIdx.y;
  const bool live = c < ncols;
  double x[TROWS];
#pragma unroll
  for (int q = 0; q < TROWS; ++q) {
    const int i = g + TGROUPS * q;
    x[q] = (live && i < b) ? B[(long long)i * s_i + (long long)c * s_c] : 0.0;
  }
  __syncthreads();
  for (int s = 0; s < b; ++s) {
    const int r = transpose ? b - 1 - s : s;
    if (g == (r & (TGROUPS - 1))) {
#pragma unroll
      for (int q = 0; q < TROWS; ++q)
        if (g + TGROUPS * q == r) {
          const double d = Ls[r][r];
          x[q] = d == 0.0 ? 0.0 : x[q] / d;
          xs[r][threadIdx.x] = x[q];
        }
    }
    __syncthreads();
    const double xr = xs[r][threadIdx.x];
#pragma unroll
    for (int q = 0; q < TROWS; ++q) {
      const int i = g + TGROUPS * q;
      if (i < b && (transpose ? i < r : i > r)) x[q] -= (transpose ? Ls[r][i] : Ls[i][r]) * xr;
    }
  }
  if (live) {
#pragma unroll
    for (int q = 0; q < TROWS; ++q) {
      const int i = g + TGROUPS * q;
      if (i < b) B[(long long)i * s_i + (long long)c * s_c] = x[q];
    }
  }
}

int tri_solve(const double* L, long long ldl, int b, double* B, long long s_i, long long s_c, int ncols, int transpose,
              cudaStream_t stream, const char* what) {
  const dim3 block(TCOLS, TGROUPS), grid((unsigned)((ncols + TCOLS - 1) / TCOLS));
  tri_solve_kernel<<<grid, block, 0, stream>>>(L, ldl, b, B, s_i, s_c, ncols, transpose);
  return pg_check_launch(what);
}

unsigned grid_for(long long total) {
  long long blocks = (total + DTHREADS - 1) / DTHREADS;
  const long long cap = (long long)pg_num_sms() * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

int gemm_f64(int transA, int transB, int m, int n, int k, double alpha, const double* A, int64_t lda, const double* B,
             int64_t ldb, double beta, double* C, int64_t ldc, int lower_only, cudaStream_t stream) {
  if (m == 0 || n == 0) return 0;
  // op(A)[i][p] = A[i * lda + p] (transA = 0) or A[p * lda + i]; op(B)[p][j] = B[p * ldb + j] (transB = 0) or
  // B[j * ldb + p].  The tiles are indexed [mn][k].
  TileLoader la{A, transA ? 1 : (long long)lda, transA ? (long long)lda : 1, m, k, !transA};
  TileLoader lb{B, transB ? (long long)ldb : 1, transB ? 1 : (long long)ldb, n, k, transB != 0};
  dim3 grid((n + GBN - 1) / GBN, (m + GBM - 1) / GBM);
  gemm_f64_kernel<<<grid, GTHREADS, 0, stream>>>(la, lb, m, n, k, alpha, beta, C, ldc, lower_only);
  return pg_check_launch("pg_gemm_f64");
}

}  // namespace

extern "C" int pg_gemm_f64(int transA, int transB, int m, int n, int k, double alpha, const double* A, int64_t lda,
                           const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int lower_only,
                           void* stream_) {
  PG_REQUIRE(m >= 0 && n >= 0 && k >= 0, "pg_gemm_f64: m = %d, n = %d, k = %d", m, n, k);
  PG_REQUIRE(m <= 65535 * GBM, "pg_gemm_f64: m = %d > %d", m, 65535 * GBM);
  PG_REQUIRE(C || m == 0 || n == 0, "pg_gemm_f64: null C");
  PG_REQUIRE(k == 0 || m == 0 || n == 0 || (A && B), "pg_gemm_f64: null operand");
  PG_REQUIRE(lda >= (transA ? m : k) && ldb >= (transB ? k : n) && ldc >= n,
             "pg_gemm_f64: lda = %lld, ldb = %lld, ldc = %lld too small for transA = %d, transB = %d, m = %d, n = %d, "
             "k = %d", (long long)lda, (long long)ldb, (long long)ldc, transA, transB, m, n, k);
  return gemm_f64(transA, transB, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, lower_only,
                  reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int pg_gp_potrf(double* A, int n, int64_t lda, double noise, int* dropped, void* stream_) {
  PG_REQUIRE(n >= 0 && lda >= n, "pg_gp_potrf: n = %d, lda = %lld (>= n)", n, (long long)lda);
  PG_REQUIRE(dropped && (A || n == 0), "pg_gp_potrf: null argument");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) {
    PG_CUDA(cudaMemsetAsync(dropped, 0, sizeof(int), stream));
    return 0;
  }
  float* scratch = nullptr;
  if (pg_scratch(sizeof(double), stream, &scratch)) return 1;
  double* tau = reinterpret_cast<double*>(scratch);
  potrf_prep_kernel<<<grid_for((long long)n * n), DTHREADS, 0, stream>>>(A, n, lda, noise, dropped);
  if (pg_check_launch("pg_gp_potrf")) return 1;
  for (int j0 = 0; j0 < n; j0 += NB) {
    potrf_diag_kernel<<<1, DTHREADS, 0, stream>>>(A, n, lda, j0, tau, dropped);
    if (pg_check_launch("pg_gp_potrf")) return 1;
    const int rest = n - j0 - NB;
    if (rest <= 0) break;
    double* L21 = A + (long long)(j0 + NB) * lda + j0;
    if (tri_solve(A + (long long)j0 * lda + j0, lda, NB, L21, 1, lda, rest, 0, stream, "pg_gp_potrf")) return 1;
    if (gemm_f64(0, 1, rest, rest, NB, -1.0, L21, lda, L21, lda, 1.0, L21 + NB, lda, 1, stream)) return 1;
  }
  return 0;
}

extern "C" int pg_gp_trsm(const double* L, int n, double* B, int ncols, int transpose, void* stream_) {
  PG_REQUIRE(n >= 0 && ncols >= 0, "pg_gp_trsm: n = %d, ncols = %d", n, ncols);
  PG_REQUIRE((L && B) || n == 0 || ncols == 0, "pg_gp_trsm: null argument");
  if (n == 0 || ncols == 0) return 0;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int T = (n + NB - 1) / NB;
  for (int s = 0; s < T; ++s) {
    const int blk = transpose ? T - 1 - s : s;
    const int i0 = blk * NB, b = min(NB, n - i0);
    if (tri_solve(L + (long long)i0 * n + i0, n, b, B + (long long)i0 * ncols, ncols, 1, ncols, transpose, stream,
                  "pg_gp_trsm"))
      return 1;
    if (s == T - 1) break;
    if (!transpose) {  // B[i0 + b :] -= L[i0 + b :, i0 : i0 + b] X_i
      if (gemm_f64(0, 0, n - i0 - b, ncols, b, -1.0, L + (long long)(i0 + b) * n + i0, n, B + (long long)i0 * ncols,
                   ncols, 1.0, B + (long long)(i0 + b) * ncols, ncols, 0, stream))
        return 1;
    } else {  // B[: i0] -= L[i0 : i0 + b, : i0]^T X_i
      if (gemm_f64(1, 0, i0, ncols, b, -1.0, L + (long long)i0 * n, n, B + (long long)i0 * ncols, ncols, 1.0, B, ncols,
                   0, stream))
        return 1;
    }
  }
  return 0;
}
