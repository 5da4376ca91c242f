// pg_fvbn.cu — the Fully Visible Belief Network (reference models/autoregressive/fvbn.py): one strictly-lower-triangular
// fp32 contraction on the CUDA cores for the logits, its gradients, and one pixel of raster-order sampling.  The D rows
// stay separate parameter tensors (the reference's nn.Linear(max(1, i), 1) modules); every kernel reads them through a
// device table of addresses (see include/pg_b200.h).  Every sum runs in a fixed order and there are no atomics.
#include "pg_common.cuh"

namespace {

constexpr int TILE = 32;            // rows x columns of a tile
constexpr int THREADS = 256;        // 8 warps: lane = the tile's column (or row), warp w takes items w, w + 8, w + 16, w + 24
constexpr int ITEMS = TILE / (THREADS / 32);
constexpr int SPLIT_IMAGES = 128;   // images per batch slice of the weight gradient (fewer slices for small batches)
constexpr int MAX_SPLITS = 32;

__device__ __forceinline__ const float* row_w(const int64_t* __restrict__ params, int i) {
  return reinterpret_cast<const float*>(params[i]);
}
__device__ __forceinline__ float row_b(const int64_t* __restrict__ params, int D, int i) {
  return *reinterpret_cast<const float*>(params[D + i]);
}
__host__ __device__ __forceinline__ long long packed_off(int i) { return i == 0 ? 0 : 1 + (long long)i * (i - 1) / 2; }

// CTA = (32 images) x (32 rows); lane = row i, warp w = images w + 8k.  The column tiles stop at the tile's last row (the
// upper triangle is never read).  Each logit is one fmaf chain over j ascending from 0, then the bias.
__global__ void __launch_bounds__(THREADS) fvbn_fwd_kernel(const int64_t* __restrict__ params, const float* __restrict__ x,
                                                          int n, int D, float* __restrict__ logits) {
  __shared__ float ws[TILE][TILE + 1];  // ws[r][c] = W_{i0 + r}[j0 + c]
  __shared__ float xs[TILE][TILE + 1];  // xs[r][c] = x[b0 + r, j0 + c]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b0 = blockIdx.x * TILE, i0 = blockIdx.y * TILE;
  const int i = i0 + lane;
  const int len = i < D ? i : 0;               // inputs of row i taken from x (row 0's constant 0 comes after the loop)
  const int jend = min(D, i0 + TILE) - 1;      // the tile's last row reads x[:, :jend]
  float acc[ITEMS];
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) acc[k] = 0.f;
  for (int j0 = 0; j0 < jend; j0 += TILE) {
    for (int r = warp; r < TILE; r += THREADS / 32) {
      const int ir = i0 + r, j = j0 + lane, b = b0 + r;
      ws[r][lane] = (ir < D && j < ir) ? row_w(params, ir)[j] : 0.f;
      xs[r][lane] = (b < n && j < D) ? x[(size_t)b * D + j] : 0.f;
    }
    __syncthreads();
    const int lim = len - j0;
#pragma unroll 8
    for (int c = 0; c < TILE; ++c) {
      if (c < lim) {
        const float w = ws[lane][c];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) acc[k] = fmaf(w, xs[warp + 8 * k][c], acc[k]);
      }
    }
    __syncthreads();
  }
  if (i >= D) return;
  const float bi = row_b(params, D, i);
  const float w0 = i == 0 ? row_w(params, 0)[0] : 0.f;
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) {
    const int b = b0 + warp + 8 * k;
    if (i == 0) acc[k] = fmaf(w0, 0.f, acc[k]);
    if (b < n) logits[(size_t)b * D + i] = acc[k] + bi;
  }
}

struct FvbnBwd {
  const int64_t* params;
  const float *x, *g;
  int n, D, nI, n_wtiles, splits, per_split;
  long long T;
  float* part;  // pg_scratch: splits x [T + D] partials, the packed weight gradient then the bias gradient
  float* dx;
};

// Grid: splits x (lower-triangular tile pairs I >= J) weight-gradient CTAs, then (image tiles x column tiles) input-gradient
// CTAs when dx is wanted.
//   weight gradient, CTA (I, J, slice): lane = column j, warp w = rows w + 8k; images of the slice in index order.  The CTAs
//     with J = 0 also sum g over the slice for the bias gradient (warp 0, lane = row).
//   input gradient, CTA (image tile, J): lane = column j, warp w = images w + 8k; rows i > j in ascending order.
__global__ void __launch_bounds__(THREADS) fvbn_bwd_kernel(FvbnBwd a) {
  __shared__ float s0[TILE][TILE + 1];
  __shared__ float s1[TILE][TILE + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D = a.D;
  float acc[ITEMS];
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) acc[k] = 0.f;
  const long long wctas = (long long)a.n_wtiles * a.splits;
  if ((long long)blockIdx.x < wctas) {
    const int slice = blockIdx.x / a.n_wtiles, t = blockIdx.x % a.n_wtiles;
    int I = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);  // t = I (I + 1) / 2 + J, J <= I
    while ((long long)(I + 1) * (I + 2) / 2 <= t) ++I;
    while ((long long)I * (I + 1) / 2 > t) --I;
    const int J = t - I * (I + 1) / 2;
    const int i0 = I * TILE, j0 = J * TILE, j = j0 + lane;
    const int bs = slice * a.per_split, be = min(a.n, bs + a.per_split);
    const bool zero_in = i0 == 0 && warp == 0;  // item k = 0 of warp 0 is row 0, whose input is the constant 0
    float bsum = 0.f;
    for (int c0 = bs; c0 < be; c0 += TILE) {
      for (int r = warp; r < TILE; r += THREADS / 32) {
        const int b = c0 + r;
        s0[r][lane] = (b < be && i0 + lane < D) ? a.g[(size_t)b * D + i0 + lane] : 0.f;  // s0[b][row]
        s1[r][lane] = (b < be && j < D) ? a.x[(size_t)b * D + j] : 0.f;              // s1[b][col]
      }
      __syncthreads();
      const int cn = min(TILE, be - c0);
      for (int c = 0; c < cn; ++c) {
        const float xv = s1[c][lane];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) acc[k] = fmaf(s0[c][warp + 8 * k], (k == 0 && zero_in) ? 0.f : xv, acc[k]);
        if (J == 0 && warp == 0) bsum += s0[c][lane];
      }
      __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int i = i0 + warp + 8 * k;
      if (i < D && j < (i == 0 ? 1 : i)) a.part[slice * (a.T + D) + packed_off(i) + j] = acc[k];
    }
    if (J == 0 && warp == 0 && i0 + lane < D) a.part[slice * (a.T + D) + a.T + i0 + lane] = bsum;
    return;
  }
  const long long t = (long long)blockIdx.x - wctas;
  const int B = (int)(t / a.nI), J = (int)(t % a.nI);
  const int b0 = B * TILE, j0 = J * TILE, j = j0 + lane;
  for (int I = J; I < a.nI; ++I) {
    const int i0 = I * TILE;
    for (int r = warp; r < TILE; r += THREADS / 32) {
      const int b = b0 + r, ir = i0 + r;
      s0[r][lane] = (b < a.n && i0 + lane < D) ? a.g[(size_t)b * D + i0 + lane] : 0.f;  // s0[b][row]
      s1[r][lane] = (ir < D && j < ir) ? row_w(a.params, ir)[j] : 0.f;                 // s1[row][col]
    }
    __syncthreads();
    const int iend = min(D, i0 + TILE) - i0;
    for (int c = 0; c < iend; ++c) {
      if (i0 + c > j) {
        const float w = s1[c][lane];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) acc[k] = fmaf(s0[warp + 8 * k][c], w, acc[k]);
      }
    }
    __syncthreads();
  }
  if (j >= D) return;
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) {
    const int b = b0 + warp + 8 * k;
    if (b < a.n) a.dx[(size_t)b * D + j] = acc[k];
  }
}

// One warp per (image, channel): the lanes load 32 consecutive weights and canvas entries, and every lane runs the same
// fmaf chain over them in ascending j through shuffles (the forward's order, so the logits are bit-identical to it).
constexpr int STEP_THREADS = 128;

__global__ void __launch_bounds__(STEP_THREADS) fvbn_sample_step_kernel(const int64_t* __restrict__ params,
                                                                       const int64_t* __restrict__ pos,
                                                                       const float* __restrict__ canvas, int n, int c,
                                                                       int hw, float* __restrict__ logits) {
  const int lane = threadIdx.x & 31;
  const long long item = (long long)blockIdx.x * (STEP_THREADS / 32) + (threadIdx.x >> 5);
  if (item >= (long long)n * c) return;
  const int b = (int)(item / c), ch = (int)(item % c);
  const int D = c * hw, i = ch * hw + (int)*pos;
  const float* w = row_w(params, i);
  const float* xr = canvas + (size_t)b * D;
  float acc = 0.f;
  if (i == 0) {
    acc = fmaf(w[0], 0.f, acc);
  } else {
    for (int j0 = 0; j0 < i; j0 += 32) {
      const int j = j0 + lane;
      const float wv = j < i ? w[j] : 0.f, xv = j < i ? xr[j] : 0.f;
      const int cnt = min(32, i - j0);
      for (int l = 0; l < cnt; ++l) acc = fmaf(__shfl_sync(0xffffffffu, wv, l), __shfl_sync(0xffffffffu, xv, l), acc);
    }
  }
  if (lane == 0) logits[(size_t)b * c + ch] = acc + row_b(params, D, i);
}

}  // namespace

extern "C" int pg_fvbn_fwd(const int64_t* params, const float* x, int n, int D, float* logits, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D > 0, "pg_fvbn_fwd: empty problem (n %d, D %d)", n, D);
  PG_REQUIRE(D <= 65535 * TILE, "pg_fvbn_fwd: D %d is too large", D);
  if (n == 0) return 0;  // an empty batch (its tensors may have no storage)
  PG_REQUIRE(params && x && logits, "pg_fvbn_fwd: null argument");
  const long long bx = ((long long)n + TILE - 1) / TILE;
  PG_REQUIRE(bx < (1LL << 31), "pg_fvbn_fwd: grid of %lld image tiles", bx);
  fvbn_fwd_kernel<<<dim3((unsigned)bx, (D + TILE - 1) / TILE), THREADS, 0, stream>>>(params, x, n, D, logits);
  return pg_check_launch("pg_fvbn_fwd");
}

extern "C" int pg_fvbn_bwd(const int64_t* params, const float* x, const float* g, int n, int D, float* dw, float* db,
                           float* dx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D > 0, "pg_fvbn_bwd: empty problem (n %d, D %d)", n, D);
  const long long T = packed_off(D - 1) + (D == 1 ? 1 : D - 1);
  PG_REQUIRE(T + D < (1LL << 31), "pg_fvbn_bwd: D %d is too large (%lld packed weights)", D, T);
  if (n == 0) return 0;  // the gradients of an empty batch: nothing to add
  PG_REQUIRE(params && x && g && dw && db, "pg_fvbn_bwd: null argument");
  FvbnBwd a{params, x, g, n, D, (D + TILE - 1) / TILE, 0, 0, 0, T, nullptr, dx};
  a.n_wtiles = a.nI * (a.nI + 1) / 2;
  // batch slices: decided by n alone, so every run of a shape adds the same partials in the same order
  int splits = (n + SPLIT_IMAGES - 1) / SPLIT_IMAGES;
  if (splits > MAX_SPLITS) splits = MAX_SPLITS;
  a.per_split = (n + splits - 1) / splits;
  a.splits = (n + a.per_split - 1) / a.per_split;
  float* scratch = nullptr;
  if (pg_scratch((size_t)a.splits * (T + D) * sizeof(float), stream, &scratch)) return 1;
  a.part = scratch;
  const long long blocks = (long long)a.n_wtiles * a.splits + (dx ? (((long long)n + TILE - 1) / TILE) * a.nI : 0);
  PG_REQUIRE(blocks < (1LL << 31), "pg_fvbn_bwd: grid of %lld CTAs", blocks);
  fvbn_bwd_kernel<<<(unsigned)blocks, THREADS, 0, stream>>>(a);
  if (pg_check_launch("pg_fvbn_bwd")) return 1;
  // one fixed-order sum when db directly follows dw (one [T + D] gradient buffer), else one per output
  if (db == dw + T) return pg_sum_partials(a.part, a.splits, T + D, 1, (int)(T + D), T + D, dw, stream);
  if (pg_sum_partials(a.part, a.splits, T + D, 1, (int)T, T, dw, stream)) return 1;
  return pg_sum_partials(a.part + T, a.splits, T + D, 1, D, D, db, stream);
}

extern "C" int pg_fvbn_sample_step(const int64_t* params, const int64_t* pos, const float* canvas, int n, int c, int hw,
                                   float* logits, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && c > 0 && hw > 0, "pg_fvbn_sample_step: empty problem (n %d, c %d, hw %d)", n, c, hw);
  if (n == 0) return 0;
  PG_REQUIRE(params && pos && canvas && logits, "pg_fvbn_sample_step: null argument");
  const long long blocks = ((long long)n * c + STEP_THREADS / 32 - 1) / (STEP_THREADS / 32);
  PG_REQUIRE(blocks < (1LL << 31), "pg_fvbn_sample_step: grid of %lld CTAs", blocks);
  fvbn_sample_step_kernel<<<(unsigned)blocks, STEP_THREADS, 0, stream>>>(params, pos, canvas, n, c, hw, logits);
  return pg_check_launch("pg_fvbn_sample_step");
}
