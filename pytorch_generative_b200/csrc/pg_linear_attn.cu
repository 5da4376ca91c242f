// pg_linear_attn.cu — the numerator of LinearCausalAttention (reference nn/attention.py:168-200,
// `_UnnormalizedLinearCausalAttention`): out_i = Q_i . S_i with the running state S_i = sum_{j <= i} K_j^T V_j, and its
// gradients, for heads of any width.
//
// The four products share one form, a causal scan with x, y of width P and z, out of width R:
//   out_i = sum_{j <= i} (x_i . y_j) z_j   (forward order)   or   sum_{j >= i}   (reverse order)
//     out:  x = Q, y = K, z = V, forward        dQ:  x = G, y = V, z = K, forward
//     dV:   x = K, y = Q, z = G, reverse        dK:  x = V, y = G, z = Q, reverse
// la_scan_kernel walks the sequence in chunks of T = 64 positions.  With S the sum of y_j^T z_j over the chunks already
// passed, chunk c computes
//   out_c = X_c S + tril(X_c Y_c^T) Z_c      then      S += Y_c^T Z_c.
// A CTA owns one block of 64 z columns: it recomputes X_c Y_c^T for its block, so only a P x 64 slice of the state is
// live.  That slice sits in pg_scratch (one per CTA, L2-resident) and passes through shared memory 64 rows at a time,
// which is what leaves P and R unbounded.  When B x column blocks would leave SMs idle the sequence is also split into
// segments of whole chunks: a first launch (SUMS) writes each segment's Y^T Z to pg_scratch, a second (la_carry_kernel)
// turns them into a running sum, and each segment starts from the sum of the segments before it (after it, in reverse
// order).  The segment count is a function of the shape and
// the SM count; there are no atomics and every sum runs in one fixed order, so two runs give the same bits.
//
// Arithmetic is fp32 FMA on the CUDA cores.  Error: out_i adds X_c S first (P terms; an element of S is a chain over the
// positions before the chunk, the segment sums at most shortening it) and then the chunk's terms j <= i, each a P-term
// dot product; masked and padded terms are exact zeros.  Every term of out_i thus passes through at most P + i + 2
// roundings, within the (L + P + 2) 2^-24 of the sequential form.  O(L (P + R)) memory plus a scratch of B x
// segments x P x R floats (rounded up to 64), which does not grow with L.
#include <algorithm>

#include "../../include/pg_b200.h"
#include "pg_common.cuh"

namespace {

constexpr int T = 64;          // chunk length = state rows per pass = z columns per CTA
constexpr int LDK = T + 4;     // pitch of the k-major tiles (X^T, Y^T, A^T): conflict-free transposed stores
constexpr int LDJ = T + 8;     // pitch of the row-major tiles (Y, Z, S)
constexpr int THREADS = 256;   // each thread owns a 4 x 4 block of every 64 x 64 product

struct LaScan {
  const float *X, *Y, *Z;
  float* out;
  float *state, *part;  // pg_scratch: [B][ncb][nseg][npb * T][T] each
  int L, P, R;
  int ncb, nch, nseg, cps;  // column blocks, chunks, segments, chunks per segment
};

// A 64 x 64 tile of a row-major matrix (pitch ld) into registers, zero outside nrows x ncols.  Warp w reads columns
// 8w .. 8w+7 of four rows per step (32-byte segments).
__device__ __forceinline__ void tile_load(float (&v)[16], const float* __restrict__ src, size_t ld, int nrows, int ncols) {
  const int lane = threadIdx.x & 31, col = (threadIdx.x >> 5) * 8 + (lane & 7);
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    const int row = 4 * m + (lane >> 3);
    v[m] = (row < nrows && col < ncols) ? __ldg(src + row * ld + col) : 0.f;
  }
}
__device__ __forceinline__ void tile_store_rows(float* s, const float (&v)[16]) {  // s[row][col], pitch LDJ
  const int lane = threadIdx.x & 31, col = (threadIdx.x >> 5) * 8 + (lane & 7);
#pragma unroll
  for (int m = 0; m < 16; ++m) s[(4 * m + (lane >> 3)) * LDJ + col] = v[m];
}
__device__ __forceinline__ void tile_store_cols(float* s, const float (&v)[16]) {  // s[col][row], pitch LDK
  const int lane = threadIdx.x & 31, col = (threadIdx.x >> 5) * 8 + (lane & 7);
#pragma unroll
  for (int m = 0; m < 16; ++m) s[col * LDK + 4 * m + (lane >> 3)] = v[m];
}

// c[a][b] += sum_{k < 64} A[k][4 ty + a] * B[k][4 tx + b], k ascending.  A warp covers 4 ty x 8 tx: two 64- and 128-byte
// shared loads per 16 FMAs.
__device__ __forceinline__ void prod64(float (&c)[4][4], const float* A, int lda, const float* B, int ldb, int ty, int tx) {
#pragma unroll 8
  for (int k = 0; k < T; ++k) {
    const float4 a4 = *reinterpret_cast<const float4*>(A + k * lda + 4 * ty);
    const float4 b4 = *reinterpret_cast<const float4*>(B + k * ldb + 4 * tx);
    const float av[4] = {a4.x, a4.y, a4.z, a4.w}, bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) c[i][j] = fmaf(av[i], bv[j], c[i][j]);
  }
}

__device__ __forceinline__ void load4x4(float (&c)[4][4], const float* p) {  // rows of pitch T
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 t = *reinterpret_cast<const float4*>(p + i * T);
    c[i][0] = t.x, c[i][1] = t.y, c[i][2] = t.z, c[i][3] = t.w;
  }
}
__device__ __forceinline__ void store4x4(float* p, int ld, const float (&c)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) *reinterpret_cast<float4*>(p + i * ld) = make_float4(c[i][0], c[i][1], c[i][2], c[i][3]);
}

// SUMS = false: the scan of one (batch, column block, segment).  SUMS = true: only the segment's Y^T Z, into `part`,
// for the segments whose sum a later one starts from (0 .. nseg-2 forward, 1 .. nseg-1 reverse).
template <bool REVERSE, bool SUMS>
__global__ void __launch_bounds__(THREADS, 2) la_scan_kernel(LaScan a) {
  extern __shared__ __align__(16) float smem[];
  float* sY = smem;              // [T][LDJ]  Y tile (j-major)
  float* sZ = sY + T * LDJ;      // [T][LDJ]  Z tile, this CTA's columns
  float* sS = sZ + T * LDJ;      // [T][LDJ]  64 rows of the state
  float* sXt = sS + T * LDJ;     // [T][LDK]  X tile (k-major); A^T once the state passes are done
  float* sYt = sXt + T * LDK;    // [T][LDK]  Y tile (k-major)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ty = (w >> 1) * 4 + (lane >> 3), tx = (w & 1) * 8 + (lane & 7);

  const int seg_grid = SUMS ? a.nseg - 1 : a.nseg;
  const int cb = blockIdx.x % a.ncb, seg = (blockIdx.x / a.ncb) % seg_grid + (SUMS && REVERSE ? 1 : 0);
  const int b = blockIdx.x / (a.ncb * seg_grid);
  const int npb = (a.P + T - 1) / T, c0 = cb * T, ncols = min(T, a.R - c0);
  const size_t slice = (size_t)npb * T * T;
  const size_t slot0 = (size_t)(b * a.ncb + cb) * a.nseg;  // this (batch, column block)'s segment 0
  float* state = (SUMS ? a.part : a.state) + (slot0 + seg) * slice;
  const float* X = a.X + (size_t)b * a.L * a.P;
  const float* Y = a.Y + (size_t)b * a.L * a.P;
  const float* Z = a.Z + (size_t)b * a.L * a.R + c0;
  float* out = a.out + (size_t)b * a.L * a.R + c0;
  const size_t own = (size_t)(4 * ty) * T + 4 * tx;  // this thread's 4 x 4 block of each 64-row pass of the state

  // Every segment but the first in scan order enters with the state la_carry_kernel wrote to its slot.
  bool have = !SUMS && seg != (REVERSE ? a.nseg - 1 : 0);
  const int ch_begin = seg * a.cps, nchunks = min(a.nch, ch_begin + a.cps) - ch_begin;
  for (int n = 0; n < nchunks; ++n) {
    const int i0 = (REVERSE ? ch_begin + nchunks - 1 - n : ch_begin + n) * T, rows = min(T, a.L - i0);
    const bool update = SUMS || n + 1 < nchunks;  // the state after a segment's last chunk is not needed
    float v[16];
    tile_load(v, Z + (size_t)i0 * a.R, a.R, rows, ncols);
    tile_store_rows(sZ, v);
    float acc[4][4] = {}, accA[4][4] = {};
    for (int pb = 0; pb < npb; ++pb) {
      const int k0 = pb * T, kcols = min(T, a.P - k0);
      float s[4][4] = {};
      if (have) load4x4(s, state + pb * T * T + own);
      if (!SUMS) {
        tile_load(v, X + (size_t)i0 * a.P + k0, a.P, rows, kcols);
        tile_store_cols(sXt, v);
        if (have) store4x4(sS + (4 * ty) * LDJ + 4 * tx, LDJ, s);
      }
      tile_load(v, Y + (size_t)i0 * a.P + k0, a.P, rows, kcols);
      if (!SUMS) tile_store_cols(sYt, v);
      tile_store_rows(sY, v);
      __syncthreads();
      if (!SUMS) {
        prod64(accA, sXt, LDK, sYt, LDK, ty, tx);     // X_c Y_c^T
        if (have) prod64(acc, sXt, LDK, sS, LDJ, ty, tx);  // X_c S, with S as it was before this chunk
      }
      if (update) {
        prod64(s, sY, LDJ, sZ, LDJ, ty, tx);  // S += Y_c^T Z_c
        store4x4(state + pb * T * T + own, T, s);
      }
      __syncthreads();
    }
    have = true;
    if (!SUMS) {
      float* sAt = sXt;  // A^T[j][i], causally masked
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ii = 4 * ty + i, jj = 4 * tx + j;
          sAt[jj * LDK + ii] = (REVERSE ? jj >= ii : jj <= ii) ? accA[i][j] : 0.f;
        }
      __syncthreads();
      prod64(acc, sAt, LDK, sZ, LDJ, ty, tx);  // + tril(A) Z_c
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = 4 * ty + i;
        if (row >= rows) break;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (4 * tx + j < ncols) out[(size_t)(i0 + row) * a.R + 4 * tx + j] = acc[i][j];
      }
      __syncthreads();
    }
  }
}

// The state each segment starts from: the segment sums before it (after it, in reverse order) as one running sum per
// state element, in scan order, so nseg reads and writes per element rather than one prefix per segment.
template <bool REVERSE>
__global__ void __launch_bounds__(THREADS) la_carry_kernel(const float* __restrict__ part, float* __restrict__ state,
                                                           long long n, int nseg, long long slice) {
  const int first = REVERSE ? nseg - 1 : 0, step = REVERSE ? -1 : 1;
  for (long long e = (long long)blockIdx.x * THREADS + threadIdx.x; e < n; e += (long long)gridDim.x * THREADS) {
    const long long base = (e / slice) * nseg * slice + e % slice;  // element e % slice of (batch, column block) e / slice
    float s = part[base + first * slice];
#pragma unroll 8
    for (int k = 1; k < nseg; ++k) {
      const long long at = base + (long long)(first + k * step) * slice;
      state[at] = s;
      if (k + 1 < nseg) s += part[at];  // the last segment in scan order has no sum
    }
  }
}

// Dynamic shared memory: the scan 3 [64][72] + 2 [64][68] floats = 90,112 bytes (88 KB: two CTAs per SM); SUMS uses only
// the first two tiles, 36,864 bytes.  ptxas (sm_90a, -O3), registers with __launch_bounds__(256, 2), no spills:
//   scan forward 123, scan reverse 120, SUMS forward 125, SUMS reverse 126; la_carry_kernel 32.
constexpr int SMEM_SCAN = (3 * T * LDJ + 2 * T * LDK) * (int)sizeof(float);
constexpr int SMEM_SUMS = 2 * T * LDJ * (int)sizeof(float);

template <bool REVERSE>
int la_scan(const float* X, const float* Y, const float* Z, float* out, int B, int L, int P, int R, cudaStream_t stream,
            const char* who) {
  LaScan a{X, Y, Z, out, nullptr, nullptr, L, P, R, (R + T - 1) / T, (L + T - 1) / T, 1, 0};
  // Segments only when B x column blocks fills at most half of the resident slots (two CTAs per SM), and never more
  // CTAs than one wave.  Splitting a sequence adds the segment sums (a quarter of a chunk's work per chunk), a running
  // sum over the segments (nseg reads and writes per state element) and two launches.
  const long long ctas = (long long)B * a.ncb, slots = 2LL * pg_num_sms();
  if (ctas * 2 <= slots) a.nseg = (int)std::min<long long>(a.nch, slots / ctas);
  a.cps = (a.nch + a.nseg - 1) / a.nseg;
  a.nseg = (a.nch + a.cps - 1) / a.cps;
  PG_REQUIRE(ctas * a.nseg < (1LL << 31), "%s: grid of %lld CTAs", who, ctas * a.nseg);
  const size_t slice = (size_t)((P + T - 1) / T) * T * T, n_slices = (size_t)ctas * a.nseg;
  float* scratch = nullptr;
  if (pg_scratch((a.nseg > 1 ? 2 : 1) * n_slices * slice * sizeof(float), stream, &scratch)) return 1;
  a.state = scratch;
  a.part = scratch + n_slices * slice;
  if (a.nseg > 1) {
    PG_CUDA(cudaFuncSetAttribute(la_scan_kernel<REVERSE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_SUMS));
    la_scan_kernel<REVERSE, true><<<(unsigned)(ctas * (a.nseg - 1)), THREADS, SMEM_SUMS, stream>>>(a);
    if (pg_check_launch(who)) return 1;
    const long long n = ctas * (long long)slice;
    const long long blocks = std::min<long long>((n + THREADS - 1) / THREADS, 8LL * pg_num_sms());
    la_carry_kernel<REVERSE><<<(unsigned)blocks, THREADS, 0, stream>>>(a.part, a.state, n, a.nseg, (long long)slice);
    if (pg_check_launch(who)) return 1;
  }
  PG_CUDA(cudaFuncSetAttribute(la_scan_kernel<REVERSE, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_SCAN));
  la_scan_kernel<REVERSE, false><<<(unsigned)(ctas * a.nseg), THREADS, SMEM_SCAN, stream>>>(a);
  return pg_check_launch(who);
}

int la_check(int B, int L, int d, int dv, const char* who) {
  PG_REQUIRE(B > 0 && L > 0 && d > 0 && dv > 0, "%s: empty problem", who);
  return 0;
}

}  // namespace

extern "C" int pg_linear_attn_fwd(const float* q, const float* k, const float* v, float* out, int B, int L, int d, int dv,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(q && k && v && out, "pg_linear_attn_fwd: null argument");
  if (la_check(B, L, d, dv, "pg_linear_attn_fwd")) return 1;
  return la_scan<false>(q, k, v, out, B, L, d, dv, stream, "pg_linear_attn_fwd");
}

extern "C" int pg_linear_attn_bwd(const float* q, const float* k, const float* v, const float* g, float* dq, float* dk,
                                  float* dv_out, int B, int L, int d, int dv, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(q && k && v && g && dq && dk && dv_out, "pg_linear_attn_bwd: null argument");
  if (la_check(B, L, d, dv, "pg_linear_attn_bwd")) return 1;
  // dQ_i = G_i S_i^T with S_i = sum_{j<=i} K_j^T V_j;  with R_i = sum_{j>=i} Q_j^T G_j: dV_i = K_i R_i, dK_i = V_i R_i^T
  if (la_scan<false>(g, v, k, dq, B, L, dv, d, stream, "pg_linear_attn_bwd(dq)")) return 1;
  if (la_scan<true>(k, q, g, dv_out, B, L, d, dv, stream, "pg_linear_attn_bwd(dv)")) return 1;
  return la_scan<true>(v, g, q, dk, B, L, dv, d, stream, "pg_linear_attn_bwd(dk)");
}
