// pg_vq.cu — the vector quantizer of VQ-VAE / VQ-VAE-2 (reference nn/utils.py `VectorQuantizer`) and the mean squared
// error of their losses.  Rows are pixel-major fp32 [P, ld_x] (the reference's flat_x); the codebook is fp32 [K, d].
//
// The nearest-code search runs in fp32 on the CUDA cores, not on bf16 tensor cores: the argmin is a discontinuous
// decision, and bf16 distances would flip it whenever two codes are within about 2^-8 of each other.  Codes are scanned
// in ascending order with a strict `<` and the per-thread winners are combined by (distance, index), so ties keep the
// lowest index as torch.argmin does.  Every sum runs in a fixed order (fmaf chains in ascending column order, per-CTA
// partials in a fixed tree, partials added by pg_sum_partials in block order), and there are no atomics: every run
// gives bit-identical results.
#include "pg_common.cuh"

#include <math.h>

namespace {

constexpr int THREADS = 256;
// pg_vq_assign: ROWS rows per CTA, each scanned by GROUPS threads that take every GROUPS-th code of a chunk
constexpr int ROWS = 64, GROUPS = THREADS / ROWS;
constexpr int REG_D4 = 16;                      // rows of up to 64 columns are held in registers
constexpr size_t ASSIGN_SMEM = 160 * 1024;      // codebook chunk + its squared norms
// pg_vq_code_sums: KB codes x CC columns per CTA; each warp scans one slice of the rows
constexpr int KB = 4, CC = 128, WARPS = THREADS / 32;

__device__ __forceinline__ float out_load(const void* p, long long i, int f32) {
  return f32 ? static_cast<const float*>(p)[i] : __bfloat162float(static_cast<const bf16*>(p)[i]);
}
__device__ __forceinline__ void out_store(void* p, long long i, float v, int f32) {
  if (f32) {
    static_cast<float*>(p)[i] = v;
  } else {
    static_cast<bf16*>(p)[i] = __float2bfloat16(v);
  }
}

// Fixed-tree block sum (THREADS threads); thread 0 gets the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < THREADS / 32; ++w) s += red[w];
  return s;
}

// x.e of one code: an fmaf chain in ascending column order (x from registers when D4 > 0, else from global memory).
template <int D4>
__device__ __forceinline__ float code_dot(const float4 (&xv)[D4 > 0 ? D4 : 1], const float* __restrict__ xr,
                                          const float4* ek, int d, int d4) {
  float dot = 0.f;
  if (D4 > 0) {
#pragma unroll
    for (int j4 = 0; j4 < (D4 > 0 ? D4 : 1); ++j4) {
      if (j4 < d4) {
        const float4 ev = ek[j4];
        dot = fmaf(xv[j4].x, ev.x, dot);
        dot = fmaf(xv[j4].y, ev.y, dot);
        dot = fmaf(xv[j4].z, ev.z, dot);
        dot = fmaf(xv[j4].w, ev.w, dot);
      }
    }
  } else {
    const float* ekf = reinterpret_cast<const float*>(ek);
    for (int j = 0; j < d; ++j) dot = fmaf(xr[j], ekf[j], dot);
  }
  return dot;
}

// dist = (|x|^2 + |e|^2) - 2 x.e, the reference's formula; x.e and both norms are fmaf chains in ascending column order.
template <int D4>
__global__ void __launch_bounds__(THREADS)
vq_assign_kernel(const float* __restrict__ x, long long ld_x, int P, int d, const float* __restrict__ emb, int K, int kc_max,
                 int* __restrict__ idx, void* __restrict__ out, long long ld_out, int col0, int out_cols, int out_f32,
                 float* __restrict__ part) {
  extern __shared__ float4 smem4[];
  const int d4 = (d + 3) / 4;
  float4* ecode = smem4;                                                   // [kc_max][d4], zero beyond d
  float* enorm = reinterpret_cast<float*>(smem4 + (size_t)kc_max * d4);  // [kc_max]
  __shared__ float best_d[GROUPS][ROWS];
  __shared__ int best_k[GROUPS][ROWS];
  __shared__ int chosen[ROWS];
  __shared__ float red[THREADS / 32];

  const int r_local = threadIdx.x % ROWS, group = threadIdx.x / ROWS;  // a group is two whole warps
  const long long row0 = (long long)blockIdx.x * ROWS;
  const long long row = row0 + r_local;
  const bool live = row < P;
  const float* xr = x + (live ? row : 0) * ld_x;

  float4 xv[D4 > 0 ? D4 : 1];
  float xn = 0.f;
  if (D4 > 0) {
#pragma unroll
    for (int j4 = 0; j4 < (D4 > 0 ? D4 : 1); ++j4) {
      float v[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int j = 4 * j4 + t;
        v[t] = (live && j < d) ? xr[j] : 0.f;
        if (j < d) xn = fmaf(v[t], v[t], xn);
      }
      xv[j4] = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
    for (int j = 0; j < d; ++j) {
      const float v = live ? xr[j] : 0.f;
      xn = fmaf(v, v, xn);
    }
  }

  float bd = INFINITY;
  int bk = 0x7fffffff;
  for (int k0 = 0; k0 < K; k0 += kc_max) {
    const int kc = min(kc_max, K - k0);
    __syncthreads();  // the previous chunk is no longer read
    float* ef = reinterpret_cast<float*>(ecode);
    for (int k = threadIdx.x >> 5; k < kc; k += THREADS / 32)
      for (int j = threadIdx.x & 31; j < d4 * 4; j += 32)
        ef[(size_t)k * d4 * 4 + j] = j < d ? emb[(long long)(k0 + k) * d + j] : 0.f;
    __syncthreads();
    for (int k = threadIdx.x; k < kc; k += THREADS) {
      float s = 0.f;
      for (int j = 0; j < d; ++j) s = fmaf(ef[(size_t)k * d4 * 4 + j], ef[(size_t)k * d4 * 4 + j], s);
      enorm[k] = s;
    }
    __syncthreads();
    if (live) {
      // two codes per step (k and k + GROUPS): two independent fmaf chains, still compared in ascending order
      for (int k = group; k < kc; k += 2 * GROUPS) {
        const int k2 = k + GROUPS < kc ? k + GROUPS : k;
        const float dot1 = code_dot<D4>(xv, xr, ecode + (size_t)k * d4, d, d4);
        const float dot2 = code_dot<D4>(xv, xr, ecode + (size_t)k2 * d4, d, d4);
        const float dist1 = __fsub_rn(__fadd_rn(xn, enorm[k]), 2.f * dot1);
        const float dist2 = __fsub_rn(__fadd_rn(xn, enorm[k2]), 2.f * dot2);
        if (dist1 < bd) {  // ascending k within this thread: the first minimum
          bd = dist1;
          bk = k0 + k;
        }
        if (k2 != k && dist2 < bd) {
          bd = dist2;
          bk = k0 + k2;
        }
      }
    }
  }
  best_d[group][r_local] = bd;
  best_k[group][r_local] = bk;
  __syncthreads();
  if (threadIdx.x < ROWS) {
    float d0 = best_d[0][threadIdx.x];
    int k0 = best_k[0][threadIdx.x];
    for (int g = 1; g < GROUPS; ++g) {
      const float dg = best_d[g][threadIdx.x];
      const int kg = best_k[g][threadIdx.x];
      if (dg < d0 || (dg == d0 && kg < k0)) {
        d0 = dg;
        k0 = kg;
      }
    }
    if (k0 == 0x7fffffff) k0 = 0;  // no finite distance: torch.argmin's index of an all-inf row
    chosen[threadIdx.x] = k0;
    if (row0 + threadIdx.x < P) idx[row0 + threadIdx.x] = k0;
  }
  __syncthreads();

  // the operand x + (q - x), zero in [d, out_cols), and this CTA's share of sum (x - q)^2
  const int rows_here = (int)min((long long)ROWS, P - row0);
  float acc = 0.f;
  for (int e = threadIdx.x; e < rows_here * out_cols; e += THREADS) {
    const int r = e / out_cols, c = e % out_cols;
    float v = 0.f;
    if (c < d) {
      const float xv1 = x[(row0 + r) * ld_x + c];
      const float q = emb[(long long)chosen[r] * d + c];
      const float diff = __fsub_rn(xv1, q);
      acc = __fadd_rn(acc, __fmul_rn(diff, diff));
      v = __fadd_rn(xv1, __fsub_rn(q, xv1));
    }
    if (out) out_store(out, (row0 + r) * ld_out + col0 + c, v, out_f32);
  }
  const float s = block_sum(acc, red);
  if (threadIdx.x == 0 && part) part[blockIdx.x] = s;
}

// Per-code counts and sums of the rows assigned to each code, or of ((q - x) scale) g when emb is given.  CTA
// (blockIdx.x, blockIdx.y) owns codes [KB x, KB x + KB) and columns [CC y, CC y + CC); warp w scans the w-th slice of
// the rows in ascending order, and the warps' sums are added in warp order.
__global__ void __launch_bounds__(THREADS)
vq_code_sums_kernel(const float* __restrict__ x, long long ld_x, int P, int d, const int* __restrict__ idx, int K,
                    const float* __restrict__ emb, const float* __restrict__ g, float scale, float* __restrict__ counts,
                    float* __restrict__ sums) {
  __shared__ float wsum[WARPS][KB][CC];
  __shared__ float wcnt[WARPS][KB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb0 = blockIdx.x * KB, c0 = blockIdx.y * CC;
  const long long slice = ((long long)P + WARPS - 1) / WARPS;
  const long long r_begin = warp * slice, r_end = min((long long)P, r_begin + slice);
  const float gs = emb ? g[0] : 0.f;
  float acc[KB][CC / 32];
  float cnt[KB];
#pragma unroll
  for (int i = 0; i < KB; ++i) {
    cnt[i] = 0.f;
#pragma unroll
    for (int t = 0; t < CC / 32; ++t) acc[i][t] = 0.f;
  }
  for (long long base = r_begin; base < r_end; base += 32) {
    const long long r = base + lane;
    const int mine = r < r_end ? idx[r] - kb0 : -1;
    unsigned hit = __ballot_sync(0xffffffffu, mine >= 0 && mine < KB);
    while (hit) {  // ascending rows
      const int src = __ffs(hit) - 1;
      hit &= hit - 1;
      const int kk = __shfl_sync(0xffffffffu, mine, src);
      const long long rr = base + src;
#pragma unroll
      for (int i = 0; i < KB; ++i) {
        if (kk != i) continue;
        cnt[i] += 1.f;
#pragma unroll
        for (int t = 0; t < CC / 32; ++t) {
          const int c = c0 + lane + 32 * t;
          if (c < d) {
            float v = x[rr * ld_x + c];
            if (emb) v = __fmul_rn(__fmul_rn(__fsub_rn(emb[(long long)(kb0 + i) * d + c], v), scale), gs);
            acc[i][t] = __fadd_rn(acc[i][t], v);
          }
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < KB; ++i) {
#pragma unroll
    for (int t = 0; t < CC / 32; ++t) wsum[warp][i][lane + 32 * t] = acc[i][t];
    if (lane == 0) wcnt[warp][i] = cnt[i];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < KB * CC; e += THREADS) {
    const int i = e / CC, cc = e % CC;
    const int k = kb0 + i, c = c0 + cc;
    if (k >= K || c >= d) continue;
    float s = 0.f;
    for (int w = 0; w < WARPS; ++w) s = __fadd_rn(s, wsum[w][i][cc]);
    sums[(long long)k * d + c] = s;
    if (counts && cc == 0 && blockIdx.y == 0) {
      float n = 0.f;
      for (int w = 0; w < WARPS; ++w) n += wcnt[w][i];
      counts[k] = n;
    }
  }
}

// One thread per code: cs = decay cs + (1 - decay) count, avg = decay avg + (1 - decay) sum, emb = avg / (cs + 1e-5).
__global__ void __launch_bounds__(THREADS)
vq_ema_kernel(const float* __restrict__ counts, const float* __restrict__ sums, int K, int d, float decay,
              float one_minus_decay, float* __restrict__ cluster_size, float* __restrict__ avg, float* __restrict__ emb) {
  const int k = blockIdx.x * THREADS + threadIdx.x;
  if (k >= K) return;
  const float cs = __fadd_rn(__fmul_rn(cluster_size[k], decay), __fmul_rn(counts[k], one_minus_decay));
  cluster_size[k] = cs;
  const float den = __fadd_rn(cs, 1e-5f);
  for (int j = 0; j < d; ++j) {
    const long long i = (long long)k * d + j;
    const float a = __fadd_rn(__fmul_rn(avg[i], decay), __fmul_rn(sums[i], one_minus_decay));
    avg[i] = a;
    emb[i] = __fdiv_rn(a, den);
  }
}

// dx = dq + ((x - q) scale) g, zero in [d, ld_dx).
__global__ void __launch_bounds__(THREADS)
vq_bwd_kernel(const float* __restrict__ x, long long ld_x, int P, int d, const float* __restrict__ emb,
              const int* __restrict__ idx, const void* __restrict__ dq, long long ld_dq, int col0, const float* __restrict__ g,
              float scale, int f32, void* __restrict__ dx, long long ld_dx) {
  const long long total = (long long)P * ld_dx;
  const float gs = g ? g[0] : 0.f;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const long long r = i / ld_dx;
    const int c = (int)(i % ld_dx);
    float v = 0.f;
    if (c < d) {
      const float xv = x[r * ld_x + c], q = emb[(long long)idx[r] * d + c];
      const float commit = __fmul_rn(__fmul_rn(__fsub_rn(xv, q), scale), gs);
      v = __fadd_rn(dq ? out_load(dq, r * ld_dq + col0 + c, f32) : 0.f, commit);
    }
    out_store(dx, i, v, f32);
  }
}

// Forward (part given): this CTA's share of sum (a - b)^2 over rows [ROWS_MSE x, ...).  Backward (g given):
// da = ((a - b) scale) g and db = -da, zero in the pad columns up to each pitch.
constexpr int ROWS_MSE = 32;
__global__ void __launch_bounds__(THREADS)
mse_kernel(const float* __restrict__ a, long long ld_a, const float* __restrict__ b, long long ld_b, int rows, int cols,
           const float* __restrict__ g, float scale, float* __restrict__ part, float* __restrict__ da, long long ld_da,
           float* __restrict__ db, long long ld_db) {
  __shared__ float red[THREADS / 32];
  const long long r0 = (long long)blockIdx.x * ROWS_MSE;
  const int rows_here = (int)min((long long)ROWS_MSE, rows - r0);
  if (part) {
    float acc = 0.f;
    for (long long e = threadIdx.x; e < (long long)rows_here * cols; e += THREADS) {
      const long long r = r0 + e / cols;
      const int c = (int)(e % cols);
      const float diff = __fsub_rn(a[r * ld_a + c], b[r * ld_b + c]);
      acc = __fadd_rn(acc, __fmul_rn(diff, diff));
    }
    const float s = block_sum(acc, red);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
    return;
  }
  const float gs = g[0];
  const long long width = ld_da > ld_db ? ld_da : ld_db;
  for (long long e = threadIdx.x; e < (long long)rows_here * width; e += THREADS) {
    const long long r = r0 + e / width;
    const int c = (int)(e % width);
    float v = 0.f;
    if (c < cols) v = __fmul_rn(__fmul_rn(__fsub_rn(a[r * ld_a + c], b[r * ld_b + c]), scale), gs);
    if (da && c < ld_da) da[r * ld_da + c] = v;
    if (db && c < ld_db) db[r * ld_db + c] = -v;
  }
}

}  // namespace

extern "C" int pg_vq_assign(const float* x, int64_t ld_x, int P, int d, const float* emb, int K, int* idx, void* out,
                            int out_f32, int64_t ld_out, int col0, int out_cols, float* loss_sum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(P >= 0 && d >= 1 && K >= 1, "pg_vq_assign: P = %d, d = %d, K = %d", P, d, K);
  PG_REQUIRE(x && emb && idx, "pg_vq_assign: null argument");
  PG_REQUIRE(ld_x >= d, "pg_vq_assign: pitch ld_x = %lld < d = %d", (long long)ld_x, d);
  PG_REQUIRE(!out || (col0 >= 0 && out_cols >= d && col0 + out_cols <= ld_out),
             "pg_vq_assign: columns [%d, %d + %d) do not fit the output pitch %lld (and must hold d = %d)", col0, col0,
             out_cols, (long long)ld_out, d);
  if (P == 0) return 0;
  const int d4 = (d + 3) / 4;
  const size_t per_code = (size_t)d4 * 16 + 4;
  PG_REQUIRE(per_code <= ASSIGN_SMEM, "pg_vq_assign: d = %d does not fit one code in shared memory", d);
  int kc_max = (int)(ASSIGN_SMEM / per_code);
  if (kc_max > K) kc_max = K;
  const size_t smem = (size_t)kc_max * per_code;
  const unsigned blocks = (unsigned)((P + ROWS - 1) / ROWS);
  float* part = nullptr;
  if (loss_sum && pg_scratch((size_t)blocks * sizeof(float), stream, &part)) return 1;
  if (d4 <= REG_D4) {
    PG_CUDA(cudaFuncSetAttribute(vq_assign_kernel<REG_D4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    vq_assign_kernel<REG_D4><<<blocks, THREADS, smem, stream>>>(x, ld_x, P, d, emb, K, kc_max, idx, out, ld_out, col0,
                                                                 out_cols, out_f32, part);
  } else {
    PG_CUDA(cudaFuncSetAttribute(vq_assign_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    vq_assign_kernel<0><<<blocks, THREADS, smem, stream>>>(x, ld_x, P, d, emb, K, kc_max, idx, out, ld_out, col0,
                                                            out_cols, out_f32, part);
  }
  if (pg_check_launch("pg_vq_assign")) return 1;
  return loss_sum ? pg_sum_partials(part, (int)blocks, 1, 1, 1, 1, loss_sum, stream) : 0;
}

extern "C" int pg_vq_code_sums(const float* x, int64_t ld_x, int P, int d, const int* idx, int K, const float* emb,
                               const float* g, float scale, float* counts, float* sums, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(P >= 0 && d >= 1 && K >= 1, "pg_vq_code_sums: P = %d, d = %d, K = %d", P, d, K);
  PG_REQUIRE(x && idx && sums && (!emb || g), "pg_vq_code_sums: null argument");
  PG_REQUIRE(ld_x >= d, "pg_vq_code_sums: pitch ld_x = %lld < d = %d", (long long)ld_x, d);
  dim3 grid((unsigned)((K + KB - 1) / KB), (unsigned)((d + CC - 1) / CC));
  vq_code_sums_kernel<<<grid, THREADS, 0, stream>>>(x, ld_x, P, d, idx, K, emb, g, scale, counts, sums);
  return pg_check_launch("pg_vq_code_sums");
}

extern "C" int pg_vq_ema_update(const float* counts, const float* sums, int K, int d, float decay, float one_minus_decay,
                                float* cluster_size, float* embedding_avg, float* embedding, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(K >= 1 && d >= 1, "pg_vq_ema_update: K = %d, d = %d", K, d);
  PG_REQUIRE(counts && sums && cluster_size && embedding_avg && embedding, "pg_vq_ema_update: null argument");
  vq_ema_kernel<<<(unsigned)((K + THREADS - 1) / THREADS), THREADS, 0, stream>>>(
      counts, sums, K, d, decay, one_minus_decay, cluster_size, embedding_avg, embedding);
  return pg_check_launch("pg_vq_ema_update");
}

extern "C" int pg_vq_bwd(const float* x, int64_t ld_x, int P, int d, const float* emb, const int* idx, const void* dq,
                         int64_t ld_dq, int col0, const float* g, float scale, int f32, void* dx, int64_t ld_dx,
                         void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(P >= 0 && d >= 1, "pg_vq_bwd: P = %d, d = %d", P, d);
  PG_REQUIRE(x && emb && idx && dx, "pg_vq_bwd: null argument");
  PG_REQUIRE(ld_x >= d && ld_dx >= d && (!dq || (col0 >= 0 && col0 + d <= ld_dq)),
             "pg_vq_bwd: pitches ld_x = %lld, ld_dq = %lld (from column %d), ld_dx = %lld for d = %d", (long long)ld_x,
             (long long)ld_dq, col0, (long long)ld_dx, d);
  const long long total = (long long)P * ld_dx;
  if (total == 0) return 0;
  long long blocks = (total + THREADS - 1) / THREADS;
  const long long cap = (long long)pg_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  vq_bwd_kernel<<<(unsigned)blocks, THREADS, 0, stream>>>(x, ld_x, P, d, emb, idx, dq, ld_dq, col0, g, scale, f32, dx,
                                                          ld_dx);
  return pg_check_launch("pg_vq_bwd");
}

extern "C" int pg_mse_mean(const float* a, int64_t ld_a, const float* b, int64_t ld_b, int rows, int cols, const float* g,
                           float scale, float* loss_sum, float* da, int64_t ld_da, float* db, int64_t ld_db,
                           void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(rows >= 0 && cols >= 1, "pg_mse_mean: rows = %d, cols = %d", rows, cols);
  PG_REQUIRE(a && b, "pg_mse_mean: null argument");
  PG_REQUIRE((loss_sum != nullptr) != (g != nullptr), "pg_mse_mean: give either loss_sum (forward) or g (backward)");
  PG_REQUIRE(ld_a >= cols && ld_b >= cols && (!da || ld_da >= cols) && (!db || ld_db >= cols),
             "pg_mse_mean: pitches narrower than cols = %d", cols);
  if (rows == 0) return 0;
  const unsigned blocks = (unsigned)((rows + ROWS_MSE - 1) / ROWS_MSE);
  float* part = nullptr;
  if (loss_sum && pg_scratch((size_t)blocks * sizeof(float), stream, &part)) return 1;
  mse_kernel<<<blocks, THREADS, 0, stream>>>(a, ld_a, b, ld_b, rows, cols, g, scale, part, da, ld_da, db, ld_db);
  if (pg_check_launch("pg_mse_mean")) return 1;
  return loss_sum ? pg_sum_partials(part, (int)blocks, 1, 1, 1, 1, loss_sum, stream) : 0;
}
