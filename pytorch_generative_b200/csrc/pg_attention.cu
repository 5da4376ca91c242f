// pg_attention.cu — causal attention core (reference nn/attention.py:147-160).
//
// Layout: q/k/v/o are pixel-major bf16 matrices; image n occupies rows [n*S, (n+1)*S); head h of q/k uses
// columns [h*dk, (h+1)*dk), of v/o columns [h*dv, (h+1)*dv).  Position i may attend to j <= i
// (strict=0, mask_center=False) or j < i (strict=1, mask_center=True; row 0 then has no keys and its
// output is defined as 0, exactly what the reference's NaN -> masked_fill(0) produces).
//
// impl 1 (this section): SIMT kernels, one warp per row — the on-device cross-check used by the tests.
// impl 0: tensor-core kernels (pg_attention_tc.cuh), the product path.  Backward impl 3 (one CTA per key tile for
// dK / dV) names the same tensor-core kernels: on sm_90a the product backward has that structure.
#include <stdlib.h>
#include <type_traits>

#include "../../include/pg_b200.h"
#include "pg_common.cuh"

namespace {

constexpr int MAX_S = 1024;   // per-warp score buffer (floats) in shared memory
constexpr int MAX_D = 128;

struct AttnArgs {
  const bf16 *q, *k, *v, *o, *d_o;
  bf16 *out, *dq, *dk_out, *dv_out;
  int64_t ld_q, ld_k, ld_v, ld_o, ld_do, ld_dq, ld_dk, ld_dv;
  float* lse;
  const float* lse_in;
  float* delta;
  int N, S, H, dk, dv, strict;
  float scale;
};

// One warp per (image, head, query row).
__global__ void __launch_bounds__(128) attn_fwd_simt(const AttnArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* sc = sm + w * (MAX_S + MAX_D);   // scores
  float* qs = sc + MAX_S;                 // the query row
  const long long gw = (long long)blockIdx.x * 4 + w;
  const long long total = (long long)a.N * a.H * a.S;
  if (gw >= total) return;
  const int i = (int)(gw % a.S);
  const int h = (int)((gw / a.S) % a.H);
  const int n = (int)(gw / ((long long)a.S * a.H));
  const size_t row0 = (size_t)n * a.S;
  for (int d = lane; d < a.dk; d += 32) qs[d] = __bfloat162float(a.q[(row0 + i) * a.ld_q + h * a.dk + d]);
  __syncwarp();
  const int nkeys = a.strict ? i : i + 1;
  float m = -INFINITY;
  for (int j = lane; j < nkeys; j += 32) {
    const bf16* kr = a.k + (row0 + j) * a.ld_k + h * a.dk;
    float s = 0.f;
    for (int d = 0; d < a.dk; ++d) s = fmaf(qs[d], __bfloat162float(kr[d]), s);
    s *= a.scale;
    sc[j] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  float l = 0.f;
  for (int j = lane; j < nkeys; j += 32) {
    const float p = __expf(sc[j] - m);
    sc[j] = p;
    l += p;
  }
  l = warp_sum(l);
  __syncwarp();
  const float inv = nkeys > 0 ? 1.f / l : 0.f;
  for (int d = lane; d < a.dv; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < nkeys; ++j) acc = fmaf(sc[j], __bfloat162float(a.v[(row0 + j) * a.ld_v + h * a.dv + d]), acc);
    a.out[(row0 + i) * a.ld_o + h * a.dv + d] = __float2bfloat16(acc * inv);
  }
  if (lane == 0 && a.lse) a.lse[((size_t)n * a.H + h) * a.S + i] = nkeys > 0 ? m + __logf(l) : 0.f;
}

// delta[n,h,i] = sum_d dO[i,d] * O[i,d].  16-byte loads: (dv/8) consecutive lanes cover one (row, head) slot, so a
// warp reads 512 contiguous bytes of each tensor per step.
__global__ void attn_delta_kernel(const AttnArgs a) {
  const int lanes_per = a.dv / 8;  // lanes per (row, head): 8 for dv=64, 16 for dv=128 (dv % 8 == 0, dv <= 256)
  const long long total = (long long)a.N * a.S * a.H * lanes_per;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int sub = (int)(idx % lanes_per);
    const long long rh = idx / lanes_per;
    const int h = (int)(rh % a.H);
    const long long row = rh / a.H;  // n * S + i
    const uint4 x = *reinterpret_cast<const uint4*>(a.d_o + row * a.ld_do + h * a.dv + sub * 8);
    const uint4 y = *reinterpret_cast<const uint4*>(a.o + row * a.ld_o + h * a.dv + sub * 8);
    const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
    float s = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 p = unpack_bf16x2(xw[t]), q = unpack_bf16x2(yw[t]);
      s = fmaf(p.x, q.x, fmaf(p.y, q.y, s));
    }
    // reduce over the lanes_per consecutive lanes of this slot (lanes_per is a power of two <= 32)
    for (int o = lanes_per >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (sub == 0) {
      const int n = (int)(row / a.S), i = (int)(row % a.S);
      a.delta[((size_t)n * a.H + h) * a.S + i] = s;
    }
  }
}

// Generic fallback (any dv): one warp per (row, head).
__global__ void attn_delta_generic_kernel(const AttnArgs a) {
  const int lane = threadIdx.x & 31;
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long total = (long long)a.N * a.H * a.S;
  if (gw >= total) return;
  const int i = (int)(gw % a.S);
  const int h = (int)((gw / a.S) % a.H);
  const int n = (int)(gw / ((long long)a.S * a.H));
  const size_t row = (size_t)n * a.S + i;
  float s = 0.f;
  for (int d = lane; d < a.dv; d += 32)
    s += __bfloat162float(a.d_o[row * a.ld_do + h * a.dv + d]) * __bfloat162float(a.o[row * a.ld_o + h * a.dv + d]);
  s = warp_sum(s);
  if (lane == 0) a.delta[((size_t)n * a.H + h) * a.S + i] = s;
}

// dQ: one warp per query row.
__global__ void __launch_bounds__(128) attn_bwd_dq_simt(const AttnArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* ds = sm + w * (MAX_S + 2 * MAX_D);
  float* qs = ds + MAX_S;
  float* dos = qs + MAX_D;
  const long long gw = (long long)blockIdx.x * 4 + w;
  const long long total = (long long)a.N * a.H * a.S;
  if (gw >= total) return;
  const int i = (int)(gw % a.S);
  const int h = (int)((gw / a.S) % a.H);
  const int n = (int)(gw / ((long long)a.S * a.H));
  const size_t row0 = (size_t)n * a.S;
  for (int d = lane; d < a.dk; d += 32) qs[d] = __bfloat162float(a.q[(row0 + i) * a.ld_q + h * a.dk + d]);
  for (int d = lane; d < a.dv; d += 32) dos[d] = __bfloat162float(a.d_o[(row0 + i) * a.ld_do + h * a.dv + d]);
  __syncwarp();
  const int nkeys = a.strict ? i : i + 1;
  const float lse = a.lse_in[((size_t)n * a.H + h) * a.S + i];
  const float delta = a.delta[((size_t)n * a.H + h) * a.S + i];
  for (int j = lane; j < nkeys; j += 32) {
    const bf16* kr = a.k + (row0 + j) * a.ld_k + h * a.dk;
    const bf16* vr = a.v + (row0 + j) * a.ld_v + h * a.dv;
    float s = 0.f, dp = 0.f;
    for (int d = 0; d < a.dk; ++d) s = fmaf(qs[d], __bfloat162float(kr[d]), s);
    for (int d = 0; d < a.dv; ++d) dp = fmaf(dos[d], __bfloat162float(vr[d]), dp);
    const float p = __expf(s * a.scale - lse);
    ds[j] = p * (dp - delta);
  }
  __syncwarp();
  for (int d = lane; d < a.dk; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < nkeys; ++j) acc = fmaf(ds[j], __bfloat162float(a.k[(row0 + j) * a.ld_k + h * a.dk + d]), acc);
    a.dq[(row0 + i) * a.ld_dq + h * a.dk + d] = __float2bfloat16(acc * a.scale);
  }
}

// dK, dV: one warp per key row j; queries i >= j (i > j when strict).
__global__ void __launch_bounds__(128) attn_bwd_dkv_simt(const AttnArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* ps = sm + w * (2 * MAX_S + 2 * MAX_D);
  float* ds = ps + MAX_S;
  float* ks = ds + MAX_S;
  float* vs = ks + MAX_D;
  const long long gw = (long long)blockIdx.x * 4 + w;
  const long long total = (long long)a.N * a.H * a.S;
  if (gw >= total) return;
  const int j = (int)(gw % a.S);
  const int h = (int)((gw / a.S) % a.H);
  const int n = (int)(gw / ((long long)a.S * a.H));
  const size_t row0 = (size_t)n * a.S;
  for (int d = lane; d < a.dk; d += 32) ks[d] = __bfloat162float(a.k[(row0 + j) * a.ld_k + h * a.dk + d]);
  for (int d = lane; d < a.dv; d += 32) vs[d] = __bfloat162float(a.v[(row0 + j) * a.ld_v + h * a.dv + d]);
  __syncwarp();
  const int i0 = a.strict ? j + 1 : j;
  for (int i = i0 + lane; i < a.S; i += 32) {
    const bf16* qr = a.q + (row0 + i) * a.ld_q + h * a.dk;
    const bf16* dor = a.d_o + (row0 + i) * a.ld_do + h * a.dv;
    float s = 0.f, dp = 0.f;
    for (int d = 0; d < a.dk; ++d) s = fmaf(ks[d], __bfloat162float(qr[d]), s);
    for (int d = 0; d < a.dv; ++d) dp = fmaf(vs[d], __bfloat162float(dor[d]), dp);
    const size_t st = ((size_t)n * a.H + h) * a.S + i;
    const float p = __expf(s * a.scale - a.lse_in[st]);
    ps[i - i0] = p;
    ds[i - i0] = p * (dp - a.delta[st]);
  }
  __syncwarp();
  const int cnt = a.S - i0;
  for (int d = lane; d < a.dv; d += 32) {
    float acc = 0.f;
    for (int t = 0; t < cnt; ++t)
      acc = fmaf(ps[t], __bfloat162float(a.d_o[(row0 + i0 + t) * a.ld_do + h * a.dv + d]), acc);
    a.dv_out[(row0 + j) * a.ld_dv + h * a.dv + d] = __float2bfloat16(acc);
  }
  for (int d = lane; d < a.dk; d += 32) {
    float acc = 0.f;
    for (int t = 0; t < cnt; ++t)
      acc = fmaf(ds[t], __bfloat162float(a.q[(row0 + i0 + t) * a.ld_q + h * a.dk + d]), acc);
    a.dk_out[(row0 + j) * a.ld_dk + h * a.dk + d] = __float2bfloat16(acc * a.scale);
  }
}

// ------------------------------------------------------------------------------------------------
// Incremental (KV-cached) attention for sampling: one new position per image.  One warp per (image, head):
// appends this position's key / value rows to the caches, then attends over cache rows [0, pos] (or [0, pos) when
// strict).  `pos` is read from device memory so that one captured CUDA graph serves every pixel of the raster scan.
// ------------------------------------------------------------------------------------------------
struct DecodeArgs {
  const bf16 *q, *k_new, *v_new;   // [N, H*dk], [N, H*dk], [N, H*dv] rows of the current position
  bf16 *k_cache, *v_cache;         // [N*S, H*dk], [N*S, H*dv]
  bf16* out;                       // [N, H*dv]
  int64_t ld_q, ld_kn, ld_vn, ld_kc, ld_vc, ld_o;
  const int* pos;
  int N, S, H, dk, dv, strict;
  float scale;
  float* part;                     // SPLIT: [N*H*splits] (m, l) pairs, then [N*H*splits, dv] unnormalised outputs
};

// One block (4 warps) per (image, head): the keys are split across the warps, partial (max, sum, output) are merged
// through shared memory.
//
// SPLIT (S > MAX_S, the score buffer cannot hold every key): grid.y = ceil(S / MAX_S) blocks per (image, head), block s
// covering cache rows [s * MAX_S, min((s + 1) * MAX_S, nkeys)).  The grid depends on the cache capacity S only, never on
// pos, so one captured graph serves every position.  Block s writes its unnormalised partial (max m, sum l, output o)
// to `a.part`; a block whose range starts at or after nkeys finds no keys and writes (-inf, 0, 0).  Only the block
// whose range holds pos appends the new key / value row, before its own reads; no other block reads that row.
// attn_decode_merge_kernel combines the partials in split order.
template <bool SPLIT>
__global__ void __launch_bounds__(128) attn_decode_kernel(const DecodeArgs a) {
  __shared__ float sc[MAX_S];
  __shared__ float qs[MAX_D];
  __shared__ float part_o[4][MAX_D];
  __shared__ float part_m[4], part_l[4];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const int pos = *a.pos;
  const size_t row0 = (size_t)n * a.S;
  const int j0 = SPLIT ? (int)blockIdx.y * MAX_S : 0;              // first cache row of this block's range
  const bool append = !SPLIT || pos / MAX_S == (int)blockIdx.y;   // this block's range holds pos
  for (int d = threadIdx.x; d < a.dk; d += 128) {
    if (append) a.k_cache[(row0 + pos) * a.ld_kc + h * a.dk + d] = a.k_new[(size_t)n * a.ld_kn + h * a.dk + d];
    qs[d] = __bfloat162float(a.q[(size_t)n * a.ld_q + h * a.dk + d]);
  }
  if (append)
    for (int d = threadIdx.x; d < a.dv; d += 128)
      a.v_cache[(row0 + pos) * a.ld_vc + h * a.dv + d] = a.v_new[(size_t)n * a.ld_vn + h * a.dv + d];
  __syncthreads();
  // SPLIT: nkeys is the end of this block's range; sc[j - j0] holds key j
  const int nkeys = SPLIT ? min(a.strict ? pos : pos + 1, j0 + MAX_S) : (a.strict ? pos : pos + 1);
  float m = -INFINITY;
  for (int j = j0 + threadIdx.x; j < nkeys; j += 128) {
    const uint4* kr = reinterpret_cast<const uint4*>(a.k_cache + (row0 + j) * a.ld_kc + h * a.dk);
    float s = 0.f;
    for (int d8 = 0; d8 < a.dk / 8; ++d8) {
      const uint4 kv = kr[d8];
      const uint32_t kw[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = unpack_bf16x2(kw[t]);
        s = fmaf(qs[d8 * 8 + 2 * t], f.x, fmaf(qs[d8 * 8 + 2 * t + 1], f.y, s));
      }
    }
    s *= a.scale;
    sc[j - j0] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  if (lane == 0) part_m[w] = m;
  __syncthreads();
  m = fmaxf(fmaxf(part_m[0], part_m[1]), fmaxf(part_m[2], part_m[3]));
  float l = 0.f;
  for (int j = j0 + threadIdx.x; j < nkeys; j += 128) {
    const float p = __expf(sc[j - j0] - m);
    sc[j - j0] = p;
    l += p;
  }
  l = warp_sum(l);
  if (lane == 0) part_l[w] = l;
  __syncthreads();
  l = (part_l[0] + part_l[1]) + (part_l[2] + part_l[3]);
  const float inv = nkeys > 0 ? 1.f / l : 0.f;
  // PV: warp w takes keys w, w+4, ...; lanes over the value channels
  for (int d = lane; d < a.dv; d += 32) {
    float acc = 0.f;
    for (int j = j0 + w; j < nkeys; j += 4)
      acc = fmaf(sc[j - j0], __bfloat162float(a.v_cache[(row0 + j) * a.ld_vc + h * a.dv + d]), acc);
    part_o[w][d] = acc;
  }
  __syncthreads();
  if constexpr (SPLIT) {
    const size_t rec = (size_t)blockIdx.x * gridDim.y + blockIdx.y;
    float* po = a.part + 2 * (size_t)gridDim.x * gridDim.y + rec * a.dv;
    for (int d = threadIdx.x; d < a.dv; d += 128) po[d] = (part_o[0][d] + part_o[1][d]) + (part_o[2][d] + part_o[3][d]);
    if (threadIdx.x == 0) {
      a.part[2 * rec] = m;
      a.part[2 * rec + 1] = l;
    }
  } else {
    for (int d = threadIdx.x; d < a.dv; d += 128)
      a.out[(size_t)n * a.ld_o + h * a.dv + d] =
          __float2bfloat16(((part_o[0][d] + part_o[1][d]) + (part_o[2][d] + part_o[3][d])) * inv);
  }
}

// One block per (image, head): out = sum_s f_s o_s / sum_s f_s l_s with f_s = exp(m_s - max_s m_s), summed in split
// order.  An empty partial (m = -inf, l = o = 0) gets f = exp(-inf) = 0 and adds exactly zero.  The split holding the
// maximum gets f = 1 exactly, so with keys in split 0 only the result has the bits of the one-block kernel.
__global__ void __launch_bounds__(128) attn_decode_merge_kernel(const DecodeArgs a, int splits) {
  const int n = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const float* ml = a.part + (size_t)blockIdx.x * splits * 2;
  const float* po = a.part + 2 * (size_t)gridDim.x * splits + (size_t)blockIdx.x * splits * a.dv;
  const int pos = *a.pos;
  const int nkeys = a.strict ? pos : pos + 1;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, ml[2 * s]);
  for (int d = threadIdx.x; d < a.dv; d += 128) {
    float l = 0.f, acc = 0.f;
    for (int s = 0; s < splits; ++s) {
      const float f = ml[2 * s] == m ? 1.f : __expf(ml[2 * s] - m);
      l = fmaf(ml[2 * s + 1], f, l);
      acc = fmaf(po[(size_t)s * a.dv + d], f, acc);
    }
    a.out[(size_t)n * a.ld_o + h * a.dv + d] = __float2bfloat16(acc * (nkeys > 0 ? 1.f / l : 0.f));
  }
}

}  // namespace

#include "pg_attention_tc.cuh"

extern "C" int pg_causal_attn_fwd(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v,
                                  int64_t ld_v, void* o, int64_t ld_o, float* lse, int N, int S, int H, int dk,
                                  int dv, float scale, int strict, int impl, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(q && k && v && o && lse, "pg_causal_attn_fwd: null argument");
  PG_REQUIRE(N > 0 && S > 0 && H > 0 && dk > 0 && dv > 0, "pg_causal_attn_fwd: empty problem");
  AttnArgs a = {};
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.out = (bf16*)o;
  a.ld_q = ld_q; a.ld_k = ld_k; a.ld_v = ld_v; a.ld_o = ld_o;
  a.lse = lse;
  a.N = N; a.S = S; a.H = H; a.dk = dk; a.dv = dv; a.strict = strict;
  a.scale = scale;
  if (impl == 1) {
    PG_REQUIRE(S <= MAX_S && dk <= MAX_D && dv <= MAX_D, "pg_causal_attn_fwd(simt): S<=%d, d<=%d", MAX_S, MAX_D);
    const long long total = (long long)N * H * S;
    const size_t smem = 4 * (MAX_S + MAX_D) * sizeof(float);
    attn_fwd_simt<<<(unsigned)((total + 3) / 4), 128, smem, stream>>>(a);
    return pg_check_launch("pg_causal_attn_fwd(simt)");
  }
  return attn_fwd_tc(a, stream);
}

extern "C" int pg_causal_attn_bwd(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v,
                                  int64_t ld_v, const void* o, int64_t ld_o, const void* d_o, int64_t ld_do,
                                  const float* lse, float* delta, float* dq_accum, void* dq, int64_t ld_dq, void* dk_,
                                  int64_t ld_dk, void* dv_, int64_t ld_dv, int N, int S, int H, int dk, int dv,
                                  float scale, int strict, int impl, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(q && k && v && o && d_o && lse && delta && dq && dk_ && dv_, "pg_causal_attn_bwd: null argument");
  PG_REQUIRE(N > 0 && S > 0 && H > 0 && dk > 0 && dv > 0, "pg_causal_attn_bwd: empty problem");
  AttnArgs a = {};
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.o = (const bf16*)o; a.d_o = (const bf16*)d_o;
  a.dq = (bf16*)dq; a.dk_out = (bf16*)dk_; a.dv_out = (bf16*)dv_;
  a.ld_q = ld_q; a.ld_k = ld_k; a.ld_v = ld_v; a.ld_o = ld_o; a.ld_do = ld_do;
  a.ld_dq = ld_dq; a.ld_dk = ld_dk; a.ld_dv = ld_dv;
  a.lse_in = lse; a.delta = delta;
  a.N = N; a.S = S; a.H = H; a.dk = dk; a.dv = dv; a.strict = strict;
  a.scale = scale;
  (void)dq_accum;  // kept in the signature; no kernel needs an fp32 dQ accumulator
  const long long total = (long long)N * H * S;
  const int lanes_per = dv / 8;
  const bool pow2 = dv % 8 == 0 && lanes_per >= 1 && lanes_per <= 32 && (lanes_per & (lanes_per - 1)) == 0;
  if (pow2 && ld_o % 8 == 0 && ld_do % 8 == 0 && (total * lanes_per) % 32 == 0) {
    long long blocks = (total * lanes_per + 255) / 256;
    if (blocks > (long long)pg_num_sms() * 32) blocks = (long long)pg_num_sms() * 32;
    attn_delta_kernel<<<(unsigned)blocks, 256, 0, stream>>>(a);
  } else {
    attn_delta_generic_kernel<<<(unsigned)((total * 32 + 255) / 256), 256, 0, stream>>>(a);
  }
  if (pg_check_launch("pg_causal_attn_bwd(delta)")) return 1;
  if (impl == 1) {
    PG_REQUIRE(S <= MAX_S && dk <= MAX_D && dv <= MAX_D, "pg_causal_attn_bwd(simt): S<=%d, d<=%d", MAX_S, MAX_D);
    const size_t smem_q = 4 * (MAX_S + 2 * MAX_D) * sizeof(float);
    const size_t smem_kv = 4 * (2 * MAX_S + 2 * MAX_D) * sizeof(float);
    attn_bwd_dq_simt<<<(unsigned)((total + 3) / 4), 128, smem_q, stream>>>(a);
    if (pg_check_launch("pg_causal_attn_bwd(dq simt)")) return 1;
    attn_bwd_dkv_simt<<<(unsigned)((total + 3) / 4), 128, smem_kv, stream>>>(a);
    return pg_check_launch("pg_causal_attn_bwd(dkv simt)");
  }
  return attn_bwd_tc(a, stream);
}

extern "C" int pg_attn_decode(const void* q, int64_t ld_q, const void* k_new, int64_t ld_kn, const void* v_new, int64_t ld_vn,
                              void* k_cache, int64_t ld_kc, void* v_cache, int64_t ld_vc, void* o, int64_t ld_o,
                              const int* pos_dev, int N, int S, int H, int dk, int dv, float scale, int strict,
                              void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(q && k_new && v_new && k_cache && v_cache && o && pos_dev, "pg_attn_decode: null argument");
  PG_REQUIRE(dk <= MAX_D && dv <= MAX_D, "pg_attn_decode: d<=%d", MAX_D);
  DecodeArgs a;
  a.q = (const bf16*)q; a.k_new = (const bf16*)k_new; a.v_new = (const bf16*)v_new;
  a.k_cache = (bf16*)k_cache; a.v_cache = (bf16*)v_cache; a.out = (bf16*)o;
  a.ld_q = ld_q; a.ld_kn = ld_kn; a.ld_vn = ld_vn; a.ld_kc = ld_kc; a.ld_vc = ld_vc; a.ld_o = ld_o;
  a.pos = pos_dev; a.N = N; a.S = S; a.H = H; a.dk = dk; a.dv = dv; a.strict = strict; a.scale = scale;
  a.part = nullptr;
  PG_REQUIRE(dk % 8 == 0 && ld_kc % 8 == 0, "pg_attn_decode: dk and the cache pitch must be multiples of 8");
  if (S <= MAX_S) {
    attn_decode_kernel<false><<<N * H, 128, 0, stream>>>(a);
    return pg_check_launch("pg_attn_decode");
  }
  // Longer caches: one block per MAX_S keys, then the fixed-order merge.  The scratch size depends on S, not on pos,
  // so the sampler's warm-up step sizes it before its graph capture.
  const int splits = (S + MAX_S - 1) / MAX_S;
  if (pg_scratch((size_t)N * H * splits * (2 + dv) * sizeof(float), stream, &a.part)) return 1;
  attn_decode_kernel<true><<<dim3(N * H, splits), 128, 0, stream>>>(a);
  if (pg_check_launch("pg_attn_decode(split)")) return 1;
  attn_decode_merge_kernel<<<N * H, 128, 0, stream>>>(a, splits);
  return pg_check_launch("pg_attn_decode(merge)");
}
