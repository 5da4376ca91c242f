// pg_attention_tc.cuh — causal attention on sm_90a wgmma tensor cores (included by pg_attention.cu).
//
// Head slots are 64 or 128 columns wide, for q/k (DK) and for v/o (DV) independently; narrower heads are zero padded
// by the caller.  Every kernel has the four <DK, DV> instances.  All operands arrive by TMA (3-D maps [N][S][cols], so
// rows past the end of an image are zero-filled) into 128B-swizzled shared memory and are read in place by wgmma
// under two views of the same bytes: a [rows][64-col swizzle atom] tile is a K-major operand with K along the
// columns, or an MN-major operand with K along the rows.  A 128-wide slot is two such atoms per row, one TMA load
// each; MMA K loops over dk or dv step through the atoms in order.
//
// Every kernel runs three warpgroups (384 threads), as the GEMM does.  Warp 0 of the first is the producer: it issues
// every TMA load, running ahead of the consumers by the depth of the ring (2-4 stages, as many as fit in shared
// memory), and it is the only warp that waits for a stage to be released; the warpgroup gives its registers to the
// two consumer warpgroups (`setmaxnreg`, 24 / 240).  The consumers take turns issuing the first MMA group of an
// iteration (S, and dP in the backward), handing the turn over with named barriers as soon as the group is issued, so
// one warpgroup's MMAs run on the tensor cores while the other does its exp2 / rescale / dS arithmetic.  The schedule
// decides when an MMA runs, not which MMAs an output element sees or in what order, so it changes no bits.
// Forward, one CTA per (image, head, 128-query tile), Q once, K / V tiles of 128 keys:
//   warpgroups 0, 1  64 query rows each: S = Q K^T into registers, online softmax on the accumulator fragments
//                 (a row is spread over the four threads of a quad), O += P V with P as the register A operand.
//                 Only the diagonal tile runs the masked code path.
// Backward dK / dV, one CTA per (image, head, 128-key tile), K / V once, looping over the 64-query tiles i (Q_i, dO_i)
// that see those keys:
//   warpgroups 0, 1  64 keys each: S^T = K Q_i^T, dP^T = V dO_i^T -> P^T = exp2(S^T c - lse),
//                 dS^T = P^T (dP^T - delta); dV += P^T dO_i and dK += dS^T Q_i with P^T / dS^T as register A operands.
//                 lse (times log2 e) and delta of the 64 queries come with the stage: the producer warp writes them to
//                 shared memory before it arms the stage's barrier, so the loop reads no global memory.
// Backward dQ, one CTA per (image, head, 128-query tile), Q / dO once, K / V tiles of 128 keys: S and dP recomputed
//   in registers, dQ += dS K with dS as the register A operand.  With DK = 128 the 64-float dQ accumulator leaves no
//   room for S / dP over 128 keys, so each tile is walked as two 64-key halves in order.  Each dQ element is summed by
//   one thread in key order (no atomics), so the backward gives the same bits on every run.
#pragma once

namespace {

constexpr int AT = 128;              // tile edge: queries (forward), keys (backward)
constexpr int ATOM_BYTES = AT * 128; // one 64-column swizzle atom of a 128-row tile
constexpr int BQ = 64;               // query tile of the backward
constexpr int QATOM_BYTES = BQ * 128;
constexpr int ATTN_THREADS = 384;    // the producer's warpgroup and two consumer warpgroups
constexpr int ATTN_PRODUCER_REGS = 24, ATTN_CONSUMER_REGS = 240;  // 128 x 24 + 256 x 240 <= 64 K registers
constexpr int ATTN_SMEM_LIMIT = 227 * 1024;
constexpr int ATTN_BAR_BYTES = 128;  // 1 + 2 x 4 mbarriers, padded
constexpr int ATTN_TURN_BAR = 1;     // named barriers 1 and 2: consumer warpgroup wg may issue its MMAs

// Ring depth of an instance: the stages that fit next to `fixed` bytes of single-buffered tiles, four at most (the
// producer is never more than a few tiles ahead of a consumer that keeps up).
constexpr int attn_stages(int fixed, int stage) {
  const int fit = (ATTN_SMEM_LIMIT - ATTN_BAR_BYTES - fixed) / stage;
  return fit < 4 ? fit : 4;
}

// The consumers' turns.  Warpgroup 0 goes first and warpgroup 1 does not hand back after its last iteration, so every
// arrival is matched by a wait.
__device__ __forceinline__ void attn_turn_wait(int wg, int it) {
  if (wg | it) named_bar_sync(ATTN_TURN_BAR + wg, 256);
}
__device__ __forceinline__ void attn_turn_pass(int wg, int it, int niter) {
  if (wg == 0 || it + 1 < niter) named_bar_arrive(ATTN_TURN_BAR + (wg ^ 1), 256);
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

struct AttnTmaps {
  CUtensorMap q, k, v, d_o;
};

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
template <int DK, int DV>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_fwd_tc_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a, const int T) {
  constexpr int K_BYTES = DK * 256;  // [128 rows][DK]: the Q tile and a K tile, DK / 64 swizzle atoms
  constexpr int V_BYTES = DV * 256;
  constexpr int ST = attn_stages(K_BYTES, K_BYTES + V_BYTES);
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + K_BYTES;             // ST stages
  uint8_t* sV = sK + ST * K_BYTES;        // ST stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * V_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;        // [ST]
  uint64_t* kv_empty = bars + 1 + ST;  // [ST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // consecutive blocks = the query tiles of one (image, head), longest first: co-resident CTAs then share the K / V
  // of a few (image, head) pairs through L2 instead of every query tile streaming its keys from HBM
  const int nh = blockIdx.x / T;
  const int i = T - 1 - blockIdx.x % T;
  const int n = nh / a.H, h = nh % a.H;
  const int ntiles = i + 1;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();  // 128B swizzle atoms need a 1024-byte aligned base
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<ATTN_PRODUCER_REGS>();
    if (warp == 0) {
      // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
      mbar_arrive_expect_tx_w(q_full, K_BYTES);
#pragma unroll
      for (int c = 0; c < DK / 64; ++c) tma_load_3d_w(sQ + c * ATOM_BYTES, &tm.q, q_full, h * DK + c * 64, i * AT, n);
      // K / V tile jj into stage jj % ST once the tile that used the stage before has been released by all eight
      // consumer warps
      for (int jj = 0; jj < ntiles; ++jj) {
        const int st = jj % ST;
        mbar_wait(&kv_empty[st], ((jj / ST) & 1) ^ 1);
        mbar_arrive_expect_tx_w(&kv_full[st], K_BYTES + V_BYTES);
#pragma unroll
        for (int c = 0; c < DK / 64; ++c)
          tma_load_3d_w(sK + st * K_BYTES + c * ATOM_BYTES, &tm.k, &kv_full[st], h * DK + c * 64, jj * AT, n);
#pragma unroll
        for (int v = 0; v < DV / 64; ++v)
          tma_load_3d_w(sV + st * V_BYTES + v * ATOM_BYTES, &tm.v, &kv_full[st], h * DV + v * 64, jj * AT, n);
      }
    }
  } else {
    setmaxnreg_inc<ATTN_CONSUMER_REGS>();
    // ===================== consumers: thread holds query rows r0 and r0 + 8 of the tile =====================
    const int wg = (warp >> 2) - 1;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int qi0 = i * AT + r0, qi1 = qi0 + 8;
    const int qlim0 = qi0 - a.strict, qlim1 = qi1 - a.strict;  // keys kj <= qlim are visible
    const float sl2 = a.scale * 1.4426950408889634f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float O[DV / 2];
#pragma unroll
    for (int d = 0; d < DV / 2; ++d) O[d] = 0.f;
    float S[64];
    const uint64_t q_d = wgmma_desc_sw128(smem_u32(sQ) + wg * 64 * 128, 16, 1024);
    mbar_wait(q_full, 0);
    for (int j = 0; j < ntiles; ++j) {
      const int st = j % ST;
      mbar_wait(&kv_full[st], (j / ST) & 1);
      const uint64_t k_d = wgmma_desc_sw128(smem_u32(sK + st * K_BYTES), 16, 1024);
      attn_turn_wait(wg, j);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DK / 16; ++kk) {  // K = dk: 4 steps of 32 B per 64-column atom (descriptor units of 16 B)
        const int off = (kk >> 2) * (ATOM_BYTES >> 4) + (kk & 3) * 2;
        Wgmma<128>::ss<0, 0>(S, q_d + off, k_d + off, kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      attn_turn_pass(wg, j, ntiles);
      wgmma_wait<0>();
      wgmma_hold(S);
      if (j == i) {  // diagonal tile: causal mask (also hides keys past the end of the image)
        const int k0 = j * AT + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kj = k0 + 8 * jj + e;
            if (kj > qlim0) S[4 * jj + e] = -INFINITY;
            if (kj > qlim1) S[4 * jj + 2 + e] = -INFINITY;
          }
        }
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        mx0 = fmaxf(mx0, fmaxf(S[4 * jj], S[4 * jj + 1]));
        mx1 = fmaxf(mx1, fmaxf(S[4 * jj + 2], S[4 * jj + 3]));
      }
      mx0 = quad_max(mx0);
      mx1 = quad_max(mx1);
      const float mu0 = (mx0 == -INFINITY) ? 0.f : mx0, mu1 = (mx1 == -INFINITY) ? 0.f : mx1;
      const float alpha0 = fast_exp2((m0 - mu0) * sl2), alpha1 = fast_exp2((m1 - mu1) * sl2);  // m = -inf -> 0
      const float mb0 = mu0 * sl2, mb1 = mu1 * sl2;
      float lt0 = 0.f, lt1 = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        S[4 * jj] = fast_exp2(fmaf(S[4 * jj], sl2, -mb0));
        S[4 * jj + 1] = fast_exp2(fmaf(S[4 * jj + 1], sl2, -mb0));
        S[4 * jj + 2] = fast_exp2(fmaf(S[4 * jj + 2], sl2, -mb1));
        S[4 * jj + 3] = fast_exp2(fmaf(S[4 * jj + 3], sl2, -mb1));
        lt0 += S[4 * jj] + S[4 * jj + 1];
        lt1 += S[4 * jj + 2] + S[4 * jj + 3];
      }
      l0 = l0 * alpha0 + lt0;  // per-thread partial sums; the quad's four are added at the end
      l1 = l1 * alpha1 + lt1;
      m0 = mx0;
      m1 = mx1;
#pragma unroll
      for (int d = 0; d < DV / 8; ++d) {
        O[4 * d] *= alpha0; O[4 * d + 1] *= alpha0;
        O[4 * d + 2] *= alpha1; O[4 * d + 3] *= alpha1;
      }
      uint32_t pa[8][4];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_frag_a(S, kk, pa[kk]);
      const uint64_t v_d = wgmma_desc_sw128(smem_u32(sV + st * V_BYTES), ATOM_BYTES, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) Wgmma<DV>::template rs<1>(O, pa[kk], v_d + kk * 128, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(O);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);  // this warp's reads of the K / V stage are done
    }
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int qi = half ? qi1 : qi0;
      const float l = half ? l1 : l0, m = half ? m1 : m0;
      if (qi < a.S) {
        const float inv = l > 0.f ? 1.f / l : 0.f;
        bf16* orow = a.out + ((size_t)n * a.S + qi) * a.ld_o + h * DV + 2 * (lane & 3);
#pragma unroll
        for (int d = 0; d < DV / 8; ++d)
          *reinterpret_cast<uint32_t*>(orow + 8 * d) = pack_bf16x2(O[4 * d + 2 * half] * inv, O[4 * d + 2 * half + 1] * inv);
        if ((lane & 3) == 0) a.lse[((size_t)n * a.H + h) * a.S + qi] = l > 0.f ? m * a.scale + __logf(l) : 0.f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward
// ------------------------------------------------------------------------------------------------
template <int DK, int DV>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_bwd_tc_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a, const int T) {
  constexpr int K_BYTES = DK * 256;   // [128 keys][DK]
  constexpr int V_BYTES = DV * 256;   // [128 keys][DV]
  constexpr int Q_BYTES = DK * 128;   // [64 queries][DK]
  constexpr int DO_BYTES = DV * 128;  // [64 queries][DV]
  constexpr int STAT_BYTES = 2 * BQ * 4;  // lse log2 e and delta of the stage's queries
  constexpr int ST = attn_stages(K_BYTES + V_BYTES, Q_BYTES + DO_BYTES + STAT_BYTES);
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sK = smem;
  uint8_t* sV = sK + K_BYTES;
  uint8_t* sQ = sV + V_BYTES;             // ST stages
  uint8_t* sdO = sQ + ST * Q_BYTES;       // ST stages
  float* sStat = reinterpret_cast<float*>(sdO + ST * DO_BYTES);  // ST stages of [2][BQ]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStat + ST * 2 * BQ);
  uint64_t* kv_full = bars;
  uint64_t* qdo_full = bars + 1;        // [ST]
  uint64_t* qdo_empty = bars + 1 + ST;  // [ST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nh = blockIdx.x % (a.N * a.H);
  const int j = blockIdx.x / (a.N * a.H);  // key tile; small j = most query tiles = scheduled first
  const int n = nh / a.H, h = nh % a.H;
  const int it0 = j * (AT / BQ);           // first query tile that sees key tile j
  const int niter = (a.S + BQ - 1) / BQ - it0;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();  // 128B swizzle atoms need a 1024-byte aligned base
    mbar_init(kv_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&qdo_full[s], 1);
      mbar_init(&qdo_empty[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<ATTN_PRODUCER_REGS>();
    if (warp == 0) {
      // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
      mbar_arrive_expect_tx_w(kv_full, K_BYTES + V_BYTES);
#pragma unroll
      for (int c = 0; c < DK / 64; ++c) tma_load_3d_w(sK + c * ATOM_BYTES, &tm.k, kv_full, h * DK + c * 64, j * AT, n);
#pragma unroll
      for (int v = 0; v < DV / 64; ++v) tma_load_3d_w(sV + v * ATOM_BYTES, &tm.v, kv_full, h * DV + v * 64, j * AT, n);
      const float* lse_nh = a.lse_in + ((size_t)n * a.H + h) * a.S;
      const float* delta_nh = a.delta + ((size_t)n * a.H + h) * a.S;
      // Q / dO tile `it` into stage it % ST once all eight consumer warps released the stage
      for (int it = 0; it < niter; ++it) {
        const int st = it % ST, i = it0 + it;
        // the tile's statistics, two queries a lane (zero past the end of the image): written by the lanes before the
        // elected one arms the barrier, so a consumer that sees the stage full sees them too
        const int qa = i * BQ + lane, qb = qa + 32;
        const float lse_a = qa < a.S ? lse_nh[qa] * 1.4426950408889634f : 0.f;
        const float lse_b = qb < a.S ? lse_nh[qb] * 1.4426950408889634f : 0.f;
        const float delta_a = qa < a.S ? delta_nh[qa] : 0.f, delta_b = qb < a.S ? delta_nh[qb] : 0.f;
        mbar_wait(&qdo_empty[st], ((it / ST) & 1) ^ 1);
        float* stat = sStat + st * 2 * BQ;
        stat[lane] = lse_a;
        stat[lane + 32] = lse_b;
        stat[BQ + lane] = delta_a;
        stat[BQ + lane + 32] = delta_b;
        __syncwarp();
        mbar_arrive_expect_tx_w(&qdo_full[st], Q_BYTES + DO_BYTES);
#pragma unroll
        for (int c = 0; c < DK / 64; ++c)
          tma_load_3d_w(sQ + st * Q_BYTES + c * QATOM_BYTES, &tm.q, &qdo_full[st], h * DK + c * 64, i * BQ, n);
#pragma unroll
        for (int v = 0; v < DV / 64; ++v)
          tma_load_3d_w(sdO + st * DO_BYTES + v * QATOM_BYTES, &tm.d_o, &qdo_full[st], h * DV + v * 64, i * BQ, n);
      }
    }
  } else {
    setmaxnreg_inc<ATTN_CONSUMER_REGS>();
    // ===================== consumers: thread holds key rows kr and kr + 8 of the tile =====================
    const int wg = (warp >> 2) - 1, wi = warp & 3;
    const int kr = wg * 64 + wi * 16 + (lane >> 2);
    const int kj0 = j * AT + kr, kj1 = kj0 + 8;
    const float sl2 = a.scale * 1.4426950408889634f;
    float dV[DV / 2], dK[DK / 2];
#pragma unroll
    for (int d = 0; d < DV / 2; ++d) dV[d] = 0.f;
#pragma unroll
    for (int d = 0; d < DK / 2; ++d) dK[d] = 0.f;
    const uint32_t k_rows = smem_u32(sK) + wg * 64 * 128;  // this warpgroup's 64 keys
    const uint32_t v_rows = smem_u32(sV) + wg * 64 * 128;
    mbar_wait(kv_full, 0);
    for (int it = 0; it < niter; ++it) {
      const int st = it % ST;
      const int q0 = (it0 + it) * BQ;
      mbar_wait(&qdo_full[st], (it / ST) & 1);
      const uint32_t q_addr = smem_u32(sQ + st * Q_BYTES), do_addr = smem_u32(sdO + st * DO_BYTES);
      const float* stat = sStat + st * 2 * BQ + 2 * (lane & 3);
      float sT[32], dpT[32];
      attn_turn_wait(wg, it);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DK / 16; ++kk)  // S^T = K Q^T: M = keys, N = queries, K = dk, in 64-column atoms
        Wgmma<64>::ss<0, 0>(sT, wgmma_desc_sw128(k_rows + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                            wgmma_desc_sw128(q_addr + (kk >> 2) * QATOM_BYTES + (kk & 3) * 32, 16, 1024),
                            kk > 0 ? 1u : 0u);
#pragma unroll
      for (int kk = 0; kk < DV / 16; ++kk)  // dP^T = V dO^T: K = dv, in 64-column atoms
        Wgmma<64>::ss<0, 0>(dpT, wgmma_desc_sw128(v_rows + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                            wgmma_desc_sw128(do_addr + (kk >> 2) * QATOM_BYTES + (kk & 3) * 32, 16, 1024),
                            kk > 0 ? 1u : 0u);
      wgmma_commit();
      attn_turn_pass(wg, it, niter);
      wgmma_wait<0>();
      wgmma_hold(sT);
      wgmma_hold(dpT);
      // column jj*8 + 2*(lane%4) + e of the fragments is query q0 + that column
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float2 lse2_pair = *reinterpret_cast<const float2*>(stat + 8 * jj);
        const float2 delta_pair = *reinterpret_cast<const float2*>(stat + BQ + 8 * jj);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qi = q0 + 8 * jj + 2 * (lane & 3) + e;
          const float lse2 = e ? lse2_pair.y : lse2_pair.x, delta = e ? delta_pair.y : delta_pair.x;
          const int qlim = qi < a.S ? qi - a.strict : -1;  // keys kj <= qlim see this query; invalid queries see none
          const float p0 = kj0 <= qlim ? fast_exp2(fmaf(sT[4 * jj + e], sl2, -lse2)) : 0.f;
          const float p1 = kj1 <= qlim ? fast_exp2(fmaf(sT[4 * jj + 2 + e], sl2, -lse2)) : 0.f;
          sT[4 * jj + e] = p0;
          sT[4 * jj + 2 + e] = p1;
          dpT[4 * jj + e] = p0 * (dpT[4 * jj + e] - delta);
          dpT[4 * jj + 2 + e] = p1 * (dpT[4 * jj + 2 + e] - delta);
        }
      }
      uint32_t pa[4][4], dsa[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        wgmma_frag_a(sT, kk, pa[kk]);
        wgmma_frag_a(dpT, kk, dsa[kk]);
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)  // dV += P^T dO: K = queries (rows of dO), N = dv
        Wgmma<DV>::template rs<1>(dV, pa[kk], wgmma_desc_sw128(do_addr + kk * 2048, QATOM_BYTES, 1024), 1u);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)  // dK += dS^T Q: N = dk
        Wgmma<DK>::template rs<1>(dK, dsa[kk], wgmma_desc_sw128(q_addr + kk * 2048, QATOM_BYTES, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(dV);
      wgmma_hold(dK);
      __syncwarp();
      if (lane == 0) mbar_arrive(&qdo_empty[st]);  // this warp's reads of the Q / dO stage are done
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int kj = half ? kj1 : kj0;
      if (kj < a.S) {
        bf16* dvrow = a.dv_out + ((size_t)n * a.S + kj) * a.ld_dv + h * DV + 2 * (lane & 3);
#pragma unroll
        for (int d = 0; d < DV / 8; ++d)
          *reinterpret_cast<uint32_t*>(dvrow + 8 * d) = pack_bf16x2(dV[4 * d + 2 * half], dV[4 * d + 2 * half + 1]);
        bf16* dkrow = a.dk_out + ((size_t)n * a.S + kj) * a.ld_dk + h * DK + 2 * (lane & 3);
#pragma unroll
        for (int d = 0; d < DK / 8; ++d)
          *reinterpret_cast<uint32_t*>(dkrow + 8 * d) =
              pack_bf16x2(dK[4 * d + 2 * half] * a.scale, dK[4 * d + 2 * half + 1] * a.scale);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward dQ
// ------------------------------------------------------------------------------------------------
template <int DK, int DV>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_dq_tc_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a, const int T) {
  constexpr int K_BYTES = DK * 256;  // [128 rows][DK]: a K tile, and the Q tile
  constexpr int V_BYTES = DV * 256;  // [128 rows][DV]: a V tile, and the dO tile of the 128 queries
  // keys per S / dP pass: a 128-wide dQ accumulator leaves room for the S / dP fragments of 64 keys only
  constexpr int KS = DK == 64 ? AT : 64;
  constexpr int ST = attn_stages(K_BYTES + V_BYTES, K_BYTES + V_BYTES);
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sdO = sQ + K_BYTES;
  uint8_t* sK = sdO + V_BYTES;            // ST stages
  uint8_t* sV = sK + ST * K_BYTES;        // ST stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * V_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;        // [ST]
  uint64_t* kv_empty = bars + 1 + ST;  // [ST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nh = blockIdx.x / T;
  const int i = T - 1 - blockIdx.x % T;  // longest first, as in the forward
  const int n = nh / a.H, h = nh % a.H;
  const int ntiles = i + 1;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();  // 128B swizzle atoms need a 1024-byte aligned base
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<ATTN_PRODUCER_REGS>();
    if (warp == 0) {  // TMA producer, as in the forward
      mbar_arrive_expect_tx_w(q_full, K_BYTES + V_BYTES);
#pragma unroll
      for (int c = 0; c < DK / 64; ++c) tma_load_3d_w(sQ + c * ATOM_BYTES, &tm.q, q_full, h * DK + c * 64, i * AT, n);
#pragma unroll
      for (int v = 0; v < DV / 64; ++v) tma_load_3d_w(sdO + v * ATOM_BYTES, &tm.d_o, q_full, h * DV + v * 64, i * AT, n);
      for (int jj = 0; jj < ntiles; ++jj) {
        const int st = jj % ST;
        mbar_wait(&kv_empty[st], ((jj / ST) & 1) ^ 1);
        mbar_arrive_expect_tx_w(&kv_full[st], K_BYTES + V_BYTES);
#pragma unroll
        for (int c = 0; c < DK / 64; ++c)
          tma_load_3d_w(sK + st * K_BYTES + c * ATOM_BYTES, &tm.k, &kv_full[st], h * DK + c * 64, jj * AT, n);
#pragma unroll
        for (int v = 0; v < DV / 64; ++v)
          tma_load_3d_w(sV + st * V_BYTES + v * ATOM_BYTES, &tm.v, &kv_full[st], h * DV + v * 64, jj * AT, n);
      }
    }
  } else {
    setmaxnreg_inc<ATTN_CONSUMER_REGS>();
    // thread holds query rows r0 and r0 + 8 of the tile
    const int wg = (warp >> 2) - 1;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int qi0 = i * AT + r0, qi1 = qi0 + 8;
    const size_t stat_base = ((size_t)n * a.H + h) * a.S;
    const float sl2 = a.scale * 1.4426950408889634f;
    // rows past the end of the image see no keys (their results are not stored)
    const int qlim0 = qi0 < a.S ? qi0 - a.strict : -1, qlim1 = qi1 < a.S ? qi1 - a.strict : -1;
    const float lse0 = qi0 < a.S ? a.lse_in[stat_base + qi0] * 1.4426950408889634f : 0.f;
    const float lse1 = qi1 < a.S ? a.lse_in[stat_base + qi1] * 1.4426950408889634f : 0.f;
    const float delta0 = qi0 < a.S ? a.delta[stat_base + qi0] : 0.f;
    const float delta1 = qi1 < a.S ? a.delta[stat_base + qi1] : 0.f;
    float dQ[DK / 2];
#pragma unroll
    for (int d = 0; d < DK / 2; ++d) dQ[d] = 0.f;
    const uint32_t q_rows = smem_u32(sQ) + wg * 64 * 128, do_rows = smem_u32(sdO) + wg * 64 * 128;
    mbar_wait(q_full, 0);
    for (int j = 0; j < ntiles; ++j) {
      const int st = j % ST;
      mbar_wait(&kv_full[st], (j / ST) & 1);
      const uint32_t k_tile = smem_u32(sK + st * K_BYTES), v_tile = smem_u32(sV + st * V_BYTES);
#pragma unroll
      for (int ks = 0; ks < AT / KS; ++ks) {  // key sub-tiles in order
        const uint32_t k_addr = k_tile + ks * KS * 128, v_addr = v_tile + ks * KS * 128;
        float S[KS / 2], dP[KS / 2];
        attn_turn_wait(wg, j * (AT / KS) + ks);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DK / 16; ++kk)  // S = Q K^T: K = dk, in 64-column atoms
          Wgmma<KS>::template ss<0, 0>(S, wgmma_desc_sw128(q_rows + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                                       wgmma_desc_sw128(k_addr + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                                       kk > 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < DV / 16; ++kk)  // dP = dO V^T: K = dv, in 64-column atoms
          Wgmma<KS>::template ss<0, 0>(dP, wgmma_desc_sw128(do_rows + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                                       wgmma_desc_sw128(v_addr + (kk >> 2) * ATOM_BYTES + (kk & 3) * 32, 16, 1024),
                                       kk > 0 ? 1u : 0u);
        wgmma_commit();
        attn_turn_pass(wg, j * (AT / KS) + ks, ntiles * (AT / KS));
        wgmma_wait<0>();
        wgmma_hold(S);
        wgmma_hold(dP);
        const int k0 = j * AT + ks * KS + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < KS / 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kj = k0 + 8 * jj + e;
            const float p0 = kj <= qlim0 ? fast_exp2(fmaf(S[4 * jj + e], sl2, -lse0)) : 0.f;
            const float p1 = kj <= qlim1 ? fast_exp2(fmaf(S[4 * jj + 2 + e], sl2, -lse1)) : 0.f;
            dP[4 * jj + e] = p0 * (dP[4 * jj + e] - delta0);
            dP[4 * jj + 2 + e] = p1 * (dP[4 * jj + 2 + e] - delta1);
          }
        }
        uint32_t dsa[KS / 16][4];
#pragma unroll
        for (int kk = 0; kk < KS / 16; ++kk) wgmma_frag_a(dP, kk, dsa[kk]);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KS / 16; ++kk)  // dQ += dS K: K = keys (rows of the K tile), N = dk
          Wgmma<DK>::template rs<1>(dQ, dsa[kk], wgmma_desc_sw128(k_addr + kk * 2048, ATOM_BYTES, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_hold(dQ);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);  // this warp's reads of the K / V stage are done
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int qi = half ? qi1 : qi0;
      if (qi < a.S) {
        bf16* drow = a.dq + ((size_t)n * a.S + qi) * a.ld_dq + h * DK + 2 * (lane & 3);
#pragma unroll
        for (int d = 0; d < DK / 8; ++d)
          *reinterpret_cast<uint32_t*>(drow + 8 * d) =
              pack_bf16x2(dQ[4 * d + 2 * half] * a.scale, dQ[4 * d + 2 * half + 1] * a.scale);
      }
    }
  }
}

int make_attn_map(CUtensorMap* out, const bf16* base, int64_t ld, int width, int S, int N, int rows) {
  uint64_t dims[3] = {(uint64_t)width, (uint64_t)S, (uint64_t)N};
  uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)S * (uint64_t)ld * 2};
  uint32_t box[3] = {64, (uint32_t)rows, 1};
  return pg_make_tmap_nd_bf16(out, base, 3, dims, strides, box, 1);
}

int attn_check_tc(const AttnArgs& a, const char* who) {
  PG_REQUIRE(a.dk == 64 || a.dk == 128, "%s: tensor-core path needs q/k head slots of 64 or 128 columns (dk=%d)", who,
             a.dk);
  PG_REQUIRE(a.dv == 64 || a.dv == 128, "%s: tensor-core path needs v head slots of 64 or 128 columns (dv=%d)", who,
             a.dv);
  return 0;
}

// Dynamic shared memory of each instance (<DK, DV>) with its ring depth (attn_stages), 128 bytes of mbarriers
// included; the opt-in limit is 227 KB.
//   forward  Q + stages of (K, V)            <64,64> 4: 144 KB   <64,128> 4: 208 KB   <128,64> 4: 224 KB   <128,128> 3: 224 KB
//   dK / dV  K + V + stages of (Q_i, dO_i,   <64,64> 4:  98 KB   <64,128> 4: 146 KB   <128,64> 4: 146 KB   <128,128> 4: 194 KB
//            512 B of lse and delta)
//   dQ       Q + dO + stages of (K, V)       <64,64> 4: 160 KB   <64,128> 3: 192 KB   <128,64> 3: 192 KB   <128,128> 2: 192 KB
template <int DK, int DV>
int launch_fwd(const AttnTmaps& tm, const AttnArgs& a, int T, unsigned grid, cudaStream_t stream) {
  constexpr int SMEM = DK * 256 + attn_stages(DK * 256, (DK + DV) * 256) * (DK + DV) * 256 + ATTN_BAR_BYTES;
  static_assert(SMEM <= ATTN_SMEM_LIMIT, "attn_fwd_tc_kernel: shared memory");
  PG_CUDA(cudaFuncSetAttribute(attn_fwd_tc_kernel<DK, DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  attn_fwd_tc_kernel<DK, DV><<<grid, ATTN_THREADS, SMEM, stream>>>(tm, a, T);
  return 0;
}
template <int DK, int DV>
int launch_bwd(const AttnTmaps& tm, const AttnArgs& a, int T, unsigned grid, cudaStream_t stream) {
  constexpr int STAGE = (DK + DV) * 128 + 2 * BQ * 4;
  constexpr int SMEM = (DK + DV) * 256 + attn_stages((DK + DV) * 256, STAGE) * STAGE + ATTN_BAR_BYTES;
  static_assert(SMEM <= ATTN_SMEM_LIMIT, "attn_bwd_tc_kernel: shared memory");
  PG_CUDA(cudaFuncSetAttribute(attn_bwd_tc_kernel<DK, DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  attn_bwd_tc_kernel<DK, DV><<<grid, ATTN_THREADS, SMEM, stream>>>(tm, a, T);
  return 0;
}
template <int DK, int DV>
int launch_dq(const AttnTmaps& tm, const AttnArgs& a, int T, unsigned grid, cudaStream_t stream) {
  constexpr int SMEM = (1 + attn_stages((DK + DV) * 256, (DK + DV) * 256)) * (DK + DV) * 256 + ATTN_BAR_BYTES;
  static_assert(SMEM <= ATTN_SMEM_LIMIT, "attn_dq_tc_kernel: shared memory");
  PG_CUDA(cudaFuncSetAttribute(attn_dq_tc_kernel<DK, DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  attn_dq_tc_kernel<DK, DV><<<grid, ATTN_THREADS, SMEM, stream>>>(tm, a, T);
  return 0;
}

// the four instances of a kernel, indexed [dk == 128][dv == 128]
using AttnLaunch = int (*)(const AttnTmaps&, const AttnArgs&, int, unsigned, cudaStream_t);
constexpr AttnLaunch kFwd[2][2] = {{launch_fwd<64, 64>, launch_fwd<64, 128>}, {launch_fwd<128, 64>, launch_fwd<128, 128>}};
constexpr AttnLaunch kBwd[2][2] = {{launch_bwd<64, 64>, launch_bwd<64, 128>}, {launch_bwd<128, 64>, launch_bwd<128, 128>}};
constexpr AttnLaunch kDq[2][2] = {{launch_dq<64, 64>, launch_dq<64, 128>}, {launch_dq<128, 64>, launch_dq<128, 128>}};

int attn_fwd_tc(const AttnArgs& a, cudaStream_t stream) {
  if (attn_check_tc(a, "pg_causal_attn_fwd")) return 1;
  PG_REQUIRE(a.ld_o % 8 == 0, "pg_causal_attn_fwd: output pitch must be a multiple of 8");
  AttnTmaps tm;
  if (make_attn_map(&tm.q, a.q, a.ld_q, a.H * a.dk, a.S, a.N, AT)) return 1;
  if (make_attn_map(&tm.k, a.k, a.ld_k, a.H * a.dk, a.S, a.N, AT)) return 1;
  if (make_attn_map(&tm.v, a.v, a.ld_v, a.H * a.dv, a.S, a.N, AT)) return 1;
  tm.d_o = tm.v;
  const int T = (a.S + AT - 1) / AT;
  const unsigned grid = (unsigned)(a.N * a.H * T);
  if (kFwd[a.dk == 128][a.dv == 128](tm, a, T, grid, stream)) return 1;
  return pg_check_launch("pg_causal_attn_fwd(wgmma)");
}

int attn_bwd_tc(const AttnArgs& a, cudaStream_t stream) {
  if (attn_check_tc(a, "pg_causal_attn_bwd")) return 1;
  PG_REQUIRE(a.ld_dq % 8 == 0 && a.ld_dk % 8 == 0 && a.ld_dv % 8 == 0, "pg_causal_attn_bwd: pitches must be multiples of 8");
  AttnTmaps tm;
  if (make_attn_map(&tm.q, a.q, a.ld_q, a.H * a.dk, a.S, a.N, BQ)) return 1;
  if (make_attn_map(&tm.k, a.k, a.ld_k, a.H * a.dk, a.S, a.N, AT)) return 1;
  if (make_attn_map(&tm.v, a.v, a.ld_v, a.H * a.dv, a.S, a.N, AT)) return 1;
  if (make_attn_map(&tm.d_o, a.d_o, a.ld_do, a.H * a.dv, a.S, a.N, BQ)) return 1;
  const int T = (a.S + AT - 1) / AT;
  const unsigned grid = (unsigned)(a.N * a.H * T);
  if (kBwd[a.dk == 128][a.dv == 128](tm, a, T, grid, stream)) return 1;
  if (pg_check_launch("pg_causal_attn_bwd(wgmma dk/dv)")) return 1;
  // dQ: Q / dO tiles of 128 rows
  if (make_attn_map(&tm.q, a.q, a.ld_q, a.H * a.dk, a.S, a.N, AT)) return 1;
  if (make_attn_map(&tm.d_o, a.d_o, a.ld_do, a.H * a.dv, a.S, a.N, AT)) return 1;
  if (kDq[a.dk == 128][a.dv == 128](tm, a, T, grid, stream)) return 1;
  return pg_check_launch("pg_causal_attn_bwd(wgmma dq)");
}

}  // namespace
