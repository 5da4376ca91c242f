// pg_gemm.cu — the channel-contraction kernel: bf16 x bf16 -> fp32 on sm_90a wgmma tensor cores.
//
// One persistent CTA per SM, warp-specialised (gemm_wgmma_kernel): a TMA producer warp fills 128B-swizzled
// shared-memory stages; two consumer warpgroups take alternate 128-row tiles and take turns on the tensor cores
// (ping-pong), so that one runs wgmma m64nBNk16 into register accumulators while the other runs the fused epilogue
// (bias / act' / residual / activation) of its previous tile.  Split-K launches write each K slice's tile to its own slice of the
// library's scratch buffer, and pg_sum_partials adds the slices to the output in slice order: no atomics, so the result
// is the same on every run.
// Operand majors are template parameters so that forward (K,K), dgrad (K,MN) and wgrad (MN,MN) all read the
// tensors where they lie: no transposed copies of activations or weights are ever materialised.
//
// Replaces: every 1x1 nn.Conv2d forward/backward on the reference path (see include/pg_b200.h).
#include <stdlib.h>
#include <string.h>

#include "../../include/pg_b200.h"
#include "pg_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one swizzle span
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int SMEM_LIMIT = 232448;  // 227 KB

// Tap-loop convolution (pg_gemm_bf16_conv): the shifted operand is read straight from the pixel-major activation
// tensor through a 4-D TMA map [C, W, H, N]; out-of-image coordinates are zero-filled by the TMA unit, which is the
// reference's zero padding.  mode 1: A is shifted (forward / dgrad, K = taps x channel slabs); mode 2: B is shifted
// (wgrad, the taps are extra N blocks).  The offsets travel in the kernel parameters as int8 (|offset| <= 64): 225 taps,
// a 15 x 15 kernel, take 450 bytes, and the whole parameter block stays far below the 4 KB limit.
constexpr int MAX_CONV_TAPS = 225;
struct ConvGeom {
  int mode, H, W, C, T;
  int cslabs;  // C / 64 (mode 1): K iterations per tap
  int nbpt;    // mode 2: N blocks per tap (C / BN)
  int8_t dy[MAX_CONV_TAPS], dx[MAX_CONV_TAPS];
};

struct GemmParams {
  ConvGeom conv;
  int M, N, K;
  int num_m_blk, num_n_blk;
  int k_iters;      // ceil(K / BK)
  int k_per_split;  // k iterations per split
  int splits;
  int stages;       // smem pipeline depth
  // TMA epilogue (epi_tma = 1: every epilogue base and pitch is 16-byte aligned, see gemm_entry): each consumer
  // warpgroup owns epi_nbuf staging buffers of epi_buf_bytes; a buffer holds one 64 x 32 sub-tile's inputs (byte
  // offsets off_*, -1 = absent) and, once they are read, its outputs.  epi_in_bytes: the inputs' bytes per sub-tile.
  int epi_tma, epi_nbuf, epi_buf_bytes, epi_in_bytes;
  int off_old, off_res0, off_res1, off_aux, off_f32, off_pre, off_bf16;
  int epi_smem;     // bytes of the epilogue region (staging buffers and bias, or the row path's transpose buffers)
  int store_deriv;  // out_pre receives act'(pre) (PG_ACT_STORE_DERIV)
  int res_bf16;     // res0 / res1 are bf16 matrices (PG_ACT_RES_BF16)
  float* a_rowsum;  // MN-major A only: fp32 [M] += sum_k A(m, k) (pg_gemm_epilogue.bias_grad), nullptr = off
  float* split_part;   // splits > 1: [splits][M][N] fp32 slices of the K-split tiles
  float* rowsum_part;  // splits > 1 with a_rowsum: [splits][M] slices of the row sums
  pg_gemm_epilogue epi;
};

// Tensor maps of the TMA epilogue (unused ones stay zeroed).  fp32 [M, N]: box {32, 64 rows}, 128B swizzle; bf16
// [M, N]: box {32, 64 rows}, 64B swizzle.  out_f32 is 3-D {N, M, splits}: a split-K launch stores slice ks of the
// library's scratch through it, any other launch uses ks = 0; accumulate launches load the old value through it too.
struct EpiMaps {
  CUtensorMap res0, res1, aux, out_f32, out_pre, out_bf16;
  CUtensorMap bias;  // 1-D [N], box BN
};

// ------------------------------------------------------------------------------------------------
// Row-segment epilogue (launches whose epilogue operands TMA cannot address, and the SIMT cross-check): `acc` = 32
// consecutive fp32 accumulator columns of output row `row`, scalar global accesses.  The TMA epilogue
// (consumer_epilogue_tma) keeps this per-element order of operations.
// ------------------------------------------------------------------------------------------------
// x[i] = act(x[i]) (BWD: act'(x[i])) for N values, the activation chosen once.  A per-element switch over `act`
// becomes an indirect branch into a different case body for every element of the unrolled epilogue, and the kernel
// then spends its epilogue fetching instructions; here the taken case runs as one straight unrolled block.
template <bool BWD, int ACT, int N>
__device__ __forceinline__ void act_as(float (&x)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) x[i] = BWD ? pg_act_bwd(ACT, x[i]) : pg_act_fwd(ACT, x[i]);
}
template <bool BWD, int N>
__device__ __forceinline__ void act_n(int act, float (&x)[N]) {
  switch (act) {
    case PG_ACT_RELU: act_as<BWD, PG_ACT_RELU>(x); break;
    case PG_ACT_GELU: act_as<BWD, PG_ACT_GELU>(x); break;
    case PG_ACT_ELU: act_as<BWD, PG_ACT_ELU>(x); break;
    case PG_ACT_TANH: act_as<BWD, PG_ACT_TANH>(x); break;
    case PG_ACT_GIVEN: act_as<BWD, PG_ACT_GIVEN>(x); break;
    case PG_ACT_RELU_OUT: act_as<BWD, PG_ACT_RELU_OUT>(x); break;
    case PG_ACT_ELU_OUT: act_as<BWD, PG_ACT_ELU_OUT>(x); break;
    default: act_as<BWD, PG_ACT_NONE>(x); break;  // the default case of pg_act_fwd / pg_act_bwd
  }
}

// out_f32 / ld_out_f32 / accumulate: the fp32 destination (a split-K launch passes its slice of the scratch).
__device__ __forceinline__ void epilogue_row32(const GemmParams& p, int row, int col0, int ncols, bool first_split,
                                               const uint32_t (&acc)[32], float* out_f32, int64_t ld_out_f32,
                                               bool accumulate) {
  const pg_gemm_epilogue& e = p.epi;
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(acc[i]) * e.alpha;

  if (first_split && e.bias) {
    for (int i = 0; i < ncols; ++i) v[i] += __ldg(e.bias + col0 + i);
  }
  if (e.dact != PG_ACT_NONE) {
    const bf16* aux = reinterpret_cast<const bf16*>(e.aux) + (size_t)row * e.ld_aux + col0;
    for (int i = 0; i < ncols; ++i) v[i] *= pg_act_bwd(e.dact, __bfloat162float(aux[i]));
  }
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    const float* rp = which == 0 ? e.res0 : e.res1;
    if (first_split && rp && p.res_bf16) {
      const bf16* r = reinterpret_cast<const bf16*>(rp) + (size_t)row * e.ld_res + col0;
      for (int i = 0; i < ncols; ++i) v[i] += __bfloat162float(r[i]);
    } else if (first_split && rp) {
      const float* r = rp + (size_t)row * e.ld_res + col0;
      for (int i = 0; i < ncols; ++i) v[i] += r[i];
    }
  }
  if (out_f32) {
    float* o = out_f32 + (size_t)row * ld_out_f32 + col0;
    if (accumulate) {
      for (int i = 0; i < ncols; ++i) o[i] += v[i];  // one writer per element (split-K goes through slices)
    } else {
      for (int i = 0; i < ncols; ++i) o[i] = v[i];
    }
  }
  if (e.out_pre) {
    bf16* o = reinterpret_cast<bf16*>(e.out_pre) + (size_t)row * e.ld_out_pre + col0;
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = v[i];
    if (p.store_deriv) act_n<true>(e.act, d);
    for (int i = 0; i < ncols; ++i) o[i] = __float2bfloat16(d[i]);
  }
  if (e.out_bf16) {
    bf16* o = reinterpret_cast<bf16*>(e.out_bf16) + (size_t)row * e.ld_out_bf16 + col0;
    if (e.act != PG_ACT_NONE) act_n<false>(e.act, v);
    for (int i = 0; i < ncols; ++i) o[i] = __float2bfloat16(v[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// wgmma kernel
// ------------------------------------------------------------------------------------------------
// One persistent CTA per SM, 384 threads.  Work items (tile, K split) are taken in a fixed sequence: blockIdx.x,
// blockIdx.x + gridDim.x, ...  The producer fills the shared-memory stage ring in that order.
//   warpgroup 0   warp 0 issues the TMA loads (global -> 128B-swizzled shared-memory stages, mbarrier expect_tx);
//                 warps 2-3 reduce the bias gradient of weight-gradient GEMMs from the staged A tiles.  It gives up
//                 registers (setmaxnreg.dec) so that the consumers can hold a whole 128 x BN accumulator each.
//   warpgroups 1, 2  consumers, ping-pong: warpgroup w takes work items w, w + 2, w + 4, ... of the CTA's sequence and
//                 owns the whole 128-row tile (two wgmma m64nBNk16 per K step, one per 64-row slab, accumulators in
//                 registers).  The warpgroups take turns on the tensor cores: a warpgroup starts its main loop once
//                 the other has issued all MMAs of the previous item, so one runs its epilogue while the other runs
//                 its MMAs.  The hand-offs are named barriers: an mbarrier wait may suspend the warp, and its wake-up
//                 latency would sit on the per-tile critical path.  Epilogues do not take turns: with K = 512 an
//                 epilogue lasts about three main loops (on the H100, 8-12 us against 3 us per 128 x 128 tile), so the
//                 two warpgroups' epilogues overlap; their outputs are disjoint.
//                 Every output element sees the same m64nBNk16 instructions in the same K order as with one 64-row
//                 slab per warpgroup.  A CTA with a single work item (one-wave split-K weight gradients) leaves one
//                 consumer idle: one warpgroup issuing both slabs keeps pace with two splitting the rows (on the
//                 H100, fc1 wgrad with one item per CTA measured 0.42 ms this way and 0.46 ms with the rows split),
//                 so there is one schedule.
// The epilogue (consumer_epilogue_tma) works on the accumulator fragments in 64 x 32 sub-tiles, each consumer warp on
// its own 16 rows of them: the warp's TMA brings its inputs into the warp's staging buffer ahead of use, and stores its
// outputs from the same buffer.
// Launches whose epilogue operands TMA cannot address take the row path (consumer_epilogue): a shared-memory transpose
// ([64 rows][64 columns] fp32 per warpgroup and step), then one 32-column row segment per thread with epilogue_row32.
constexpr int GEMM_THREADS = 384;
constexpr int XP_LD = 68;  // transpose row pitch in floats: the float4 row reads of a warp hit 32 distinct banks
constexpr int XP_BYTES = 64 * XP_LD * 4;
constexpr int MAX_STAGES = 8;
constexpr int MAX_EPI_BUFS = 4;                  // staging buffers per consumer warp
constexpr int EPI_F32_BYTES = 16 * 32 * 4;       // one warp's fp32 piece of a 64 x 32 sub-tile
constexpr int EPI_BF16_BYTES = 16 * 32 * 2;      // one warp's bf16 piece
constexpr int EPI_BIAS_BYTES = 128 * 4;          // a tile's bias, per consumer warpgroup
// 128 * 56 + 256 * 224 = 384 * 168: the register file split unevenly between the three warpgroups.  56 is what the
// bias-gradient warps need to keep their sixteen 16-byte shared-memory loads per stage in flight: they release every
// stage, so with fewer registers (40, loads four at a time) they paced the weight-gradient launches; the consumers
// spill at BN = 128 below 224.
constexpr int PRODUCER_REGS = 56;
constexpr int CONSUMER_REGS = 224;
// named barrier ids (0 is __syncthreads)
constexpr uint32_t XPOSE_BAR = 1;     // + w: warpgroup w's transpose buffer on the row path (128 threads)
constexpr uint32_t ROWSUM_BAR = 3;    // warps 2-3 (64 threads)
constexpr uint32_t MMA_TURN_BAR = 4;  // + w: warpgroup w may start its main loop (256 threads: one arrives, one waits)

struct WorkItem {
  int m_blk, n_blk, ks, k0, k1;  // output tile, K split, and its k-block range [k0, k1)
};
__device__ __forceinline__ WorkItem work_item(const GemmParams& p, int tile) {
  WorkItem w;
  w.n_blk = tile % p.num_n_blk;
  const int rest = tile / p.num_n_blk;
  w.m_blk = rest % p.num_m_blk;
  w.ks = rest / p.num_m_blk;
  w.k0 = w.ks * p.k_per_split;
  w.k1 = min(w.k0 + p.k_per_split, p.k_iters);
  return w;
}

// Consumer main loop over one work item: 64-row slab sl of the tile accumulates in acc[sl], stages from ring position
// (s, ph).  Once the last MMAs are issued, arrives on turn_bar (when >= 0) so that the other warpgroup may start.
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void consumer_mainloop(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int stages,
                                                  const WorkItem& w, int& s, uint32_t& ph, float (&acc)[2][BN / 2],
                                                  int turn_bar) {
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * BK * 2;
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int kit = w.k0; kit < w.k1; ++kit) {
    mbar_wait(&full_bar[s], ph);
    // 64-row slab sl of A: the sl-th 64-row block (K-major) or the sl-th 64-wide atom (MN-major)
    const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES);
    const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_STAGE_BYTES;
    // a K step (16 elements) only moves the start address: K-major 32 bytes inside the swizzle span, MN-major
    // 16 k-rows of 128 B = 2048 bytes (LBO = the stride between 64-wide MN atoms)
    const uint64_t b_base = B_MN ? wgmma_desc_sw128(b_addr, BK * 128, 1024) : wgmma_desc_sw128(b_addr, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        const uint32_t sa = a_addr + sl * (64 * 128);
        const uint64_t a_base = A_MN ? wgmma_desc_sw128(sa, BK * 128, 1024) : wgmma_desc_sw128(sa, 16, 1024);
        Wgmma<BN>::template ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[sl], a_base + (uint64_t)(A_MN ? kk * 128 : kk * 2),
                                                         b_base + (uint64_t)(B_MN ? kk * 128 : kk * 2),
                                                         (kit > w.k0 || kk > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();  // the MMAs of the previous stage have completed: release it
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = s;
    if (++s == stages) { s = 0; ph ^= 1; }
  }
  if (turn_bar >= 0) named_bar_arrive((uint32_t)turn_bar, 256);
  wgmma_wait<0>();
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) wgmma_hold(acc[sl]);
  if (prev >= 0) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
  }
}

// Epilogue of one work item: 64 columns of one slab per step through the transpose; thread t finishes row (t % 64) of
// the slab, columns 32 * (t / 64) + [0, 32).  The step loop is not unrolled, so that the kernel holds one copy of
// epilogue_row32.
template <int BN>
__device__ __forceinline__ void consumer_epilogue(const GemmParams& p, const WorkItem& w, const float (&acc)[2][BN / 2],
                                                  float* xp, uint32_t xbar) {
  constexpr int CSTEPS = (BN + 63) / 64;  // 64-column steps per slab
  const int t = threadIdx.x & 127, lane = threadIdx.x & 31, wi = (threadIdx.x >> 5) & 3;
  const int r = t & 63, half = t >> 6;
#pragma unroll 1
  for (int step = 0; step < 2 * CSTEPS; ++step) {
    const int sl = step / CSTEPS, c0 = (step - sl * CSTEPS) * 64;
    const int row = w.m_blk * BM + sl * 64 + r;
    named_bar_sync(xbar, 128);  // the previous step's reads of xp are done
#pragma unroll
    for (int q = 0; q < 2; ++q) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {  // fully unrolled: the accumulator stays in registers
        if (q == sl && j * 8 >= c0 && j * 8 < c0 + 64) {
          const int col = j * 8 - c0 + 2 * (lane & 3), fr = wi * 16 + (lane >> 2);
          *reinterpret_cast<float2*>(xp + fr * XP_LD + col) = make_float2(acc[q][4 * j], acc[q][4 * j + 1]);
          *reinterpret_cast<float2*>(xp + (fr + 8) * XP_LD + col) = make_float2(acc[q][4 * j + 2], acc[q][4 * j + 3]);
        }
      }
    }
    named_bar_sync(xbar, 128);
    const int col0 = w.n_blk * BN + c0 + half * 32;
    if (c0 + half * 32 < BN && row < p.M && col0 < p.N) {
      uint32_t v[32];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float4 x = *reinterpret_cast<const float4*>(xp + r * XP_LD + half * 32 + 4 * u);
        v[4 * u] = __float_as_uint(x.x); v[4 * u + 1] = __float_as_uint(x.y);
        v[4 * u + 2] = __float_as_uint(x.z); v[4 * u + 3] = __float_as_uint(x.w);
      }
      // split-K: this split's slice; pg_sum_partials adds the slices in order after the launch
      const bool split = p.split_part != nullptr;
      epilogue_row32(p, row, col0, min(32, p.N - col0), w.ks == 0, v,
                     split ? p.split_part + (size_t)w.ks * p.M * p.N : p.epi.out_f32,
                     split ? (int64_t)p.N : p.epi.ld_out_f32, !split && p.epi.accumulate);
    }
  }
}

// ---- TMA epilogue ----
// Per warp: the wgmma fragment gives warp wi rows wi * 16 ... wi * 16 + 15 of each 64-row slab, and each consumer warp
// moves those rows itself.  Sub-tile j of a work item is 64-row slab j / (BN / 32) and 32-column group j % (BN / 32);
// the warp's piece of it is a 16 x 32 box.  A thread holds 16 of its elements in the fragment layout: rows lane / 4
// (+ 8) of the box, columns 8 jj + 2 (lane % 4) (+ 1), jj < 4.  Staging layouts are the tensor maps' swizzles: fp32
// rows of 128 bytes (128B swizzle), bf16 rows of 64 bytes (64B swizzle).  The fragment's 8-byte fp32 accesses put two
// words in every bank (the minimum for 256 bytes), the 4-byte bf16 accesses one.
// Each warp owns epi_nbuf staging buffers and their mbarriers, and lane 0 issues its loads and stores and waits for
// its own bulk groups, so only __syncwarp orders a warp's compute, proxy fence and store: no barrier of the warpgroup
// runs inside the epilogue.  The warp's sub-tiles are numbered across its work items (g = item * NSUB + sub-tile):
// sub-tile g uses buffer g % epi_nbuf, whose barrier completes for the (g / epi_nbuf)-th time.  Nothing of the ring is
// held in registers across the main loop, where the BN = 128 consumer has none to spare.
struct EpiRing {
  uint8_t* buf;       // the warp's epi_nbuf staging buffers
  float* bias;        // [BN], one per warpgroup
  uint64_t* in_bar;   // [epi_nbuf]: the inputs of the warp's sub-tile in buffer b have landed
  uint64_t* bias_bar;
};
__device__ __forceinline__ EpiRing epi_ring(const GemmParams& p, uint8_t* epi, int cw) {
  const int wq = cw * 4 + ((threadIdx.x >> 5) & 3);  // the warp's index among the 8 consumer warps
  EpiRing r;
  r.buf = epi + wq * p.epi_nbuf * p.epi_buf_bytes;
  r.bias = reinterpret_cast<float*>(epi + 8 * p.epi_nbuf * p.epi_buf_bytes + cw * EPI_BIAS_BYTES);
  r.in_bar = reinterpret_cast<uint64_t*>(epi + p.epi_smem) + 2 * MAX_STAGES + wq * MAX_EPI_BUFS;
  r.bias_bar = reinterpret_cast<uint64_t*>(epi + p.epi_smem) + 2 * MAX_STAGES + 8 * MAX_EPI_BUFS + cw;
  return r;
}

// Compile-time epilogue kinds: the combinations of epilogue operands that the ImageGPT step and the conv stacks launch
// at BN = 128 with K-major A, each built without the loads, branches, alpha multiply and activation switch of the
// others (epi_kind in launch_tc picks one).  EK_GENERIC reads every choice from the launch parameters at run time.
constexpr int EK_GENERIC = 0;
constexpr int EK_BIAS = 1, EK_GIVEN = 2, EK_RES0 = 4, EK_RES1 = 8, EK_F32 = 16, EK_BF16 = 32, EK_GELU2 = 64;
constexpr int EK_PLAIN = EK_BF16;                                // dgrad: bf16 output
constexpr int EK_BIAS_BF16 = EK_BIAS | EK_BF16;                  // qkv forward
constexpr int EK_BIAS_GELU2 = EK_BIAS | EK_GELU2;                // fc1 forward: out_bf16 = GELU, out_pre = GELU'
constexpr int EK_GIVEN_BF16 = EK_GIVEN | EK_BF16;                // fc2 dgrad: x act' given in aux
constexpr int EK_BIAS_RES_F32 = EK_BIAS | EK_RES0 | EK_F32;      // proj forward
constexpr int EK_BIAS_RES2_F32 = EK_BIAS | EK_RES0 | EK_RES1 | EK_F32;  // fc2 forward

__device__ __forceinline__ bool subtile_live(const GemmParams& p, int row, int col) { return row < p.M && col < p.N; }

// Issued by lane 0 of the warp: the inputs of the warp's piece of sub-tile j of the item (g0 + j across items) into
// its staging buffer (whose previous store has been read).
template <int BN>
__device__ __forceinline__ void epi_load(const GemmParams& p, const EpiMaps& tm, const WorkItem& w, const EpiRing& r,
                                         int g0, int j) {
  constexpr int CG = BN / 32;
  const int wi = (threadIdx.x >> 5) & 3;
  const int b = (g0 + j) % p.epi_nbuf;
  uint8_t* buf = r.buf + b * p.epi_buf_bytes;
  const int col = w.n_blk * BN + (j % CG) * 32, row = w.m_blk * BM + (j / CG) * 64 + wi * 16;
  if (!subtile_live(p, row, col)) {  // nothing to load or store: complete the phase without bytes
    mbar_arrive(&r.in_bar[b]);
    return;
  }
  mbar_arrive_expect_tx(&r.in_bar[b], (uint32_t)p.epi_in_bytes);
  if (p.off_old >= 0) tma_load_3d(buf + p.off_old, &tm.out_f32, &r.in_bar[b], col, row, 0);
  if (p.off_res0 >= 0) tma_load_2d(buf + p.off_res0, &tm.res0, &r.in_bar[b], col, row);
  if (p.off_res1 >= 0) tma_load_2d(buf + p.off_res1, &tm.res1, &r.in_bar[b], col, row);
  if (p.off_aux >= 0) tma_load_2d(buf + p.off_aux, &tm.aux, &r.in_bar[b], col, row);
}

// Before the work item's main loop, lane 0 of each warp requests the inputs of the warp's first epi_nbuf - 1
// sub-tiles, so that they land while the MMAs run.  Those sub-tiles reuse the buffers of every earlier sub-tile but
// the last, so only the warp's stores before the previous item's last one must have been read, and without inputs
// nothing waits here: the warp's first wgmma is not held up by the previous item's stores.
template <int BN>
__device__ __forceinline__ void epi_prologue(const GemmParams& p, const EpiMaps& tm, const WorkItem& w, const EpiRing& r,
                                             int item) {
  if ((threadIdx.x & 31) != 0 || !p.epi_in_bytes) return;
  bulk_wait_group_read<1>();
  for (int j = 0; j < p.epi_nbuf - 1 && j < 2 * (BN / 32); ++j) epi_load<BN>(p, tm, w, r, item * 2 * (BN / 32), j);
}

// The tile's bias, requested by thread 0 of the warpgroup once every warp of it has finished the previous item's
// epilogue (the turn barrier before the main loop), so the buffer is free.  Split-K launches have no bias.
template <int BN>
__device__ __forceinline__ void epi_bias(const GemmParams& p, const EpiMaps& tm, const WorkItem& w, const EpiRing& r) {
  if ((threadIdx.x & 127) != 0 || !p.epi.bias) return;
  mbar_arrive_expect_tx(r.bias_bar, BN * 4);
  tma_load_1d(r.bias, &tm.bias, r.bias_bar, w.n_blk * BN);
}

// Per element, the order of epilogue_row32: x alpha, + bias, x act'(aux), + res0, + res1, then out_f32 (+= old when
// accumulating), out_pre (act'(pre) with store_deriv), out_bf16 (act).  Sub-tile i: wait for its inputs, compute,
// __syncwarp (every lane has read the buffer, and lane 0 has waited for the store that last used it), write the
// outputs over the inputs, __syncwarp, lane 0 stores them, and once the store of sub-tile i - 1 has been read it
// requests the inputs of sub-tile i + epi_nbuf - 1 into that buffer.  Without inputs a buffer is only needed again
// epi_nbuf sub-tiles later, and so are the reads of its store.
// EK: the epilogue kind.  The specialised kinds unroll the sub-tile loop, so the accumulator is indexed statically.
// EK_GENERIC keeps one copy of the loop and picks the sub-tile's 16 accumulators at run time; ACT = false: the
// launch has no activation, no activation derivative and no act'(pre) output, and the generic epilogue is built
// without the activation code.  The unrolled activation bodies are tens of kilobytes of instructions that the other
// launches branch over, and on the H100 that cost a plain bf16 epilogue 15 % of its time.
template <int BN, int EK, bool ACT>
__device__ __forceinline__ void consumer_epilogue_tma(const GemmParams& p, const EpiMaps& tm, const WorkItem& w,
                                                      const float (&acc)[2][BN / 2], const EpiRing& r, int item) {
  constexpr int CG = BN / 32, NSUB = 2 * CG;
  constexpr bool G = EK == EK_GENERIC;
  const pg_gemm_epilogue& e = p.epi;
  const int lane = threadIdx.x & 31, wi = (threadIdx.x >> 5) & 3;
  const int nb = p.epi_nbuf, g0 = item * NSUB;
  // what the launch computes: fixed by the kind, or read from the parameters (generic)
  const bool bias = G ? e.bias != nullptr : (EK & EK_BIAS) != 0;
  const bool has_in = G ? p.epi_in_bytes != 0 : (EK & (EK_GIVEN | EK_RES0)) != 0;
  const bool f32_out = G ? p.off_f32 >= 0 : (EK & EK_F32) != 0;
  const bool bf16_out = G ? p.off_bf16 >= 0 : (EK & (EK_BF16 | EK_GELU2)) != 0;
  const bool pre_out = G ? p.off_pre >= 0 : (EK & EK_GELU2) != 0;
  if (bias) mbar_wait(r.bias_bar, (uint32_t)item & 1u);
  // Byte offsets of the thread's pair (jj, hi) inside an fp32 / bf16 piece.  Row rb + 8 hi; the 16-byte chunk index
  // (2 jj + bit 1 of the lane for fp32, jj for bf16) is XORed with the row's swizzle bits (rb % 8 for 128B,
  // (rb / 2) % 4 for 64B), and rows 8 apart share them, so jj enters as one XOR on a per-thread base.
  const uint32_t rb = lane >> 2;
  const uint32_t f32_base = rb * 128 + ((((uint32_t)lane >> 1) & 1u) ^ (rb & 7u)) * 16 + (lane & 1) * 8;
  const uint32_t bf_base = rb * 64 + ((rb >> 1) & 3u) * 16 + (lane & 3) * 4;
  auto f32_at = [&](int jj, int hi) { return (f32_base ^ (uint32_t)(jj << 5)) + hi * 1024; };
  auto bf_at = [&](int jj, int hi) { return (bf_base ^ (uint32_t)(jj << 4)) + hi * 512; };
  int b = g0 % nb;
  uint32_t par = (uint32_t)(g0 / nb) & 1u;
#pragma unroll(G ? 1 : NSUB)
  for (int i = 0; i < NSUB; ++i) {
    const int sl = i / CG, cg = i - sl * CG;
    uint8_t* buf = r.buf + b * p.epi_buf_bytes;
    float v[16];
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int c = 0; c < CG; ++c)
        if (q == sl && c == cg) {
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = acc[q][c * 16 + k];
        }
    if (has_in) mbar_wait(&r.in_bar[b], par);
    if (G) {
#pragma unroll
      for (int k = 0; k < 16; ++k) v[k] *= e.alpha;
    }
    if (bias) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float2 bb = *reinterpret_cast<const float2*>(r.bias + cg * 32 + jj * 8 + 2 * (lane & 3));
        v[4 * jj] += bb.x; v[4 * jj + 1] += bb.y; v[4 * jj + 2] += bb.x; v[4 * jj + 3] += bb.y;
      }
    }
    if ((G && ACT && e.dact != PG_ACT_NONE) || (EK & EK_GIVEN)) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // eight at a time: registers
        float g[8];
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
#pragma unroll
          for (int hi = 0; hi < 2; ++hi) {
            const float2 f =
                unpack_bf16x2(*reinterpret_cast<const uint32_t*>(buf + p.off_aux + bf_at(2 * h + jj, hi)));
            g[4 * jj + 2 * hi] = f.x;
            g[4 * jj + 2 * hi + 1] = f.y;
          }
        if (G) act_n<true>(e.dact, g);  // EK_GIVEN: aux is act' itself (pg_act_bwd(PG_ACT_GIVEN, x) = x)
#pragma unroll
        for (int k = 0; k < 8; ++k) v[8 * h + k] *= g[k];
      }
    }
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      const bool res = G ? (which == 0 ? p.off_res0 : p.off_res1) >= 0 : (EK & (which == 0 ? EK_RES0 : EK_RES1)) != 0;
      if (!res) continue;
      const int off = which == 0 ? p.off_res0 : p.off_res1;
      const bool res_bf16 = G && p.res_bf16;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
          const float2 f = res_bf16 ? unpack_bf16x2(*reinterpret_cast<const uint32_t*>(buf + off + bf_at(jj, hi)))
                                    : *reinterpret_cast<const float2*>(buf + off + f32_at(jj, hi));
          v[4 * jj + 2 * hi] += f.x;
          v[4 * jj + 2 * hi + 1] += f.y;
        }
    }
    __syncwarp();  // the buffer's inputs are read (and lane 0 has waited for the buffer's previous store)
    if (f32_out) {
      // the old value of an accumulate launch lies where its sum goes (both at offset 0): each thread reads and
      // overwrites only its own elements there, so this read may follow the __syncwarp
      const bool old = G && p.off_old >= 0;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
          float2* o = reinterpret_cast<float2*>(buf + p.off_f32 + f32_at(jj, hi));
          float2 f = make_float2(v[4 * jj + 2 * hi], v[4 * jj + 2 * hi + 1]);
          if (old) {
            const float2 ov = *o;
            f = make_float2(ov.x + f.x, ov.y + f.y);
          }
          *o = f;
        }
    }
    bool v_act = false;  // v already holds act(v)
    if (pre_out) {
      float d[16];
      if ((EK & EK_GELU2) || (G && ACT && p.store_deriv && e.act == PG_ACT_GELU)) {
        // GELU and GELU' of the same value share one tanh
#pragma unroll
        for (int k = 0; k < 16; ++k) pg_gelu_both(v[k], v[k], d[k]);
        v_act = true;
      } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) d[k] = v[k];
        if (G && ACT && p.store_deriv) act_n<true>(e.act, d);
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int hi = 0; hi < 2; ++hi)
          *reinterpret_cast<uint32_t*>(buf + p.off_pre + bf_at(jj, hi)) =
              pack_bf16x2(d[4 * jj + 2 * hi], d[4 * jj + 2 * hi + 1]);
    }
    if (bf16_out) {
      if (G && ACT && !v_act && e.act != PG_ACT_NONE) act_n<false>(e.act, v);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int hi = 0; hi < 2; ++hi)
          *reinterpret_cast<uint32_t*>(buf + p.off_bf16 + bf_at(jj, hi)) =
              pack_bf16x2(v[4 * jj + 2 * hi], v[4 * jj + 2 * hi + 1]);
    }
    fence_proxy_async_smem();  // the generic-proxy writes become visible to the TMA unit
    __syncwarp();
    if (lane == 0) {
      const int col = w.n_blk * BN + cg * 32, row = w.m_blk * BM + sl * 64 + wi * 16;
      if (subtile_live(p, row, col)) {
        if (f32_out) tma_store_3d(&tm.out_f32, buf + p.off_f32, col, row, w.ks);
        if (pre_out) tma_store_2d(&tm.out_pre, buf + p.off_pre, col, row);
        if (bf16_out) tma_store_2d(&tm.out_bf16, buf + p.off_bf16, col, row);
      }
      bulk_commit_group();
      if (has_in) {
        bulk_wait_group_read<1>();  // the store of sub-tile i - 1 has left its buffer: its next inputs may come in
        if (i + nb - 1 < NSUB) epi_load<BN>(p, tm, w, r, g0, i + nb - 1);
      } else if (nb == 4) {  // no inputs: sub-tile i + 1 writes the buffer of sub-tile i + 1 - nb
        bulk_wait_group_read<3>();
      } else if (nb == 3) {
        bulk_wait_group_read<2>();
      } else {
        bulk_wait_group_read<1>();
      }
    }
    if (++b == nb) { b = 0; par ^= 1u; }
  }
}

// Warps 2-3 of weight-gradient GEMMs: the bias gradient from the staged A tiles.  A = dY read MN-major, so
// sum_k A(m, k) is the bias gradient of the layer whose weight gradient this launch computes.  The two otherwise idle
// warps add up the A stages while the MMAs run, so dY is not re-read from HBM by a separate column-sum pass.  Every
// N block of a (m block, split) stages the same A tiles, so the tile's 128 rows are shared out between the CTAs of N
// blocks 0 .. R - 1 (R = 8 / W, as many as the launch has N blocks, up to 4): each sums its 128 / R rows, W per thread.
// With the whole tile in one CTA, its two warps had to read and add 16 KB per stage against the MMAs' 2 MFLOP, and
// those CTAs finished last (fc2 of the C5 step: 8 of 128 CTAs, and the launch took 1.8 times as long as without the
// bias gradient).  Each row has one writer: added to a_rowsum directly, or, split-K, stored to the split's slice of
// rowsum_part.  Thread (u, g) sums k-rows g, g + 4, ... of every stage in k order for its W rows, and the four k-row
// groups are combined in a fixed order, so each row's sum is the same whatever R is.  Every CTA's warps 2-3 release
// every stage, whether they read it or not.
template <int BN, int W>
__device__ __forceinline__ void rowsum_warps(const GemmParams& p, const uint8_t* smem, uint64_t* full_bar,
                                             uint64_t* empty_bar, float* rowsum_xch, int stages, int num_tiles) {
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * BK * 2;
  constexpr int R = 8 / W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = (warp - 2) * 32 + lane;  // 0..63
  const int u = t & 15, g = t >> 4;      // W consecutive rows of the CTA's 128 / R, k-row group
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const WorkItem w = work_item(p, tile);
    const bool mine = w.n_blk < R;
    const int mo = w.n_blk * (BM / R) + u * W;  // the thread's first row in the tile
    // 64-wide MN atom, 16-byte chunk (8 rows) inside its 128-byte k-row, and the byte offset inside the chunk
    const uint32_t atom = (uint32_t)(mo >> 6) * (BK * 128), cc = (uint32_t)((mo & 63) >> 3), sub = (uint32_t)(mo & 7) * 2;
    float acc[W];
#pragma unroll
    for (int q = 0; q < W; ++q) acc[q] = 0.f;
    for (int kit = w.k0; kit < w.k1; ++kit) {
      mbar_wait(&full_bar[s], ph);
      if (mine) {
        const uint8_t* sA = smem + s * STAGE_BYTES + atom + sub;
#pragma unroll
        for (int i = 0; i < BK / 4; ++i) {
          const uint32_t k = (uint32_t)(g + 4 * i);
          const uint8_t* src = sA + k * 128 + ((cc ^ (k & 7u)) << 4);
          uint32_t ww[W / 2];
          if constexpr (W == 8) {
            const uint4 v = *reinterpret_cast<const uint4*>(src);
            ww[0] = v.x; ww[1] = v.y; ww[2] = v.z; ww[3] = v.w;
          } else if constexpr (W == 4) {
            const uint2 v = *reinterpret_cast<const uint2*>(src);
            ww[0] = v.x; ww[1] = v.y;
          } else {
            ww[0] = *reinterpret_cast<const uint32_t*>(src);
          }
#pragma unroll
          for (int j = 0; j < W / 2; ++j) {
            const float2 f = unpack_bf16x2(ww[j]);
            acc[2 * j] += f.x;
            acc[2 * j + 1] += f.y;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);  // release: this warp's reads of the stage are done
      if (++s == stages) { s = 0; ph ^= 1; }
    }
    if (mine) {
#pragma unroll
      for (int q = 0; q < W; ++q) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], 16);  // the warp's two k-row groups
      // warp 3 hands its sums to warp 2, which adds them (a fixed order) and is the only writer
      named_bar_sync(ROWSUM_BAR, 64);  // warp 2 has read the previous tile's exchange
      if (warp == 3 && lane < 16) {
#pragma unroll
        for (int q = 0; q < W; ++q) rowsum_xch[lane * 8 + q] = acc[q];
      }
      named_bar_sync(ROWSUM_BAR, 64);
      if (warp == 2 && lane < 16) {
#pragma unroll
        for (int q = 0; q < W; ++q) acc[q] += rowsum_xch[lane * 8 + q];
        const int m0 = w.m_blk * BM + mo;
#pragma unroll
        for (int q = 0; q < W; ++q)
          if (m0 + q < p.M) {
            if (p.rowsum_part) p.rowsum_part[(size_t)w.ks * p.M + m0 + q] = acc[q];
            else p.a_rowsum[m0 + q] += acc[q];
          }
      }
    }
  }
}

template <int BN, bool A_MN, bool B_MN, int EK>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ EpiMaps tmE, const GemmParams p) {
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * BK * 2;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms need 1024-byte aligned stage bases.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int STAGES = p.stages;
  // TMA epilogue: [8 consumer warps][epi_nbuf][epi_buf_bytes] staging, then [2][BN] fp32 bias; row path: [2][64][XP_LD]
  uint8_t* const epi = smem + STAGES * STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi + p.epi_smem);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* in_bar = empty_bar + MAX_STAGES;      // [8 consumer warps][MAX_EPI_BUFS]
  uint64_t* bias_bar = in_bar + 8 * MAX_EPI_BUFS;  // [2]
  float* rowsum_xch = reinterpret_cast<float*>(bias_bar + 2);  // [16][8]: warp 3's row sums for warp 2

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool rowsum = A_MN && p.a_rowsum != nullptr;
  const int num_tiles = p.num_m_blk * p.num_n_blk * p.splits;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      // freed by the four warps of the consuming warpgroup and, when the side reduction over A is on, by its two
      // warps as well
      mbar_init(&empty_bar[i], rowsum ? 6 : 4);
    }
    for (int i = 0; i < 8 * MAX_EPI_BUFS + 2; ++i) mbar_init(&in_bar[i], 1);  // in_bar and bias_bar
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0) {
      // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const WorkItem w = work_item(p, tile);
        const int m_blk = w.m_blk, n_blk = w.n_blk;
        for (int kit = w.k0; kit < w.k1; ++kit) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sA = smem + s * STAGE_BYTES;
          uint8_t* sB = sA + A_STAGE_BYTES;
          mbar_arrive_expect_tx_w(&full_bar[s], STAGE_BYTES);
          if (p.conv.mode != 0) {
            const int hw = p.conv.H * p.conv.W;
            if (p.conv.mode == 1) {  // A = activations under tap t (forward / dgrad)
              const int t = kit / p.conv.cslabs, cs = kit - t * p.conv.cslabs;
              const int row0 = m_blk * BM, n = row0 / hw, h0 = (row0 - n * hw) / p.conv.W;
              tma_load_4d_w(sA, &tmA, &full_bar[s], cs * 64, p.conv.dx[t], h0 + p.conv.dy[t], n);
              if (!B_MN) {
                tma_load_2d_w(sB, &tmB, &full_bar[s], kit * BK, n_blk * BN);
              } else {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)
                  tma_load_2d_w(sB + j * (BK * 128), &tmB, &full_bar[s], t * p.N + n_blk * BN + j * 64, cs * 64);
              }
            } else {  // wgrad: A = dY (MN-major), B = activations under the tap this N block belongs to
              const int t = n_blk / p.conv.nbpt, nb = n_blk - t * p.conv.nbpt;
              const int pix0 = kit * BK, n = pix0 / hw, h0 = (pix0 - n * hw) / p.conv.W;
#pragma unroll
              for (int j = 0; j < BM / 64; ++j)
                tma_load_2d_w(sA + j * (BK * 128), &tmA, &full_bar[s], m_blk * BM + j * 64, kit * BK);
#pragma unroll
              for (int j = 0; j < BN / 64; ++j)
                tma_load_4d_w(sB + j * (BK * 128), &tmB, &full_bar[s], nb * BN + j * 64, p.conv.dx[t], h0 + p.conv.dy[t], n);
            }
          } else {
            if (!A_MN) {
              tma_load_2d_w(sA, &tmA, &full_bar[s], kit * BK, m_blk * BM);  // box {64 k, 128 rows}
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j)  // box {64 m, 64 k-rows} per 64-wide MN atom
                tma_load_2d_w(sA + j * (BK * 128), &tmA, &full_bar[s], m_blk * BM + j * 64, kit * BK);
            }
            if (!B_MN) {
              tma_load_2d_w(sB, &tmB, &full_bar[s], kit * BK, n_blk * BN);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j)
                tma_load_2d_w(sB + j * (BK * 128), &tmB, &full_bar[s], n_blk * BN + j * 64, kit * BK);
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    } else if (A_MN && (warp == 2 || warp == 3)) {
      // ===================== warps 2-3, weight-gradient GEMMs: bias gradient from the staged A tiles =====================
      if (rowsum) {
        if (p.num_n_blk >= 4) {
          rowsum_warps<BN, 2>(p, smem, full_bar, empty_bar, rowsum_xch, STAGES, num_tiles);
        } else if (p.num_n_blk >= 2) {
          rowsum_warps<BN, 4>(p, smem, full_bar, empty_bar, rowsum_xch, STAGES, num_tiles);
        } else {
          rowsum_warps<BN, 8>(p, smem, full_bar, empty_bar, rowsum_xch, STAGES, num_tiles);
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup cw = 0, 1 =====================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = (warp - 4) >> 2;
    float* const xp = reinterpret_cast<float*>(epi) + cw * 64 * XP_LD;
    float acc[2][BN / 2];
    int s = 0;
    uint32_t ph = 0;
    int i = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++i) {
      const WorkItem w = work_item(p, tile);
      if ((i & 1) != cw) {  // the other warpgroup's item: step the ring position past its k-blocks
        const int pos = s + (w.k1 - w.k0);
        ph ^= (uint32_t)((pos / STAGES) & 1);
        s = pos % STAGES;
        continue;
      }
      // item i waits for the other warpgroup's turn on item i - 1 and hands the turn on if item i + 1 exists
      const bool has_next = tile + (int)gridDim.x < num_tiles;
      if (p.epi_tma) epi_prologue<BN>(p, tmE, w, epi_ring(p, epi, cw), i >> 1);
      if (i > 0) named_bar_sync(MMA_TURN_BAR + cw, 256);
      if (p.epi_tma) epi_bias<BN>(p, tmE, w, epi_ring(p, epi, cw));
      consumer_mainloop<BN, A_MN, B_MN>(smem, full_bar, empty_bar, STAGES, w, s, ph, acc,
                                        has_next ? (int)(MMA_TURN_BAR + (cw ^ 1)) : -1);
      if constexpr (BN <= 64) {  // the row path runs at BN <= 64 (dispatch_bn): no registers to spare at 128
        if (!p.epi_tma) consumer_epilogue<BN>(p, w, acc, xp, XPOSE_BAR + cw);
      }
      if (p.epi_tma) {
        const EpiRing r = epi_ring(p, epi, cw);
        if constexpr (EK != EK_GENERIC)
          consumer_epilogue_tma<BN, EK, false>(p, tmE, w, acc, r, i >> 1);
        else if (p.epi.act == PG_ACT_NONE && p.epi.dact == PG_ACT_NONE && !p.store_deriv)
          consumer_epilogue_tma<BN, EK, false>(p, tmE, w, acc, r, i >> 1);
        else
          consumer_epilogue_tma<BN, EK, true>(p, tmE, w, acc, r, i >> 1);
      }
    }
    if (lane == 0) bulk_wait_group_all();  // each warp's stores are complete before the CTA exits
  }
}

// ------------------------------------------------------------------------------------------------
// SIMT cross-check kernel (tests only): one thread per 1x32 output segment, same epilogue arithmetic.
// ------------------------------------------------------------------------------------------------
__global__ void gemm_simt_kernel(const bf16* __restrict__ A, int a_mn, int64_t lda, const bf16* __restrict__ B,
                                 int b_mn, int64_t ldb, const GemmParams p) {
  const int nseg = (p.N + 31) / 32;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)p.M * nseg) return;
  const int row = (int)(idx / nseg);
  const int col0 = (int)(idx % nseg) * 32;
  const int ncols = min(32, p.N - col0);
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int k = 0; k < p.K; ++k) {
    const float a = __bfloat162float(a_mn ? A[(size_t)k * lda + row] : A[(size_t)row * lda + k]);
    for (int i = 0; i < ncols; ++i) {
      const int n = col0 + i;
      const float b = __bfloat162float(b_mn ? B[(size_t)k * ldb + n] : B[(size_t)n * ldb + k]);
      acc[i] = fmaf(a, b, acc[i]);
    }
  }
  uint32_t accu[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) accu[i] = __float_as_uint(acc[i]);
  epilogue_row32(p, row, col0, ncols, true, accu, p.epi.out_f32, p.epi.ld_out_f32, p.epi.accumulate != 0);
}

// ------------------------------------------------------------------------------------------------
// Skinny forward GEMM (M <= 32 rows): the per-pixel step of incremental sampling multiplies a handful of rows (one per
// image) by the full weight matrices.  A 128-row tensor-core tile would run on N/256 SMs and be latency-bound; here
// every warp owns one output column, streams its weight row once (16-byte loads) against the A rows held in shared
// memory, and the whole chip participates.  Same fused epilogue semantics (bias, residuals, activation).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gemm_skinny_kernel(const bf16* __restrict__ A, int64_t lda, const bf16* __restrict__ B, int64_t ldb, const GemmParams p) {
  extern __shared__ uint4 sA4[];  // [M][K/8] 16-byte units
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int K8 = p.K / 8;
  for (int i = threadIdx.x; i < p.M * K8; i += blockDim.x)
    sA4[i] = *reinterpret_cast<const uint4*>(A + (size_t)(i / K8) * lda + (i % K8) * 8);
  __syncthreads();
  const int n = blockIdx.x * 8 + warp;
  if (n >= p.N) return;
  float acc[32];
#pragma unroll
  for (int m = 0; m < 32; ++m) acc[m] = 0.f;
  const uint4* wrow = reinterpret_cast<const uint4*>(B + (size_t)n * ldb);
  for (int k8 = lane; k8 < K8; k8 += 32) {
    const uint4 wv = __ldg(wrow + k8);
    const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
    float wf[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(ww[j]);
      wf[2 * j] = f.x;
      wf[2 * j + 1] = f.y;
    }
#pragma unroll
    for (int m = 0; m < 32; ++m) {
      if (m < p.M) {
        const uint4 av = sA4[m * K8 + k8];
        const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(aw[j]);
          acc[m] = fmaf(f.x, wf[2 * j], fmaf(f.y, wf[2 * j + 1], acc[m]));
        }
      }
    }
  }
  float mine = 0.f;
#pragma unroll
  for (int m = 0; m < 32; ++m) {
    if (m < p.M) {
      const float v = warp_sum(acc[m]);
      if (lane == m) mine = v;
    }
  }
  if (lane < p.M) {
    const pg_gemm_epilogue& e = p.epi;
    const int m = lane;
    float t = mine * e.alpha;
    if (e.bias) t += e.bias[n];
    if (p.res_bf16) {
      if (e.res0) t += __bfloat162float(reinterpret_cast<const bf16*>(e.res0)[(size_t)m * e.ld_res + n]);
      if (e.res1) t += __bfloat162float(reinterpret_cast<const bf16*>(e.res1)[(size_t)m * e.ld_res + n]);
    } else {
      if (e.res0) t += e.res0[(size_t)m * e.ld_res + n];
      if (e.res1) t += e.res1[(size_t)m * e.ld_res + n];
    }
    if (e.out_f32) e.out_f32[(size_t)m * e.ld_out_f32 + n] = t;
    if (e.out_pre)
      reinterpret_cast<bf16*>(e.out_pre)[(size_t)m * e.ld_out_pre + n] =
          __float2bfloat16(p.store_deriv ? pg_act_bwd(e.act, t) : t);
    if (e.out_bf16) reinterpret_cast<bf16*>(e.out_bf16)[(size_t)m * e.ld_out_bf16 + n] = __float2bfloat16(pg_act_fwd(e.act, t));
  }
}

// The compile-time epilogue kind of a TMA-epilogue launch (EK_GENERIC when no specialised kind computes exactly its
// epilogue: alpha != 1, bf16 residuals, other activations, accumulation and split-K slices take the generic one).
int epi_kind(const GemmParams& p) {
  const pg_gemm_epilogue& e = p.epi;
  if (!p.epi_tma || e.alpha != 1.f || p.res_bf16 || p.off_old >= 0 || p.splits > 1) return EK_GENERIC;
  const bool bias = e.bias != nullptr, f32 = e.out_f32 != nullptr, bf = e.out_bf16 != nullptr;
  const bool pre = e.out_pre != nullptr, res0 = e.res0 != nullptr, res1 = e.res1 != nullptr;
  const bool no_act = e.act == PG_ACT_NONE && !p.store_deriv;
  if (bf && !f32 && !pre && !res0 && !res1 && no_act && e.dact == PG_ACT_NONE) return bias ? EK_BIAS_BF16 : EK_PLAIN;
  if (bf && !f32 && !pre && !res0 && !res1 && no_act && e.dact == PG_ACT_GIVEN && !bias) return EK_GIVEN_BF16;
  if (bf && pre && !f32 && !res0 && !res1 && bias && e.act == PG_ACT_GELU && p.store_deriv && e.dact == PG_ACT_NONE)
    return EK_BIAS_GELU2;
  if (f32 && !bf && !pre && res0 && bias && no_act && e.dact == PG_ACT_NONE)
    return res1 ? EK_BIAS_RES2_F32 : EK_BIAS_RES_F32;
  return EK_GENERIC;
}

template <int BN, bool A_MN, bool B_MN>
int launch_tc(const void* A, int64_t lda, const void* B, int64_t ldb, GemmParams& p, cudaStream_t stream) {
  CUtensorMap tmA, tmB;
  const ConvGeom& cg = p.conv;
  auto conv_map = [&](CUtensorMap* out, const void* base, int64_t ld, int pixels_per_box) {
    const int64_t n_img = (cg.mode == 1 ? (int64_t)p.M : (int64_t)p.K) / ((int64_t)cg.H * cg.W);
    uint64_t dims[4] = {(uint64_t)cg.C, (uint64_t)cg.W, (uint64_t)cg.H, (uint64_t)n_img};
    uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)cg.W * ld * 2, (uint64_t)cg.H * cg.W * ld * 2};
    uint32_t box[4] = {64, (uint32_t)cg.W, (uint32_t)(pixels_per_box / cg.W), 1};
    return pg_make_tmap_nd_bf16(out, base, 4, dims, strides, box, 1);
  };
  if (cg.mode == 1) {
    if (conv_map(&tmA, A, lda, BM)) return 1;
  } else if (!A_MN) {
    if (pg_make_tmap_2d_bf16(&tmA, A, p.M, p.K, lda, BM, BK)) return 1;
  } else {
    if (pg_make_tmap_2d_bf16(&tmA, A, p.K, p.M, lda, BK, 64)) return 1;
  }
  if (cg.mode == 2) {
    PG_REQUIRE(B_MN && cg.C % BN == 0, "pg_gemm_bf16_conv(wgrad): channels (%d) must be a multiple of the N tile (%d)", cg.C, BN);
    p.conv.nbpt = cg.C / BN;
    if (conv_map(&tmB, B, ldb, BK)) return 1;
  } else if (!B_MN) {
    if (pg_make_tmap_2d_bf16(&tmB, B, p.N, p.K, ldb, BN, BK)) return 1;
  } else if (cg.mode == 1) {  // dgrad: the packed weight [Cout, T * Cin] read K-rows x N-columns, tap t at column t * Cin
    if (pg_make_tmap_2d_bf16(&tmB, B, cg.C, (uint64_t)cg.T * p.N, ldb, BK, 64)) return 1;
  } else {
    if (pg_make_tmap_2d_bf16(&tmB, B, p.K, p.N, ldb, BK, 64)) return 1;
  }
  EpiMaps tmE;
  memset(&tmE, 0, sizeof(tmE));
  if (p.epi_tma) {
    const pg_gemm_epilogue& e = p.epi;
    auto f32_map = [&](CUtensorMap* out, const void* base, int64_t ld) {
      return pg_make_tmap_2d(out, base, 4, p.M, p.N, ld, 16, 32, 128);
    };
    auto bf16_map = [&](CUtensorMap* out, const void* base, int64_t ld) {
      return pg_make_tmap_2d(out, base, 2, p.M, p.N, ld, 16, 32, 64);
    };
    if (e.res0 && (p.res_bf16 ? bf16_map(&tmE.res0, e.res0, e.ld_res) : f32_map(&tmE.res0, e.res0, e.ld_res))) return 1;
    if (e.res1 && (p.res_bf16 ? bf16_map(&tmE.res1, e.res1, e.ld_res) : f32_map(&tmE.res1, e.res1, e.ld_res))) return 1;
    if (p.off_aux >= 0 && bf16_map(&tmE.aux, e.aux, e.ld_aux)) return 1;
    if (e.out_pre && bf16_map(&tmE.out_pre, e.out_pre, e.ld_out_pre)) return 1;
    if (e.out_bf16 && bf16_map(&tmE.out_bf16, e.out_bf16, e.ld_out_bf16)) return 1;
    if (e.out_f32) {  // split-K: the [splits][M][N] slices; otherwise out_f32 itself
      const float* base = p.split_part ? p.split_part : e.out_f32;
      const uint64_t ld = p.split_part ? (uint64_t)p.N : (uint64_t)e.ld_out_f32;
      const uint64_t dims[3] = {(uint64_t)p.N, (uint64_t)p.M, (uint64_t)p.splits};
      const uint64_t strides[2] = {ld * 4, ld * 4 * (uint64_t)p.M};
      const uint32_t box[3] = {32, 16, 1};
      if (pg_make_tmap_nd(&tmE.out_f32, base, 4, 3, dims, strides, box, 128)) return 1;
    }
    if (e.bias) {
      const uint64_t dims[1] = {(uint64_t)p.N};
      const uint32_t box[1] = {(uint32_t)BN};
      if (pg_make_tmap_nd(&tmE.bias, e.bias, 4, 1, dims, nullptr, box, 0)) return 1;
    }
  }
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * BK * 2;
  const int fixed = 1024 /*align slack*/ + (2 * MAX_STAGES + 8 * MAX_EPI_BUFS + 2) * 8 /*barriers*/ +
                    16 * 8 * 4 /*row-sum exchange*/;
  const int avail = SMEM_LIMIT - fixed;
  if (p.epi_tma) {
    // Staging buffers first, as many as leave four stages (up to MAX_EPI_BUFS per warp, no more than the tile's
    // sub-tiles): with nb buffers the inputs are requested nb - 1 sub-tiles ahead.  At BN = 128 that is 5 stages with
    // 4 buffers of 2 KB per warp (a fp32 input or output), 4 stages with 3 buffers of 4 KB (two fp32 residuals).
    const int bufs_room = (avail - 2 * EPI_BIAS_BYTES - 4 * STAGE_BYTES) / (8 * p.epi_buf_bytes);
    p.epi_nbuf = min(min(MAX_EPI_BUFS, 2 * (BN / 32)), max(2, bufs_room));
    p.epi_smem = 8 * p.epi_nbuf * p.epi_buf_bytes + 2 * EPI_BIAS_BYTES;
  } else {
    p.epi_nbuf = 0;
    p.epi_smem = 2 * XP_BYTES;
  }
  int stages = (avail - p.epi_smem) / STAGE_BYTES;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  if (stages > p.k_iters + 1) stages = p.k_iters + 1 > 2 ? p.k_iters + 1 : 2;
  PG_REQUIRE(stages >= 2, "pg_gemm_bf16: %d bytes of epilogue staging leave no room for two pipeline stages",
             p.epi_smem);
  p.stages = stages;
  const int smem_bytes = stages * STAGE_BYTES + p.epi_smem + fixed;
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_GENERIC>;
  if constexpr (BN == 128 && !A_MN) {
    switch (epi_kind(p)) {
      case EK_PLAIN: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_PLAIN>; break;
      case EK_BIAS_BF16: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_BIAS_BF16>; break;
      case EK_BIAS_GELU2: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_BIAS_GELU2>; break;
      case EK_GIVEN_BF16: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_GIVEN_BF16>; break;
      case EK_BIAS_RES_F32: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_BIAS_RES_F32>; break;
      case EK_BIAS_RES2_F32: kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EK_BIAS_RES2_F32>; break;
      default: break;
    }
  }
  PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  const int num_tiles = p.num_m_blk * p.num_n_blk * p.splits;
  const int grid = min(num_tiles, pg_num_sms());
  kern<<<grid, GEMM_THREADS, smem_bytes, stream>>>(tmA, tmB, tmE, p);
  if (pg_check_launch("pg_gemm_bf16(wgmma)")) return 1;
  if (p.split_part &&
      pg_sum_partials(p.split_part, p.splits, (long long)p.M * p.N, p.M, p.N, p.epi.ld_out_f32, p.epi.out_f32, stream))
    return 1;
  if (p.rowsum_part && pg_sum_partials(p.rowsum_part, p.splits, p.M, 1, p.M, p.M, p.a_rowsum, stream)) return 1;
  return 0;
}

template <bool A_MN, bool B_MN>
int dispatch_bn(const void* A, int64_t lda, const void* B, int64_t ldb, GemmParams& p, cudaStream_t stream) {
  // Tile width: the smallest of {32, 64, 128} covering N, 128 beyond (128 x 128 fp32 accumulators per consumer
  // warpgroup leave registers for the epilogue).
  int bn;
  if (p.N > 64) bn = 128;
  else if (p.N > 32) bn = 64;
  else bn = 32;
  if (!p.epi_tma && bn > 64) bn = 64;  // the row-segment epilogue is built for BN <= 64 only
  if (B_MN && bn < 64) bn = 64;  // MN-major operands are staged in 64-wide swizzle atoms
  if (p.conv.mode == 2) bn = (p.conv.C % 128 == 0 && p.epi_tma) ? 128 : 64;  // taps are whole N blocks
  p.num_n_blk = (p.N + bn - 1) / bn;
  switch (bn) {
    case 128: return launch_tc<128, A_MN, B_MN>(A, lda, B, ldb, p, stream);
    case 64: return launch_tc<64, A_MN, B_MN>(A, lda, B, ldb, p, stream);
    default: return launch_tc<32, A_MN, B_MN>(A, lda, B, ldb, p, stream);
  }
}

}  // namespace

static int gemm_entry(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb, int M, int N,
                      int K, int split_k, const pg_gemm_epilogue* epi, int impl, const ConvGeom* conv, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(A && B && epi, "pg_gemm_bf16: null operand");
  PG_REQUIRE(M > 0 && N > 0 && K > 0, "pg_gemm_bf16: empty problem M=%d N=%d K=%d", M, N, K);
  PG_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "pg_gemm_bf16: pitches must be multiples of 8 elements (lda=%lld ldb=%lld)",
             (long long)lda, (long long)ldb);
  PG_REQUIRE(epi->out_bf16 || epi->out_pre || epi->out_f32, "pg_gemm_bf16: no output requested");
  PG_REQUIRE(epi->dact == PG_ACT_NONE || epi->aux, "pg_gemm_bf16: dact needs aux");
  if (split_k < 1) split_k = 1;
  if (split_k > 1)
    PG_REQUIRE(epi->accumulate && epi->out_f32 && !epi->out_bf16 && !epi->out_pre && epi->dact == PG_ACT_NONE &&
                   !epi->bias && !epi->res0 && !epi->res1,
               "pg_gemm_bf16: split_k > 1 requires accumulate=1 into out_f32 only (no bias / residuals)");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  if (conv) p.conv = *conv;
  p.M = M; p.N = N; p.K = K;
  p.num_m_blk = (M + BM - 1) / BM;
  p.num_n_blk = 0;
  p.k_iters = (K + BK - 1) / BK;
  if (split_k > p.k_iters) split_k = p.k_iters;
  p.k_per_split = (p.k_iters + split_k - 1) / split_k;
  p.splits = (p.k_iters + p.k_per_split - 1) / p.k_per_split;  // no empty split
  p.epi = *epi;
  p.store_deriv = (epi->act & PG_ACT_STORE_DERIV) ? 1 : 0;
  p.res_bf16 = (epi->act & PG_ACT_RES_BF16) ? 1 : 0;
  p.epi.act = epi->act & 0xff;
  p.a_rowsum = epi->bias_grad;
  PG_REQUIRE(!epi->bias_grad || (a_mn_major && impl == 0),
             "pg_gemm_bf16: bias_grad rides on the weight-gradient GEMM (a_mn_major = 1, impl 0)");
  PG_REQUIRE(!p.store_deriv || epi->out_pre, "pg_gemm_bf16: PG_ACT_STORE_DERIV needs out_pre");
  // TMA addresses a tensor from a 16-byte aligned base with a pitch of a multiple of 16 bytes
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool vec_ok = true;
  if (epi->bias && !al16(epi->bias)) vec_ok = false;
  const bool aux = epi->dact != PG_ACT_NONE;
  if (aux && (!al16(epi->aux) || epi->ld_aux % 8)) vec_ok = false;
  const int res_mult = p.res_bf16 ? 8 : 4;
  if (epi->res0 && (!al16(epi->res0) || epi->ld_res % res_mult)) vec_ok = false;
  if (epi->res1 && (!al16(epi->res1) || epi->ld_res % res_mult)) vec_ok = false;
  if (epi->out_f32 && (!al16(epi->out_f32) || epi->ld_out_f32 % 4)) vec_ok = false;
  if (epi->out_pre && (!al16(epi->out_pre) || epi->ld_out_pre % 8)) vec_ok = false;
  if (epi->out_bf16 && (!al16(epi->out_bf16) || epi->ld_out_bf16 % 8)) vec_ok = false;
  // A TMA store writes whole 16-byte pieces of a row: with rows of N elements that end inside one, it would write up
  // to 3 (fp32) or 7 (bf16) elements past N.  N % 8 == 0 also makes the [M][N] fp32 split-K slices addressable.
  if (N % 8) vec_ok = false;
  p.epi_tma = vec_ok ? 1 : 0;
  // Staging-buffer layout of the TMA epilogue: the sub-tile's inputs from offset 0, and its outputs from offset 0 too
  // (they are written once every thread has read the inputs).
  p.off_old = p.off_res0 = p.off_res1 = p.off_aux = p.off_f32 = p.off_pre = p.off_bf16 = -1;
  if (p.epi_tma) {
    const int res_bytes = p.res_bf16 ? EPI_BF16_BYTES : EPI_F32_BYTES;
    int in = 0, out = 0;
    if (epi->accumulate && epi->out_f32 && p.splits == 1) { p.off_old = in; in += EPI_F32_BYTES; }
    if (epi->res0) { p.off_res0 = in; in += res_bytes; }
    if (epi->res1) { p.off_res1 = in; in += res_bytes; }
    if (aux) { p.off_aux = in; in += EPI_BF16_BYTES; }
    if (epi->out_f32) { p.off_f32 = out; out += EPI_F32_BYTES; }
    if (epi->out_pre) { p.off_pre = out; out += EPI_BF16_BYTES; }
    if (epi->out_bf16) { p.off_bf16 = out; out += EPI_BF16_BYTES; }
    p.epi_in_bytes = in;
    p.epi_buf_bytes = in > out ? in : out;
  }

  if (impl == 1) {
    p.splits = 1;
    p.k_per_split = p.k_iters;
    const int nseg = (N + 31) / 32;
    const long long total = (long long)M * nseg;
    const int threads = 128;
    const long long blocks = (total + threads - 1) / threads;
    gemm_simt_kernel<<<(unsigned)blocks, threads, 0, stream>>>(reinterpret_cast<const bf16*>(A), a_mn_major, lda,
                                                                 reinterpret_cast<const bf16*>(B), b_mn_major, ldb, p);
    return pg_check_launch("pg_gemm_bf16(simt)");
  }
  if (impl == 2) {
    // explicit opt-in (incremental sampling): never chosen implicitly, so forward() keeps one summation order
    // whatever the number of rows
    PG_REQUIRE(!a_mn_major && !b_mn_major && M <= 32 && !epi->accumulate && epi->dact == PG_ACT_NONE && K % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                   (size_t)M * K * 2 <= 160 * 1024,
               "pg_gemm_bf16(skinny): needs a K-major forward GEMM with M <= 32 rows (M=%d K=%d)", M, K);
    const size_t smem = (size_t)M * K * 2;
    PG_CUDA(cudaFuncSetAttribute(gemm_skinny_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    gemm_skinny_kernel<<<(N + 7) / 8, 256, smem, stream>>>(reinterpret_cast<const bf16*>(A), lda,
                                                           reinterpret_cast<const bf16*>(B), ldb, p);
    return pg_check_launch("pg_gemm_bf16(skinny)");
  }
  if (p.splits > 1) {  // fixed-order split-K: slices in the scratch buffer (split_k > 1 implies pure accumulation)
    const size_t mn = (size_t)M * N, rows = p.a_rowsum ? (size_t)M : 0;
    float* part = nullptr;
    if (pg_scratch((size_t)p.splits * (mn + rows) * sizeof(float), stream, &part)) return 1;
    p.split_part = part;
    if (p.a_rowsum) p.rowsum_part = part + (size_t)p.splits * mn;
  }
  if (!a_mn_major && !b_mn_major) return dispatch_bn<false, false>(A, lda, B, ldb, p, stream);
  if (!a_mn_major && b_mn_major) return dispatch_bn<false, true>(A, lda, B, ldb, p, stream);
  if (a_mn_major && b_mn_major) return dispatch_bn<true, true>(A, lda, B, ldb, p, stream);
  return dispatch_bn<true, false>(A, lda, B, ldb, p, stream);
}

extern "C" int pg_gemm_bf16(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                            int M, int N, int K, int split_k, const pg_gemm_epilogue* epi, int impl, void* stream_) {
  return gemm_entry(A, a_mn_major, lda, B, b_mn_major, ldb, M, N, K, split_k, epi, impl, nullptr, stream_);
}

// Tap-loop convolution on the same kernel (see ConvGeom): forward / dgrad read the activation (or output-gradient)
// tensor under each tap's shift, wgrad reads the shifted activations as its B operand.
extern "C" int pg_gemm_bf16_conv_taps(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K,
                                      int split_k, const pg_gemm_epilogue* epi, int mode, int n_img, int H, int W, int C,
                                      int n_taps, const int* dy, const int* dx, void* stream_) {
  PG_REQUIRE(mode >= PG_CONV_FWD && mode <= PG_CONV_WGRAD, "pg_gemm_bf16_conv: mode %d", mode);
  PG_REQUIRE(n_taps >= 1 && n_taps <= MAX_CONV_TAPS, "pg_gemm_bf16_conv: 1..%d taps (got %d)", MAX_CONV_TAPS, n_taps);
  PG_REQUIRE(dy && dx, "pg_gemm_bf16_conv: null tap offsets");
  PG_REQUIRE(C % 64 == 0 && W >= 1 && W <= 64 && 64 % W == 0 && ((int64_t)H * W) % 128 == 0,
             "pg_gemm_bf16_conv: needs C %% 64 == 0, W | 64 and H*W %% 128 == 0 (C=%d H=%d W=%d); use pg_tap_gather otherwise",
             C, H, W);
  const int64_t P = (int64_t)n_img * H * W;
  ConvGeom cg;
  memset(&cg, 0, sizeof(cg));
  cg.H = H; cg.W = W; cg.C = C; cg.T = n_taps;
  cg.cslabs = C / 64;
  for (int t = 0; t < n_taps; ++t) {
    PG_REQUIRE(dy[t] >= -64 && dy[t] <= 64 && dx[t] >= -64 && dx[t] <= 64, "pg_gemm_bf16_conv: tap offset out of range");
    cg.dy[t] = (int8_t)dy[t];
    cg.dx[t] = (int8_t)dx[t];
  }
  if (mode == PG_CONV_WGRAD) {
    // dW[cout, t*C + c] += sum_p dY[p, cout] * X[p + off_t, c]:  A = dY (MN-major), B = X (shifted), K = pixels
    PG_REQUIRE(K == P && N == n_taps * C, "pg_gemm_bf16_conv(wgrad): K must be N*H*W and N = taps * C");
    cg.mode = 2;
    return gemm_entry(A, 1, lda, B, 1, ldb, M, N, K, split_k, epi, 0, &cg, stream_);
  }
  // forward: A = X (shifted), B = W [Cout, T*C] K-major.  dgrad: A = dY (shifted by -off), B = W [C, T*N] read MN-major.
  PG_REQUIRE(M == P && K == n_taps * C, "pg_gemm_bf16_conv: M must be N*H*W and K = taps * C");
  cg.mode = 1;
  return gemm_entry(A, 0, lda, B, mode == PG_CONV_DGRAD ? 1 : 0, ldb, M, N, K, split_k, epi, 0, &cg, stream_);
}

// The same launch with the geometry in a pg_conv_geom, whose offset arrays hold 32 taps.
extern "C" int pg_gemm_bf16_conv(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, int split_k,
                                 const pg_gemm_epilogue* epi, const pg_conv_geom* g, void* stream_) {
  PG_REQUIRE(g, "pg_gemm_bf16_conv: null geometry");
  PG_REQUIRE(g->n_taps >= 1 && g->n_taps <= 32, "pg_gemm_bf16_conv: 1..32 taps in a pg_conv_geom (got %d)", g->n_taps);
  return pg_gemm_bf16_conv_taps(A, lda, B, ldb, M, N, K, split_k, epi, g->mode, g->N, g->H, g->W, g->C, g->n_taps, g->dy,
                                g->dx, stream_);
}
