// pg_nade.cu — NADE (reference models/autoregressive/nade.py): the scan over the input dimensions that gives every
// conditional probability (training, forward with entries to draw, and sampling in one launch) and its reverse scan for
// the gradients.  fp32 on the CUDA cores; every reduction runs in a fixed order and there are no atomics.
//
// Per image, with x~ the effective input (x where x >= 0, a Bernoulli draw (u < p_d) where x < 0):
//   a_0 = in_b,   a_d = a_{d-1} + x~_{d-1} in_W[:, d-1],   p_d = sigmoid(h_W[d] . relu(a_d) + h_b[d]).
// `a` is accumulated in index order with a separately rounded multiply and add, the reference's own arithmetic
// (`x_i @ W[:, i].t()` is one product, then `a + ...`), so the hidden pre-activations carry the reference's bits; only
// the H-long dot is summed in another (fixed) order.
#include "pg_common.cuh"

namespace {

constexpr int T = PG_NADE_CHUNK;  // dimensions per checkpoint of `a` (and per chunk of the reverse scan)
constexpr int UMAX = 16;          // hidden units a thread keeps in registers in the forward scan
constexpr int BWD_THREADS = 128;  // hidden units per CTA of the reverse scan (one per thread)
constexpr int BWD_MAX_TILES = 16; // image tiles of the reverse scan: bounds the weight-gradient partials

// winT[d, h] = in_w[h, d]: the scan reads one contiguous row of in_W^T per dimension.
__global__ void nade_transpose_kernel(const float* __restrict__ in_w, int H, int D, float* __restrict__ winT) {
  __shared__ float tile[32][33];
  const int d0 = blockIdx.x * 32, h0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int h = h0 + r, d = d0 + threadIdx.x;
    if (h < H && d < D) tile[r][threadIdx.x] = in_w[(size_t)h * D + d];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int d = d0 + r, h = h0 + threadIdx.x;
    if (h < H && d < D) winT[(size_t)d * H + h] = tile[threadIdx.x][r];
  }
}

// One image per TPI threads (a power of two >= 32); thread t keeps a[h] for h = t, t + TPI, ... (at most UMAX) in
// registers and walks d = 0 .. D-1.  The logit of step d is complete (a fixed butterfly per warp, then the image's warps
// in index order through shared memory) before `a` takes x~_d, so entries < 0 are drawn inside the scan.  An image's
// arithmetic does not depend on the other images of the batch or on the grid.
template <int TPI>
__global__ void __launch_bounds__(TPI < 64 ? 64 : TPI) nade_scan_kernel(
    const float* __restrict__ x, const float* __restrict__ u, const float* __restrict__ winT,
    const float* __restrict__ in_b, const float* __restrict__ h_w, const float* __restrict__ h_b, int n, int D, int H,
    float* __restrict__ p, float* __restrict__ xt, float* __restrict__ ckpt) {
  constexpr int WPI = TPI / 32;
  __shared__ float red[2][WPI];
  const int t = threadIdx.x % TPI, img = blockIdx.x * (blockDim.x / TPI) + threadIdx.x / TPI;
  const bool live = img < n;  // a CTA's spare image slot still meets its barriers
  const int mine = t < H ? (H - t + TPI - 1) / TPI : 0;  // this thread's hidden units
  const int nch = (D + T - 1) / T;
  float a[UMAX];
#pragma unroll
  for (int j = 0; j < UMAX; ++j) a[j] = j < mine ? in_b[t + j * TPI] : 0.f;
  const float* xr = x + (size_t)img * D;
  const float* ur = u + (size_t)img * D;
  for (int d = 0; d < D; ++d) {
    if (ckpt && live && d % T == 0) {
      float* cr = ckpt + ((size_t)img * nch + d / T) * H + t;
#pragma unroll
      for (int j = 0; j < UMAX; ++j)
        if (j < mine) cr[j * TPI] = a[j];
    }
    const float* whr = h_w + (size_t)d * H + t;
    float s0 = 0.f, s1 = 0.f;  // two chains: even and odd j
#pragma unroll
    for (int j = 0; j < UMAX; j += 2) {
      if (j < mine) s0 = fmaf(fmaxf(a[j], 0.f), __ldg(whr + j * TPI), s0);
      if (j + 1 < mine) s1 = fmaf(fmaxf(a[j + 1], 0.f), __ldg(whr + (j + 1) * TPI), s1);
    }
    float z = warp_sum(s0 + s1);
    if (WPI > 1) {
      if ((threadIdx.x & 31) == 0) red[d & 1][t / 32] = z;
      __syncthreads();  // double-buffered: one barrier per step
      z = 0.f;
#pragma unroll
      for (int w = 0; w < WPI; ++w) z += red[d & 1][w];
    }
    const float pd = 1.f / (1.f + expf(-(z + h_b[d])));
    float xv = 0.f;
    if (live) {
      xv = xr[d];
      if (xv < 0.f) xv = ur[d] < pd ? 1.f : 0.f;
      if (t == 0) {
        if (p) p[(size_t)img * D + d] = pd;
        xt[(size_t)img * D + d] = xv;
      }
    }
    const float* wr = winT + (size_t)d * H + t;
#pragma unroll
    for (int j = 0; j < UMAX; ++j)
      if (j < mine) a[j] = __fadd_rn(a[j], __fmul_rn(xv, __ldg(wr + j * TPI)));
  }
}

// Layers wider than 1024 * UMAX units: one image per CTA of 1024 threads, `a` in a global row of the library's scratch
// (each thread reads and writes only its own units h = t, t + 1024, ..., so no barrier guards it).  Same arithmetic
// and the same order of the draw as nade_scan_kernel; the dot is summed per thread, per warp, then over the 32 warps.
__global__ void __launch_bounds__(1024) nade_scan_wide_kernel(
    const float* __restrict__ x, const float* __restrict__ u, const float* __restrict__ winT,
    const float* __restrict__ in_b, const float* __restrict__ h_w, const float* __restrict__ h_b, int D, int H,
    float* __restrict__ abuf, float* __restrict__ p, float* __restrict__ xt, float* __restrict__ ckpt) {
  __shared__ float red[2][32];
  const int t = threadIdx.x, img = blockIdx.x, nch = (D + T - 1) / T;
  float* ar = abuf + (size_t)img * H;
  for (int h = t; h < H; h += 1024) ar[h] = in_b[h];
  for (int d = 0; d < D; ++d) {
    if (ckpt && d % T == 0) {
      float* cr = ckpt + ((size_t)img * nch + d / T) * H;
      for (int h = t; h < H; h += 1024) cr[h] = ar[h];
    }
    const float* whr = h_w + (size_t)d * H;
    float z = 0.f;
    for (int h = t; h < H; h += 1024) z = fmaf(fmaxf(ar[h], 0.f), __ldg(whr + h), z);
    z = warp_sum(z);
    if ((t & 31) == 0) red[d & 1][t / 32] = z;
    __syncthreads();  // double-buffered: one barrier per step
    z = 0.f;
#pragma unroll
    for (int w = 0; w < 32; ++w) z += red[d & 1][w];
    const float pd = 1.f / (1.f + expf(-(z + h_b[d])));
    float xv = x[(size_t)img * D + d];
    if (xv < 0.f) xv = u[(size_t)img * D + d] < pd ? 1.f : 0.f;
    if (t == 0) {
      if (p) p[(size_t)img * D + d] = pd;
      xt[(size_t)img * D + d] = xv;
    }
    const float* wr = winT + (size_t)d * H;
    for (int h = t; h < H; h += 1024) ar[h] = __fadd_rn(ar[h], __fmul_rn(xv, __ldg(wr + h)));
  }
}

struct NadeBwd {
  const float *x, *xt, *p, *g, *ckpt, *in_w, *h_w;
  int n, D, H, nt, slices, nch;
  float *s, *phw, *pinw, *phb, *pinb, *pdx;  // pg_scratch
};

// One CTA per (image tile, slice of 128 hidden units); thread = hidden unit h.  Chunks of T dimensions in reverse: the
// chunk's `a` is recomputed from its checkpoint in registers (the forward's exact arithmetic), then walked backwards
// carrying s = sum_{d > i} da_d, da_d = gz_d h_W[d] [a_d > 0], gz = g (1 - p) p.  The tile's images are visited in
// order, so each partial below is a sum over images in a fixed order:
//   phw[tile][d][h]  = sum gz[n,d] relu(a[n,d,h])       pinw[tile][h][i] = sum x~[n,i] s_i[n,h]
//   phb[tile][d]     = sum gz[n,d]                      pinb[tile][h]    = sum s_{-1}[n,h]
//   pdx[slice][n][i] = sum over the slice's h of in_W[h,i] s_i[n,h] (a butterfly per warp, then the 4 warps), 0 where
//                      x[n,i] < 0
// s[n][h] carries each image's running sum from one chunk to the next.
__global__ void __launch_bounds__(BWD_THREADS) nade_bwd_kernel(NadeBwd a) {
  __shared__ float red[2][BWD_THREADS / 32][T];
  const int tile = blockIdx.x / a.slices, slice = blockIdx.x % a.slices;
  const int h = slice * BWD_THREADS + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool hv = h < a.H;
  const int n0 = tile * a.nt, n1 = min(a.n, n0 + a.nt);
  const int D = a.D, H = a.H;
  int buf = 0;
  for (int c = a.nch - 1; c >= 0; --c) {
    const int c0 = c * T, len = min(T, D - c0);
    float win[T], wh[T], dhw[T], dinw[T];
#pragma unroll
    for (int j = 0; j < T; ++j) {
      const bool ok = hv && j < len;
      win[j] = ok ? a.in_w[(size_t)h * D + c0 + j] : 0.f;
      wh[j] = ok ? a.h_w[(size_t)(c0 + j) * H + h] : 0.f;
      dhw[j] = 0.f;
      dinw[j] = 0.f;
    }
    for (int img = n0; img < n1; ++img) {
      const size_t row = (size_t)img * D + c0;
      const float* xr = a.xt + row;
      float s = (hv && c + 1 < a.nch) ? a.s[(size_t)img * H + h] : 0.f;
      float ah[T];
      ah[0] = hv ? a.ckpt[((size_t)img * a.nch + c) * H + h] : 0.f;
#pragma unroll
      for (int j = 1; j < T; ++j) ah[j] = j < len ? __fadd_rn(ah[j - 1], __fmul_rn(xr[j - 1], win[j - 1])) : 0.f;
      float dxv[T];
#pragma unroll
      for (int j = T - 1; j >= 0; --j) {
        dxv[j] = 0.f;
        if (j < len) {
          const float pd = a.p[row + j];
          const float gz = (a.g[row + j] * (1.f - pd)) * pd;
          dinw[j] = fmaf(xr[j], s, dinw[j]);
          dxv[j] = win[j] * s;
          dhw[j] = fmaf(gz, fmaxf(ah[j], 0.f), dhw[j]);
          if (ah[j] > 0.f) s += gz * wh[j];
        }
      }
      if (hv) a.s[(size_t)img * H + h] = s;
      if (a.pdx) {
        // reduce-scatter of the 16 values over the warp: lanes 2k and 2k+1 end with the warp's sum for j = k
#pragma unroll
        for (int w = T / 2, o = 16; w >= 1; w >>= 1, o >>= 1) {
          const bool hi = lane & o;
#pragma unroll
          for (int k = 0; k < w; ++k) {
            const float send = hi ? dxv[k] : dxv[k + w];
            const float keep = hi ? dxv[k + w] : dxv[k];
            dxv[k] = keep + __shfl_xor_sync(0xffffffffu, send, o);
          }
        }
        dxv[0] += __shfl_xor_sync(0xffffffffu, dxv[0], 1);
        if ((lane & 1) == 0) red[buf][warp][lane >> 1] = dxv[0];
        __syncthreads();  // double-buffered: one barrier per image and chunk
        if (threadIdx.x < len) {
          float v = 0.f;
#pragma unroll
          for (int w = 0; w < BWD_THREADS / 32; ++w) v += red[buf][w][threadIdx.x];
          if (a.x[row + threadIdx.x] < 0.f) v = 0.f;
          a.pdx[((size_t)slice * a.n + img) * D + c0 + threadIdx.x] = v;
        }
        buf ^= 1;
      }
    }
    if (hv) {
#pragma unroll
      for (int j = 0; j < T; ++j) {
        if (j < len) {
          a.phw[((size_t)tile * D + c0 + j) * H + h] = dhw[j];
          a.pinw[((size_t)tile * H + h) * D + c0 + j] = dinw[j];
        }
      }
    }
    if (slice == 0 && threadIdx.x < len) {
      float v = 0.f;
      for (int img = n0; img < n1; ++img) {
        const size_t at = (size_t)img * D + c0 + threadIdx.x;
        v += (a.g[at] * (1.f - a.p[at])) * a.p[at];
      }
      a.phb[(size_t)tile * D + c0 + threadIdx.x] = v;
    }
  }
  if (hv) {
    float v = 0.f;
    for (int img = n0; img < n1; ++img) v += a.s[(size_t)img * H + h];
    a.pinb[(size_t)tile * H + h] = v;
  }
}

template <int TPI>
int launch_scan(const float* x, const float* u, const float* winT, const float* in_b, const float* h_w, const float* h_b,
                int n, int D, int H, float* p, float* xt, float* ckpt, cudaStream_t stream) {
  constexpr int threads = TPI < 64 ? 64 : TPI, per_cta = threads / TPI;
  const long long blocks = ((long long)n + per_cta - 1) / per_cta;
  PG_REQUIRE(blocks < (1LL << 31), "pg_nade_fwd: grid of %lld CTAs", blocks);
  nade_scan_kernel<TPI><<<(unsigned)blocks, threads, 0, stream>>>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt);
  return pg_check_launch("pg_nade_fwd");
}

}  // namespace

extern "C" int pg_nade_fwd(const float* x, const float* u, const float* in_w, const float* in_b, const float* h_w,
                           const float* h_b, int n, int D, int H, float* p, float* xt, float* ckpt, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D > 0 && H > 0, "pg_nade_fwd: empty problem (n %d, D %d, H %d)", n, D, H);
  if (n == 0) return 0;  // an empty batch (its tensors may have no storage)
  PG_REQUIRE(x && u && in_w && in_b && h_w && h_b && xt, "pg_nade_fwd: null argument");
  const bool wide = H > 1024 * UMAX;
  float* winT = nullptr;
  if (pg_scratch((size_t)D * H * sizeof(float) + (wide ? (size_t)n * H * sizeof(float) : 0), stream, &winT)) return 1;
  nade_transpose_kernel<<<dim3((D + 31) / 32, (H + 31) / 32), dim3(32, 8), 0, stream>>>(in_w, H, D, winT);
  if (pg_check_launch("pg_nade_fwd(transpose)")) return 1;
  if (wide) {
    nade_scan_wide_kernel<<<n, 1024, 0, stream>>>(x, u, winT, in_b, h_w, h_b, D, H, winT + (size_t)D * H, p, xt, ckpt);
    return pg_check_launch("pg_nade_fwd");
  }
  // the fewest threads per image that hold H in UMAX registers a thread
  const int warps = (H + 32 * UMAX - 1) / (32 * UMAX);
  if (warps <= 1) return launch_scan<32>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
  if (warps <= 2) return launch_scan<64>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
  if (warps <= 4) return launch_scan<128>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
  if (warps <= 8) return launch_scan<256>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
  if (warps <= 16) return launch_scan<512>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
  return launch_scan<1024>(x, u, winT, in_b, h_w, h_b, n, D, H, p, xt, ckpt, stream);
}

extern "C" int pg_nade_bwd(const float* x, const float* xt, const float* p, const float* g, const float* ckpt,
                           const float* in_w, const float* h_w, int n, int D, int H, float* d_in_w, float* d_in_b,
                           float* d_h_w, float* d_h_b, float* dx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(n >= 0 && D > 0 && H > 0, "pg_nade_bwd: empty problem (n %d, D %d, H %d)", n, D, H);
  if (n == 0) return 0;  // the gradients of an empty batch: nothing to add
  PG_REQUIRE(x && xt && p && g && ckpt && in_w && h_w && d_in_w && d_in_b && d_h_w && d_h_b,
             "pg_nade_bwd: null argument");
  NadeBwd a{x, xt, p, g, ckpt, in_w, h_w, n, D, H, 0, (H + BWD_THREADS - 1) / BWD_THREADS, (D + T - 1) / T};
  int tiles = (n + 31) / 32;
  if (tiles > BWD_MAX_TILES) tiles = BWD_MAX_TILES;
  a.nt = (n + tiles - 1) / tiles;
  tiles = (n + a.nt - 1) / a.nt;
  const size_t nD = (size_t)n * D, DH = (size_t)D * H;
  const size_t floats = (size_t)n * H + 2 * tiles * DH + (size_t)tiles * (D + H) + (dx ? a.slices * nD : 0);
  float* scratch = nullptr;
  if (pg_scratch(floats * sizeof(float), stream, &scratch)) return 1;
  a.s = scratch;
  a.phw = a.s + (size_t)n * H;
  a.pinw = a.phw + tiles * DH;
  a.phb = a.pinw + tiles * DH;
  a.pinb = a.phb + (size_t)tiles * D;
  a.pdx = dx ? a.pinb + (size_t)tiles * H : nullptr;
  nade_bwd_kernel<<<(unsigned)(tiles * a.slices), BWD_THREADS, 0, stream>>>(a);
  if (pg_check_launch("pg_nade_bwd")) return 1;
  if (pg_sum_partials(a.phw, tiles, (long long)DH, D, H, H, d_h_w, stream)) return 1;
  if (pg_sum_partials(a.pinw, tiles, (long long)DH, H, D, D, d_in_w, stream)) return 1;
  if (pg_sum_partials(a.phb, tiles, D, 1, D, D, d_h_b, stream)) return 1;
  if (pg_sum_partials(a.pinb, tiles, H, 1, H, H, d_in_b, stream)) return 1;
  if (dx && pg_sum_partials(a.pdx, a.slices, (long long)nD, n, D, D, dx, stream)) return 1;
  return 0;
}
