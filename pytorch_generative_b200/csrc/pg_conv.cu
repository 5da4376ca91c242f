// pg_conv.cu — CausalConv2d input layers with tiny Cin (1 or 3 image channels):
// reference nn/convolution.py:41-43 called from pixel_cnn.py:86-92, pixel_snail.py:155-161,
// image_gpt.py:87-93.  K = Cin*kh*kw is 9..49, far below a tensor-core K slab, and the layer is
// <= 0.01 % of the step's FLOPs at the ImageGPT/PixelSNAIL configs, so this is a direct CUDA-core kernel
// that reads the NCHW fp32 image and writes the pixel-major activation the GEMM path consumes.
// Masked taps are zero in `w` (the caller zeroes the Parameter in place, as the reference does), so the
// forward simply runs all kh*kw taps; wgrad is dense over the taps, matching autograd in the reference.
#include "../../include/pg_b200.h"
#include "pg_common.cuh"

namespace {

constexpr int PIX_PER_BLOCK = 32;
constexpr int MAX_K = 160;  // Cin*kh*kw upper bound (3*7*7 = 147)

struct ConvArgs {
  int N, Cin, H, W, Cout, kh, kw, ph, pw, K;
  int dh, dw;   // dilation: kernel position (i, j) reads the input at (y + i*dh - ph, x + j*dw - pw)
  int pre_act;  // activation applied to the input before the convolution (act(0) = 0, so it commutes with padding)
};

// Gathers the K-vector of input values under the kernel window of pixel p (zero padding).
__device__ __forceinline__ float patch_value(const float* __restrict__ x, const ConvArgs& a, int n, int y, int xx, int k) {
  const int ci = k / (a.kh * a.kw);
  const int r = k % (a.kh * a.kw);
  const int i = r / a.kw, j = r % a.kw;
  const int yy = y + i * a.dh - a.ph, xc = xx + j * a.dw - a.pw;
  if (yy < 0 || yy >= a.H || xc < 0 || xc >= a.W) return 0.f;
  return pg_act_fwd(a.pre_act, x[(((size_t)n * a.Cin + ci) * a.H + yy) * a.W + xc]);
}

__global__ void __launch_bounds__(256)
conv_small_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                      const ConvArgs a, float* __restrict__ out_f32, bf16* __restrict__ out_bf16, int act_bf16) {
  __shared__ float patch[PIX_PER_BLOCK][MAX_K + 1];
  const int HW = a.H * a.W;
  const long long P = (long long)a.N * HW;
  const long long p0 = (long long)blockIdx.x * PIX_PER_BLOCK;
  for (int t = threadIdx.x; t < PIX_PER_BLOCK * a.K; t += blockDim.x) {
    const int pi = t / a.K, k = t % a.K;
    const long long p = p0 + pi;
    float v = 0.f;
    if (p < P) {
      const int n = (int)(p / HW), rem = (int)(p % HW);
      v = patch_value(x, a, n, rem / a.W, rem % a.W, k);
    }
    patch[pi][k] = v;
  }
  __syncthreads();
  for (int co = threadIdx.x; co < a.Cout; co += blockDim.x) {
    float acc[PIX_PER_BLOCK];
    const float b = bias ? bias[co] : 0.f;
#pragma unroll
    for (int pi = 0; pi < PIX_PER_BLOCK; ++pi) acc[pi] = b;
    const float* wr = w + (size_t)co * a.K;
    for (int k = 0; k < a.K; ++k) {
      const float wv = __ldg(wr + k);
#pragma unroll
      for (int pi = 0; pi < PIX_PER_BLOCK; ++pi) acc[pi] = fmaf(wv, patch[pi][k], acc[pi]);
    }
#pragma unroll
    for (int pi = 0; pi < PIX_PER_BLOCK; ++pi) {
      const long long p = p0 + pi;
      if (p < P) {
        if (out_f32) out_f32[p * a.Cout + co] = acc[pi];
        if (out_bf16) out_bf16[p * a.Cout + co] = __float2bfloat16(pg_act_fwd(act_bf16, acc[pi]));
      }
    }
  }
}

// wgrad: dw[co, k] += sum_p dy[p, co] * patch[p, k].  Persistent blocks; each thread owns a strided set of
// (co, k) outputs and accumulates over the block's pixel chunks, then writes them to slice blockIdx.x of `part`
// ([blocks][Cout*K], summed in block order by pg_sum_partials).
constexpr int WG_PIX = 32;
constexpr int WG_MAX_OUT_PER_THREAD = 64;

__global__ void __launch_bounds__(256)
conv_small_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, const ConvArgs a,
                        float* __restrict__ part, const int o_base) {
  extern __shared__ float smw[];
  float* patch = smw;                          // [WG_PIX][K]
  float* dys = smw + WG_PIX * a.K;             // [WG_PIX][Cout]
  const int HW = a.H * a.W;
  const long long P = (long long)a.N * HW;
  const int n_out = a.Cout * a.K;
  float acc[WG_MAX_OUT_PER_THREAD];
#pragma unroll
  for (int i = 0; i < WG_MAX_OUT_PER_THREAD; ++i) acc[i] = 0.f;
  for (long long p0 = (long long)blockIdx.x * WG_PIX; p0 < P; p0 += (long long)gridDim.x * WG_PIX) {
    __syncthreads();
    for (int t = threadIdx.x; t < WG_PIX * a.K; t += blockDim.x) {
      const int pi = t / a.K, k = t % a.K;
      const long long p = p0 + pi;
      float v = 0.f;
      if (p < P) {
        const int n = (int)(p / HW), rem = (int)(p % HW);
        v = patch_value(x, a, n, rem / a.W, rem % a.W, k);
      }
      patch[pi * a.K + k] = v;
    }
    for (int t = threadIdx.x; t < WG_PIX * a.Cout; t += blockDim.x) {
      const int pi = t / a.Cout, co = t % a.Cout;
      const long long p = p0 + pi;
      dys[pi * a.Cout + co] = p < P ? dy[p * a.Cout + co] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < WG_MAX_OUT_PER_THREAD; ++i) {
      const int o = o_base + threadIdx.x + i * blockDim.x;
      if (o < n_out) {
        const int co = o / a.K, k = o % a.K;
        float s = 0.f;
#pragma unroll 8
        for (int pi = 0; pi < WG_PIX; ++pi) s = fmaf(dys[pi * a.Cout + co], patch[pi * a.K + k], s);
        acc[i] += s;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < WG_MAX_OUT_PER_THREAD; ++i) {
    const int o = o_base + threadIdx.x + i * blockDim.x;
    if (o < n_out) part[(size_t)blockIdx.x * n_out + o] = acc[i];
  }
}

// dgrad w.r.t. the input image: dx[n,ci,y,x] = act'(x) * sum_{co,i,j} dy[(y-i*dh+ph, x-j*dw+pw), co] * w[co,ci,i,j].
// The weight is staged once per block in shared memory as [tap][ci][co] (co contiguous: conflict-free, coalesced with
// the dy rows); one warp per input pixel, lanes over output channels.
__global__ void __launch_bounds__(256)
conv_small_dgrad_kernel(const float* __restrict__ w, const float* __restrict__ dy, const ConvArgs a,
                        const float* __restrict__ x, float* __restrict__ dx) {
  extern __shared__ float wt[];  // [kh*kw][Cin][Cout]
  const int taps = a.kh * a.kw;
  for (int t = threadIdx.x; t < taps * a.Cin * a.Cout; t += blockDim.x) {
    const int co = t % a.Cout, ci = (t / a.Cout) % a.Cin, tap = t / (a.Cout * a.Cin);
    wt[t] = w[((size_t)co * a.Cin + ci) * taps + tap];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int HW = a.H * a.W;
  const long long P = (long long)a.N * HW;
  const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; gw < P; gw += warps) {
    const int n = (int)(gw / HW), rem = (int)(gw % HW);
    const int y = rem / a.W, xx = rem % a.W;
    for (int c0 = 0; c0 < a.Cin; c0 += 4) {  // input channels in groups of 4 accumulators
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int i = 0; i < a.kh; ++i) {
        const int yo = y - i * a.dh + a.ph;
        if (yo < 0 || yo >= a.H) continue;
        for (int j = 0; j < a.kw; ++j) {
          const int xo = xx - j * a.dw + a.pw;
          if (xo < 0 || xo >= a.W) continue;
          const float* dyr = dy + ((size_t)n * HW + (size_t)yo * a.W + xo) * a.Cout;
          const float* wr = wt + ((size_t)(i * a.kw + j) * a.Cin + c0) * a.Cout;
          for (int co = lane; co < a.Cout; co += 32) {
            const float d = dyr[co];
#pragma unroll
            for (int ci = 0; ci < 4; ++ci)
              if (c0 + ci < a.Cin) acc[ci] = fmaf(d, wr[ci * a.Cout + co], acc[ci]);
          }
        }
      }
#pragma unroll
      for (int ci = 0; ci < 4; ++ci) {
        if (c0 + ci >= a.Cin) break;
        const float v = warp_sum(acc[ci]);
        if (lane == 0) {
          const size_t off = (((size_t)n * a.Cin + c0 + ci) * a.H + y) * a.W + xx;
          dx[off] = a.pre_act == PG_ACT_NONE ? v : v * pg_act_bwd(a.pre_act, x[off]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Tap gather / scatter: the convolutions whose contraction runs on the wgmma GEMM over a gathered tap matrix.
// Two geometries: the grid of GEMM rows (N, Hg, Wg) and the spatial tensor (N, Hs, Ws).  Row p_o = (n, yo, xo) of the
// gathered matrix reads the spatial pixel (yo * s + dy_t, xo * s + dx_t) for tap t:
//   gather:  X_cat[p_o, t*C + c] = act(x[(yo * s + dy_t, xo * s + dx_t), c])       (zero outside the spatial tensor)
//   scatter: out[q, c] = sum over (p_o, t) with that pixel = q, ascending t, of Y_cat[p_o, t*C + c]   (the adjoint)
// Stride 1 with rows = spatial = the image is the wide-channel CausalConv2d (Cin >= 8, the GatedPixelCNN 1xN / Nx1 and
// PixelSNAIL 2x2 convs: reference gated_pixel_cnn.py:63-99,115,121, pixel_snail.py:41-56, nn/convolution.py:41-43):
// conv(x)[p] = sum_t W_t . x[p + (dy_t, dx_t)] with zero fill outside the image (the reference's pad + crop, SURVEY
// Appendix A).  act(0) = 0 for every activation on that path (ReLU / ELU), so it commutes with the zero padding.
// Stride 2 is Conv2d (rows = output pixels, spatial = input) and ConvTranspose2d (rows = input pixels, spatial =
// output) of reference models/vae/vaes.py Encoder / Decoder.  kUnitStride builds s = 1 without the scatter's per-tap
// divisibility test and divisions.
// ------------------------------------------------------------------------------------------------
// The offsets travel in the kernel parameters: 225 taps (a 15 x 15 kernel) take 1800 bytes of the 4 KB.
constexpr int MAX_TAPS = 225;
struct StridedArgs {
  int N, Hg, Wg, Hs, Ws, C, T, s;
  int dy[MAX_TAPS], dx[MAX_TAPS];
};

template <bool kUnitStride>
__global__ void __launch_bounds__(256)
strided_gather_kernel(const bf16* __restrict__ x, int64_t ld_x, const StridedArgs a, int act, bf16* __restrict__ out) {
  const int s = kUnitStride ? 1 : a.s;
  const int c8n = a.C / 8;
  const int HWg = a.Hg * a.Wg;
  const long long total = (long long)a.N * HWg * a.T * c8n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % c8n);
    const int t = (int)((idx / c8n) % a.T);
    const long long p = idx / ((long long)c8n * a.T);
    const int n = (int)(p / HWg), rem = (int)(p % HWg);
    const int ys = (rem / a.Wg) * s + a.dy[t], xs = (rem % a.Wg) * s + a.dx[t];
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (ys >= 0 && ys < a.Hs && xs >= 0 && xs < a.Ws) {
      v = *reinterpret_cast<const uint4*>(x + ((size_t)n * a.Hs * a.Ws + (size_t)ys * a.Ws + xs) * ld_x + c8 * 8);
      if (act != PG_ACT_NONE) {
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(w[i]);
          w[i] = pack_bf16x2(pg_act_fwd(act, f.x), pg_act_fwd(act, f.y));
        }
        v = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    *reinterpret_cast<uint4*>(out + (size_t)p * a.T * a.C + (size_t)t * a.C + c8 * 8) = v;
  }
}

__device__ __forceinline__ void load8(const float* p, float* v) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void load8(const bf16* p, float* v) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

// v = sum_t Y_cat (ascending t) + bias;  v *= dact'(x_pre) when x_pre is given;  out_f32 = v, out_bf16 = act(v).
template <typename Tin, bool kUnitStride>
__global__ void __launch_bounds__(256)
strided_scatter_kernel(const Tin* __restrict__ ycat, const StridedArgs a, const float* __restrict__ bias, int n_bias,
                       int act, int dact, const bf16* __restrict__ x_pre, int64_t ld_pre, float* __restrict__ out_f32,
                       bf16* __restrict__ out_bf16, int64_t ld_out) {
  const int c8n = a.C / 8;
  const int HWs = a.Hs * a.Ws, HWg = a.Hg * a.Wg;
  const long long total = (long long)a.N * HWs * c8n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % c8n);
    const long long q = idx / c8n;
    const int n = (int)(q / HWs), rem = (int)(q % HWs);
    const int y = rem / a.Ws, xx = rem % a.Ws;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int t = 0; t < a.T; ++t) {
      const int ny = y - a.dy[t], nx = xx - a.dx[t];
      if (ny < 0 || nx < 0) continue;
      if (!kUnitStride && (ny % a.s || nx % a.s)) continue;
      const int yo = kUnitStride ? ny : ny / a.s, xo = kUnitStride ? nx : nx / a.s;
      if (yo >= a.Hg || xo >= a.Wg) continue;
      float v[8];
      load8(ycat + ((size_t)n * HWg + (size_t)yo * a.Wg + xo) * a.T * a.C + (size_t)t * a.C + c8 * 8, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i];
    }
    if (bias) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = c8 * 8 + i;
        if (c < n_bias) acc[i] += bias[c];
      }
    }
    if (x_pre) {
      float v[8];
      load8(x_pre + (size_t)q * ld_pre + c8 * 8, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] *= pg_act_bwd(dact, v[i]);
    }
    if (out_f32) {
      float* o = out_f32 + (size_t)q * ld_out + c8 * 8;
      *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    if (out_bf16) {
      if (act != PG_ACT_NONE) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = pg_act_fwd(act, acc[i]);
      }
      *reinterpret_cast<uint4*>(out_bf16 + (size_t)q * ld_out + c8 * 8) =
          make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                     pack_bf16x2(acc[6], acc[7]));
    }
  }
}

int fill_strided(StridedArgs& a, int N, int Hg, int Wg, int Hs, int Ws, int C, int T, int s, const int* dy,
                 const int* dx, const char* who) {
  PG_REQUIRE(T >= 1 && T <= MAX_TAPS, "%s: %d taps (max %d)", who, T, MAX_TAPS);
  PG_REQUIRE(C % 8 == 0, "%s: channel count %d must be a multiple of 8", who, C);
  PG_REQUIRE(s >= 1, "%s: stride %d must be positive", who, s);
  PG_REQUIRE(N >= 0 && Hg >= 1 && Wg >= 1 && Hs >= 1 && Ws >= 1, "%s: empty geometry (%d x %d rows, %d x %d spatial)", who,
             Hg, Wg, Hs, Ws);
  a.N = N; a.Hg = Hg; a.Wg = Wg; a.Hs = Hs; a.Ws = Ws; a.C = C; a.T = T; a.s = s;
  for (int t = 0; t < T; ++t) { a.dy[t] = dy[t]; a.dx[t] = dx[t]; }
  return 0;
}

unsigned grid_for(long long total) {
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)pg_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks < 1 ? 1 : blocks);
}

// The launchers behind pg_strided_* and pg_tap_*; `who` names the entry point in error messages.
int strided_gather(const void* x_pm, int64_t ld_x, int N, int Hg, int Wg, int Hs, int Ws, int C, int T, int stride,
                   const int* dy, const int* dx, int act, void* out, void* stream_, const char* who) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x_pm && out && dy && dx, "%s: null argument", who);
  PG_REQUIRE(ld_x % 8 == 0 && ld_x >= C, "%s: pitch %lld must be a multiple of 8 and at least C = %d", who,
             (long long)ld_x, C);
  PG_REQUIRE(pg_aligned16(x_pm) && pg_aligned16(out), "%s: x and out must be 16-byte aligned", who);
  StridedArgs a;
  if (fill_strided(a, N, Hg, Wg, Hs, Ws, C, T, stride, dy, dx, who)) return 1;
  const long long total = (long long)N * Hg * Wg * T * (C / 8);
  if (total == 0) return 0;
  auto kernel = stride == 1 ? strided_gather_kernel<true> : strided_gather_kernel<false>;
  kernel<<<grid_for(total), 256, 0, stream>>>((const bf16*)x_pm, ld_x, a, act, (bf16*)out);
  return pg_check_launch(who);
}

int strided_scatter(const void* ycat, int ycat_f32, int N, int Hg, int Wg, int Hs, int Ws, int C, int T, int stride,
                    const int* dy, const int* dx, const float* bias, int n_bias, int act, int dact, const void* x_pre,
                    int64_t ld_pre, float* out_f32, void* out_bf16, int64_t ld_out, void* stream_, const char* who) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(ycat && dy && dx && (out_f32 || out_bf16), "%s: null argument", who);
  PG_REQUIRE(ld_out % 8 == 0 && ld_out >= C && (!x_pre || (ld_pre % 8 == 0 && ld_pre >= C)),
             "%s: pitches must be multiples of 8 and at least C = %d", who, C);
  PG_REQUIRE(pg_aligned16(ycat) && pg_aligned16(x_pre) && pg_aligned16(out_f32) && pg_aligned16(out_bf16),
             "%s: ycat, x_pre, out_f32 and out_bf16 must be 16-byte aligned", who);
  PG_REQUIRE(!bias || (n_bias >= 0 && n_bias <= C), "%s: %d bias entries for %d channels", who, n_bias, C);
  StridedArgs a;
  if (fill_strided(a, N, Hg, Wg, Hs, Ws, C, T, stride, dy, dx, who)) return 1;
  const long long total = (long long)N * Hs * Ws * (C / 8);
  if (total == 0) return 0;
  const bf16* pre = (const bf16*)x_pre;
  if (ycat_f32) {
    auto kernel = stride == 1 ? strided_scatter_kernel<float, true> : strided_scatter_kernel<float, false>;
    kernel<<<grid_for(total), 256, 0, stream>>>((const float*)ycat, a, bias, n_bias, act, dact, pre, ld_pre, out_f32,
                                                (bf16*)out_bf16, ld_out);
  } else {
    auto kernel = stride == 1 ? strided_scatter_kernel<bf16, true> : strided_scatter_kernel<bf16, false>;
    kernel<<<grid_for(total), 256, 0, stream>>>((const bf16*)ycat, a, bias, n_bias, act, dact, pre, ld_pre, out_f32,
                                                (bf16*)out_bf16, ld_out);
  }
  return pg_check_launch(who);
}

}  // namespace

extern "C" int pg_conv_small_fwd_d(const float* x_nchw, const float* w_oihw, const float* bias, int N, int Cin, int H,
                                   int W, int Cout, int kh, int kw, int pad_h, int pad_w, int dil_h, int dil_w, int pre_act,
                                   float* out_f32, void* out_bf16, int act_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x_nchw && w_oihw && (out_f32 || out_bf16), "pg_conv_small_fwd: null argument");
  PG_REQUIRE(dil_h >= 1 && dil_w >= 1, "pg_conv_small_fwd: dilation (%d, %d) must be positive", dil_h, dil_w);
  ConvArgs a = {N, Cin, H, W, Cout, kh, kw, pad_h, pad_w, Cin * kh * kw, dil_h, dil_w, pre_act};
  PG_REQUIRE(a.K <= MAX_K, "pg_conv_small_fwd: Cin*kh*kw = %d exceeds %d", a.K, MAX_K);
  const long long P = (long long)N * H * W;
  const unsigned blocks = (unsigned)((P + PIX_PER_BLOCK - 1) / PIX_PER_BLOCK);
  conv_small_fwd_kernel<<<blocks, 256, 0, stream>>>(x_nchw, w_oihw, bias, a, out_f32, (bf16*)out_bf16, act_bf16);
  return pg_check_launch("pg_conv_small_fwd");
}

extern "C" int pg_conv_small_fwd(const float* x_nchw, const float* w_oihw, const float* bias, int N, int Cin, int H,
                                 int W, int Cout, int kh, int kw, int pad_h, int pad_w, int pre_act, float* out_f32,
                                 void* out_bf16, int act_bf16, void* stream_) {
  return pg_conv_small_fwd_d(x_nchw, w_oihw, bias, N, Cin, H, W, Cout, kh, kw, pad_h, pad_w, 1, 1, pre_act, out_f32,
                             out_bf16, act_bf16, stream_);
}

extern "C" int pg_conv_small_bwd_d(const float* x_nchw, const float* w_oihw, const float* dy_pm, int N, int Cin, int H,
                                   int W, int Cout, int kh, int kw, int pad_h, int pad_w, int dil_h, int dil_w, int pre_act,
                                   float* dw_oihw, float* dbias, float* dx_nchw, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(x_nchw && w_oihw && dy_pm, "pg_conv_small_bwd: null argument");
  PG_REQUIRE(dil_h >= 1 && dil_w >= 1, "pg_conv_small_bwd: dilation (%d, %d) must be positive", dil_h, dil_w);
  ConvArgs a = {N, Cin, H, W, Cout, kh, kw, pad_h, pad_w, Cin * kh * kw, dil_h, dil_w, pre_act};
  PG_REQUIRE(a.K <= MAX_K, "pg_conv_small_bwd: Cin*kh*kw = %d exceeds %d", a.K, MAX_K);
  const long long P = (long long)N * H * W;
  if (dw_oihw) {
    const size_t smem = (size_t)WG_PIX * (a.K + a.Cout) * sizeof(float);
    PG_REQUIRE(smem <= 200 * 1024, "pg_conv_small_bwd: shared memory %zu too large", smem);
    PG_CUDA(cudaFuncSetAttribute(conv_small_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    long long blocks = (P + WG_PIX - 1) / WG_PIX;
    const long long cap = (long long)pg_num_sms() * 2;
    if (blocks > cap) blocks = cap;
    float* part = nullptr;
    if (pg_scratch((size_t)blocks * a.Cout * a.K * sizeof(float), stream, &part)) return 1;
    // each launch covers WG_MAX_OUT_PER_THREAD * 256 = 16384 of the Cout*K outputs (one launch at every SURVEY.md §8 config)
    for (int o_base = 0; o_base < a.Cout * a.K; o_base += WG_MAX_OUT_PER_THREAD * 256) {
      conv_small_wgrad_kernel<<<(unsigned)blocks, 256, smem, stream>>>(x_nchw, dy_pm, a, part, o_base);
      if (pg_check_launch("pg_conv_small_bwd(wgrad)")) return 1;
    }
    const int n_out = a.Cout * a.K;
    if (pg_sum_partials(part, (int)blocks, n_out, 1, n_out, n_out, dw_oihw, stream)) return 1;
  }
  if (dbias) {
    if (pg_colsum_f32(dy_pm, Cout, (int)P, Cout, dbias, 1, stream_)) return 1;
  }
  if (dx_nchw) {
    const size_t smem_w = (size_t)a.K * Cout * sizeof(float);
    PG_REQUIRE(smem_w <= 200 * 1024, "pg_conv_small_bwd: weight tile %zu B too large for shared memory", smem_w);
    PG_CUDA(cudaFuncSetAttribute(conv_small_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    long long blocks = (P * 32 + 255) / 256;
    const long long cap = (long long)pg_num_sms() * 4;
    if (blocks > cap) blocks = cap;
    conv_small_dgrad_kernel<<<(unsigned)blocks, 256, smem_w, stream>>>(w_oihw, dy_pm, a, x_nchw, dx_nchw);
    if (pg_check_launch("pg_conv_small_bwd(dgrad)")) return 1;
  }
  return 0;
}

extern "C" int pg_conv_small_bwd(const float* x_nchw, const float* w_oihw, const float* dy_pm, int N, int Cin, int H,
                                 int W, int Cout, int kh, int kw, int pad_h, int pad_w, int pre_act, float* dw_oihw,
                                 float* dbias, float* dx_nchw, void* stream_) {
  return pg_conv_small_bwd_d(x_nchw, w_oihw, dy_pm, N, Cin, H, W, Cout, kh, kw, pad_h, pad_w, 1, 1, pre_act, dw_oihw,
                             dbias, dx_nchw, stream_);
}

extern "C" int pg_tap_gather(const void* x_pm, int64_t ld_x, int N, int H, int W, int C, int T, const int* dy,
                             const int* dx, int act, void* out, void* stream_) {
  return strided_gather(x_pm, ld_x, N, H, W, H, W, C, T, 1, dy, dx, act, out, stream_, "pg_tap_gather");
}

extern "C" int pg_tap_scatter(const void* dxcat, int N, int H, int W, int C, int T, const int* dy, const int* dx,
                              int act, const void* x_pre, int64_t ld_pre, float* dx_f32, void* dx_bf16, int64_t ld_dx,
                              void* stream_) {
  PG_REQUIRE(act == PG_ACT_NONE || x_pre, "pg_tap_scatter: activation backward needs the pre-activation input");
  return strided_scatter(dxcat, 0, N, H, W, H, W, C, T, 1, dy, dx, nullptr, 0, PG_ACT_NONE, act,
                         act == PG_ACT_NONE ? nullptr : x_pre, ld_pre, dx_f32, dx_bf16, ld_dx, stream_,
                         "pg_tap_scatter");
}

extern "C" int pg_strided_gather(const void* x_pm, int64_t ld_x, int N, int Hg, int Wg, int Hs, int Ws, int C, int T,
                                 int stride, const int* dy, const int* dx, void* out, void* stream_) {
  return strided_gather(x_pm, ld_x, N, Hg, Wg, Hs, Ws, C, T, stride, dy, dx, PG_ACT_NONE, out, stream_,
                        "pg_strided_gather");
}

extern "C" int pg_strided_scatter(const void* ycat, int ycat_f32, int N, int Hg, int Wg, int Hs, int Ws, int C, int T,
                                  int stride, const int* dy, const int* dx, const float* bias, int n_bias, int act,
                                  int dact, const void* x_pre, int64_t ld_pre, float* out_f32, void* out_bf16,
                                  int64_t ld_out, void* stream_) {
  return strided_scatter(ycat, ycat_f32, N, Hg, Wg, Hs, Ws, C, T, stride, dy, dx, bias, n_bias, act, dact, x_pre, ld_pre,
                         out_f32, out_bf16, ld_out, stream_, "pg_strided_scatter");
}
