// pg_made.cu — MADE (reference models/autoregressive/made.py): the connectivity mask applied to a weight and cast to the
// bf16 GEMM operand in one pass, and the per-dimension step of incremental sampling.
#include "pg_common.cuh"

// One block per output row (grid-stride over the padded rows): the row's connectivity is read once, the threads walk the
// columns.  A masked entry is written back only when multiplying it by zero changes its bits, so once a mask set has been
// applied, applying it again writes nothing to the fp32 weight.
__global__ void made_mask_cast_kernel(float* __restrict__ w, int rows, int cols, const int* __restrict__ conn_in,
                                      const int* __restrict__ conn_out, int strict, bf16* __restrict__ wq, int rows_p,
                                      int64_t ld_q, float* __restrict__ mask) {
  for (int r = blockIdx.x; r < rows_p; r += gridDim.x) {
    bf16* qrow = wq + (int64_t)r * ld_q;
    if (r >= rows) {
      for (int64_t c = threadIdx.x; c < ld_q; c += blockDim.x) qrow[c] = __float2bfloat16(0.f);
      continue;
    }
    const int co = conn_out[r];
    float* wrow = w + (int64_t)r * cols;
    float* mrow = mask ? mask + (int64_t)r * cols : nullptr;
    for (int64_t c = threadIdx.x; c < ld_q; c += blockDim.x) {
      float v = 0.f;
      if (c < cols) {
        const int ci = conn_in[c];
        const float m = (strict ? ci < co : ci <= co) ? 1.f : 0.f;
        const float x = wrow[c];
        v = x * m;  // the reference's `weight *= mask` (a negative weight becomes -0)
        if (__float_as_uint(v) != __float_as_uint(x)) wrow[c] = v;
        if (mrow) mrow[c] = m;
      }
      qrow[c] = __float2bfloat16(v);
    }
  }
}

extern "C" int pg_made_mask_cast(float* w, int rows, int cols, const int* conn_in, const int* conn_out, int strict,
                                 void* w_bf16, int rows_p, int64_t ld_bf16, float* mask, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(w && conn_in && conn_out && w_bf16 && rows > 0 && cols > 0, "pg_made_mask_cast: null/empty argument");
  PG_REQUIRE(rows_p >= rows && ld_bf16 >= cols, "pg_made_mask_cast: the bf16 operand [%d, %lld] is smaller than the weight "
             "[%d, %d]", rows_p, (long long)ld_bf16, rows, cols);
  const int blocks = rows_p < pg_num_sms() * 16 ? rows_p : pg_num_sms() * 16;
  made_mask_cast_kernel<<<blocks, 256, 0, stream>>>(w, rows, cols, conn_in, conn_out, strict, (bf16*)w_bf16, rows_p,
                                                    ld_bf16, mask);
  return pg_check_launch("pg_made_mask_cast");
}

// One block per image; thread k owns hidden units k, k + blockDim, ... of h1, so the rank-1 update and the read of relu(h1)
// that follows it need no synchronisation between threads.  Every sum runs in a fixed order.
constexpr int kStepThreads = 256;

__global__ void __launch_bounds__(kStepThreads) made_sample_step_kernel(
    const int64_t* __restrict__ pos, const int* __restrict__ order, int D, const float* __restrict__ canvas,
    float* __restrict__ x_in, const float* __restrict__ w1t, float* __restrict__ h1, int H, int update,
    bf16* __restrict__ a1, int64_t ld_a1, const bf16* __restrict__ hl, int64_t ld_hl, const float* __restrict__ w_out,
    int K, const float* __restrict__ b_out, float* __restrict__ logits) {
  const int b = blockIdx.x;
  const int t = (int)*pos;
  float* hb = h1 + (int64_t)b * H;
  const float* cb = canvas + (int64_t)b * D;
  float* xb = x_in + (int64_t)b * D;
  if (update == 2) {  // every dimension, in index order
    for (int k = threadIdx.x; k < H; k += blockDim.x) {
      float acc = hb[k];
      for (int i = 0; i < D; ++i) {
        const float delta = cb[i] - xb[i];
        if (delta != 0.f) acc += delta * w1t[(int64_t)i * H + k];
      }
      hb[k] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x) xb[i] = cb[i];
  } else if (update == 1 && t > 0) {  // the dimension drawn at the previous step
    const int i = order[t - 1];
    const float delta = cb[i] - xb[i];
    if (delta != 0.f) {
      const float* col = w1t + (int64_t)i * H;
      for (int k = threadIdx.x; k < H; k += blockDim.x) hb[k] += delta * col[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) xb[i] = cb[i];
  }
  if (a1) {
    for (int k = threadIdx.x; k < H; k += blockDim.x) a1[(int64_t)b * ld_a1 + k] = __float2bfloat16(fmaxf(hb[k], 0.f));
  }
  if (logits) {
    const int d = order[t];
    const float* row = w_out + (int64_t)d * K;
    float acc = 0.f;
    if (hl) {
      const bf16* hrow = hl + (int64_t)b * ld_hl;
      for (int k = threadIdx.x; k < K; k += blockDim.x) acc += __bfloat162float(hrow[k]) * row[k];
    } else {
      for (int k = threadIdx.x; k < K; k += blockDim.x) acc += fmaxf(hb[k], 0.f) * row[k];
    }
    __shared__ float part[kStepThreads / 32];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w = 0; w < kStepThreads / 32; ++w) s += part[w];
      logits[b] = s + b_out[d];
    }
  }
}

extern "C" int pg_made_sample_step(const int64_t* pos, const int* order, int D, int n, const float* canvas, float* x_in,
                                   const float* w1t, float* h1, int H, int update, void* a1_bf16, int64_t ld_a1,
                                   const void* hl_bf16, int64_t ld_hl, const float* w_out, int K, const float* b_out,
                                   float* logits, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  PG_REQUIRE(pos && order && D > 0 && n > 0, "pg_made_sample_step: null/empty argument");
  PG_REQUIRE(update >= 0 && update <= 2, "pg_made_sample_step: update must be 0, 1 or 2 (got %d)", update);
  PG_REQUIRE(update == 0 || (canvas && x_in && w1t && h1 && H > 0), "pg_made_sample_step: the update needs canvas, x_in, "
             "w1t and h1");
  PG_REQUIRE(!a1_bf16 || (h1 && H > 0 && ld_a1 >= H), "pg_made_sample_step: a1 needs h1 and ld_a1 >= H");
  PG_REQUIRE(!logits || (w_out && b_out && K > 0), "pg_made_sample_step: logits need w_out, b_out and K");
  PG_REQUIRE(!logits || hl_bf16 || (h1 && K == H), "pg_made_sample_step: logits from relu(h1) need K == H");
  PG_REQUIRE(!hl_bf16 || ld_hl >= K, "pg_made_sample_step: ld_hl < K");
  made_sample_step_kernel<<<n, kStepThreads, 0, stream>>>(pos, order, D, canvas, x_in, w1t, h1, H, update, (bf16*)a1_bf16,
                                                          ld_a1, (const bf16*)hl_bf16, ld_hl, w_out, K, b_out, logits);
  return pg_check_launch("pg_made_sample_step");
}
