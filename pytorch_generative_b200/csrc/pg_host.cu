// pg_host.cu — host-side plumbing of the C ABI: error strings, device query, CUtensorMap encoding.
#include <stdarg.h>

#include <atomic>
#include <string.h>

#include "../../include/pg_b200.h"
#include "pg_common.cuh"

static thread_local char g_err[1024] = "";

void pg_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static std::atomic<unsigned long long> g_launches{0};

int pg_check_launch(const char* what) {
  ++g_launches;  // one call per kernel launch: the count bench.py reports as gpu_launches
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    pg_set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

static float* g_scratch[64] = {nullptr};
static size_t g_scratch_bytes[64] = {0};

// A buffer is never freed: launches captured into a CUDA graph keep its address, so a superseded buffer must stay valid
// for every later replay.  Growth is geometric, so the superseded buffers add up to less than the current one.
int pg_scratch(size_t bytes, cudaStream_t stream, float** out) {
  int dev = 0;
  PG_CUDA(cudaGetDevice(&dev));
  PG_REQUIRE(dev >= 0 && dev < 64, "pg_scratch: device %d", dev);
  if (g_scratch_bytes[dev] < bytes) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    PG_CUDA(cudaStreamIsCapturing(stream, &st));
    PG_REQUIRE(st == cudaStreamCaptureStatusNone,
               "pg_scratch: %zu bytes of reduction scratch needed while a CUDA graph is being captured (run the step "
               "once before capturing it)", bytes);
    size_t want = 2 * g_scratch_bytes[dev];
    if (want < bytes) want = bytes;
    if (want < ((size_t)1 << 24)) want = (size_t)1 << 24;
    float* fresh = nullptr;
    PG_CUDA(cudaMalloc(&fresh, want));
    g_scratch[dev] = fresh;  // the previous buffer (if any) stays allocated, see above
    g_scratch_bytes[dev] = want;
  }
  *out = g_scratch[dev];
  return 0;
}

__global__ void sum_partials_kernel(const float* __restrict__ part, int nparts, long long part_stride, int M, int N,
                                    int64_t ld_out, float* __restrict__ out) {
  const long long total = (long long)M * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += part[p * part_stride + i];
    out[(i / N) * ld_out + i % N] += s;
  }
}
// Many partials of few outputs (block partials of a column reduction): one warp per output element, lane l adds
// partials l, l + 32, ... and the warp combines its lanes with a fixed butterfly, so the order is still fixed.
__global__ void sum_partials_warp_kernel(const float* __restrict__ part, int nparts, long long part_stride, int M, int N,
                                         int64_t ld_out, float* __restrict__ out) {
  const long long total = (long long)M * N;
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < total; i += warps) {
    float s = 0.f;
    for (int p = lane; p < nparts; p += 32) s += part[p * part_stride + i];
    s = warp_sum(s);
    if (lane == 0) out[(i / N) * ld_out + i % N] += s;
  }
}

int pg_sum_partials(const float* part, int nparts, long long part_stride, int M, int N, int64_t ld_out, float* out,
                    cudaStream_t stream) {
  const long long total = (long long)M * N;
  const bool per_warp = nparts >= 64;  // decided by the shape alone: the same order on every run
  long long blocks = ((per_warp ? total * 32 : total) + 255) / 256;
  if (blocks > (long long)pg_num_sms() * 8) blocks = (long long)pg_num_sms() * 8;
  if (blocks < 1) blocks = 1;
  if (per_warp)
    sum_partials_warp_kernel<<<(unsigned)blocks, 256, 0, stream>>>(part, nparts, part_stride, M, N, ld_out, out);
  else
    sum_partials_kernel<<<(unsigned)blocks, 256, 0, stream>>>(part, nparts, part_stride, M, N, ld_out, out);
  return pg_check_launch("pg_sum_partials");
}

extern "C" int pg_abi_version(void) { return PG_ABI_VERSION; }
extern "C" const char* pg_last_error(void) { return g_err; }

// SMs the persistent kernels leave free (pg_reserve_sms): under data parallelism the NCCL all-reduce kernels of the
// gradient buckets run next to the backward GEMMs; a persistent grid that claims every SM makes them queue behind it (or
// pushes GEMM CTAs into a ragged second wave), so the grid is sized to what is left.
static std::atomic<int> g_reserved_sms{0};
extern "C" int pg_reserve_sms(int n) {
  const int old = g_reserved_sms.load();
  g_reserved_sms.store(n < 0 ? 0 : n);
  return old;
}

static int device_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}
int pg_num_sms() {
  const int n = device_sms() - g_reserved_sms.load();
  return n < 2 ? 2 : (n & ~1);  // an even count: the 2-CTA kernels launch whole pairs
}
extern "C" int pg_sm_count(void) { return pg_num_sms(); }
extern "C" unsigned long long pg_launch_count(void) { return g_launches.load(); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

// Generic tiled map.  elem_bytes in {2 (bf16), 4 (fp32)}; swizzle_bytes in {0, 32, 64, 128}.
int pg_make_tmap_nd(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode();
  PG_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  PG_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer %p not 16-byte aligned", base);
  PG_REQUIRE(elem_bytes == 2 || elem_bytes == 4, "TMA element size %d unsupported", elem_bytes);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    PG_REQUIRE(box[i] >= 1 && box[i] <= 256, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    PG_REQUIRE((strides_bytes[i] & 15) == 0, "TMA stride %d = %llu bytes not a multiple of 16", i,
               (unsigned long long)strides_bytes[i]);
  }
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  if (swizzle_bytes)
    PG_REQUIRE((int)box[0] * elem_bytes <= swizzle_bytes, "TMA inner box %u x %dB exceeds the %dB swizzle span", box[0],
               elem_bytes, swizzle_bytes);
  CUresult r = enc(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                   (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PG_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int pg_make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, int swizzle128) {
  return pg_make_tmap_nd(out, base, 2, rank, dims, strides_bytes, box, swizzle128 ? 128 : 0);
}

int pg_make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                    uint32_t box_rows, uint32_t box_cols, int swizzle_bytes) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  uint32_t box[2] = {box_cols, box_rows};
  return pg_make_tmap_nd(out, base, elem_bytes, 2, dims, strides, box, swizzle_bytes);
}

int pg_make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                         uint32_t box_rows, uint32_t box_cols) {
  return pg_make_tmap_2d(out, base, 2, rows, cols, ld, box_rows, box_cols, 128);
}
