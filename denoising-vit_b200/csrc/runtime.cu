// Host runtime pieces shared by every entry point: error strings, debug implementation switch, SM count and TMA
// descriptor encoding (cuTensorMapEncodeTiled resolved through the runtime so that the library does not link
// against libcuda and can be dlopen'ed on a machine without a driver).
#include "common.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace dvt {

namespace {
thread_local char g_err[1024] = "";
int g_debug_impl_set = -1;  // dvt_set_debug_impl; -1: DVT_GEMM_IMPL decides
}

int debug_impl() {
  if (g_debug_impl_set >= 0) return g_debug_impl_set;
  static const int from_env = [] {
    const char* v = getenv("DVT_GEMM_IMPL");
    return (v && v[0] == 's') ? GEMM_SIMT_DEBUG : GEMM_TC;
  }();
  return from_env;
}

void set_debug_impl(int impl) { g_debug_impl_set = impl; }

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_err; }

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_last_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return DVT_ERR_CUDA;
}

static long long g_launches = 0;
void count_launch(long long n) { g_launches += n; }
long long launch_count() { return g_launches; }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode(CUtensorMap* out, const void* base, TmapDtype dt, int rank, const cuuint64_t* dims,
                  const cuuint64_t* strides, const cuuint32_t* box, int swizzle_bytes = 128) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled is not available (no CUDA driver?)");
    return DVT_ERR_CUDA;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUtensorMapDataType cdt = dt == TMAP_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(out, cdt, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u pitch %llu)",
                   (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1],
                   (unsigned long long)strides[0]);
    return DVT_ERR_CUDA;
  }
  return DVT_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* base, TmapDtype dt, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_bytes, uint32_t box_rows, uint32_t box_cols) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  return encode(out, base, dt, 2, dims, strides, box);
}

int make_tmap_3d(CUtensorMap* out, const void* base, TmapDtype dt, uint64_t d0, uint64_t d1, uint64_t d2,
                 uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2,
                 int swizzle_bytes) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, box2};
  return encode(out, base, dt, 3, dims, strides, box, swizzle_bytes);
}

}  // namespace dvt
