// Library-level pieces of the C ABI: error reporting, device check, TMA descriptor encoding.
#include "host_util.h"
#include "pdl.cuh"

#include <atomic>
#include <mutex>
#include <stdarg.h>
#include <string.h>

namespace mivos {

std::atomic<int64_t> g_launches{0};

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

int encode_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                   uint64_t pitch_elems, uint32_t box_cols, uint32_t box_rows, int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point not available (driver too old?)");
    return MIVOS_ERR_CUDA;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * static_cast<uint64_t>(elem_bytes)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rows=%llu cols=%llu pitch=%llu box=%ux%u base=%p)",
                   static_cast<int>(r), (unsigned long long)rows, (unsigned long long)cols,
                   (unsigned long long)pitch_elems, box_cols, box_rows, (const void*)base);
    return MIVOS_ERR_CUDA;
  }
  return MIVOS_OK;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;  // H100 SXM (no device visible: host-side planning only)
  }
  return n;
}

int* device_error_flag() {
  // one flag per device; allocated on first use (cudaMalloc is outside any timed region: the
  // Python side calls mivos_check_device() at import, which touches this)
  static int* flags[64] = {nullptr};
  static std::mutex mu;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  if (!flags[dev]) {
    int* p = nullptr;
    if (cudaMalloc(&p, sizeof(int)) != cudaSuccess) return nullptr;
    cudaMemset(p, 0, sizeof(int));
    flags[dev] = p;
  }
  return flags[dev];
}

}  // namespace mivos

using namespace mivos;

extern "C" MIVOS_API int mivos_abi_version(void) { return MIVOS_ABI_VERSION; }

extern "C" MIVOS_API const char* mivos_last_error(void) { return g_err; }

extern "C" MIVOS_API int mivos_check_device(void) {
  int dev = 0;
  MIVOS_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  MIVOS_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) {
    set_last_error("mivos_b200 needs an sm_90 (H100) device; device %d is sm_%d%d — there is no fallback path",
                   dev, prop.major, prop.minor);
    return MIVOS_ERR_DEVICE;
  }
  if (!device_error_flag()) {
    set_last_error("could not allocate the device error flag");
    return MIVOS_ERR_CUDA;
  }
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_poll_kernel_error(mivos_stream_t stream_, int* code_out) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int* flag = device_error_flag();
  MIVOS_REQUIRE(flag != nullptr, "no device error flag");
  int code = 0;
  MIVOS_CUDA_OK(cudaMemcpyAsync(&code, flag, sizeof(int), cudaMemcpyDeviceToHost, stream));
  MIVOS_CUDA_OK(cudaStreamSynchronize(stream));
  if (code != 0) {
    MIVOS_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), stream));
  }
  if (code_out) *code_out = code;
  if (code != 0) {
    set_last_error("kernel error flag = %d", code);
    return MIVOS_ERR_KERNEL;
  }
  return MIVOS_OK;
}

namespace mivos {
bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("MIVOS_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}
}  // namespace mivos

extern "C" MIVOS_API int64_t mivos_launch_count(void) { return g_launches.load(); }

// A replayed CUDA graph launches the kernels that were captured through this library without
// passing through its entry points again; the host runtime reports them here so that
// mivos_launch_count() stays the number of kernels actually executed.
extern "C" MIVOS_API int64_t mivos_add_launch_count(int64_t n) {
  return g_launches.fetch_add(n, std::memory_order_relaxed) + n;
}
