// Error text, launch counter and version for the C-ABI (include/dpvo_b200.h), and the tensor-map encoder (tc.cuh).
#include "common.cuh"
#include "tc.cuh"
#include <stdarg.h>

namespace dpvo {
static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int encode_tmap(CUtensorMap* m, const char* op, int rank, const void* ptr, const cuuint64_t* dims, const cuuint64_t* strides,
                const cuuint32_t* box) {
  // the encoder is a driver symbol, the same for every device of the process: looked up once, by a thread-safe static
  // initialiser, so that later calls cost one guarded load and no lock
  using EncodeTiledFn = decltype(&cuTensorMapEncodeTiled);
  static const EncodeTiledFn encode = []() -> EncodeTiledFn {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return (EncodeTiledFn)f;
  }();
  if (!encode) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the driver", op);
    return DPVO_ERR_CUDA;
  }
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("%s: cuTensorMapEncodeTiled failed (%d)", op, (int)r); return DPVO_ERR_CUDA; }
  return DPVO_OK;
}
}  // namespace dpvo

extern "C" const char* dpvo_version(void) { return "dpvo_b200 0.1 (sm_90a)"; }
extern "C" const char* dpvo_last_error(void) { return dpvo::g_err; }
extern "C" int64_t dpvo_launch_count(void) { return (int64_t)dpvo::g_launches.load(); }
