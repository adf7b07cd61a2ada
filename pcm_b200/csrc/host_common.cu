#include "host_common.h"
#include <stdio.h>
#include <stdlib.h>
#include <cudaTypedefs.h>
#include "../../include/pcm_b200.h"

namespace pcm {

static thread_local char g_err[512] = "";

int set_error(const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return -1;
}
int set_cuda_error(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s", static_cast<int>(e),
           cudaGetErrorString(e), what);
  return -2;
}
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) v = getenv("PCM_NO_PDL") ? 0 : 1;
  return v == 1;
}
int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                             const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}

int encode_tmap(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* estr,
                int swizzle_bytes) {
  EncodeFn fn = get_encode();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                  const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] box "
             "[%u,%u,%u,%u] stride0 %llu",
             static_cast<int>(r), rank, (unsigned long long)dims[0],
             (unsigned long long)(rank > 1 ? dims[1] : 0), (unsigned long long)(rank > 2 ? dims[2] : 0),
             (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], rank > 1 ? box[1] : 0,
             rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, (unsigned long long)strides_bytes[0]);
    return set_error(buf);
  }
  return 0;
}

const char* last_error() { return g_err; }

}  // namespace pcm

extern "C" const char* pcm_last_error(void) { return pcm::last_error(); }
extern "C" int pcm_version(void) { return 1; }
extern "C" int pcm_num_sms(void) { return pcm::num_sms(); }
