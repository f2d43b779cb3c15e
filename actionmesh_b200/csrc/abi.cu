// C-ABI plumbing: last-error buffer, tensor-map encoder, device query.
#include <cstdarg>
#include <mutex>
#include "common.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
    set_last_error("cuTensorMapEncodeTiled unavailable (%s)", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return AMB_ERR_DRIVER;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_last_error("tensor map base %p not 16-byte aligned", base);
    return AMB_ERR_ARG;
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim, gstr, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u stride0 %llu)",
                   (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                   rank > 1 ? box[1] : 0, (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
    return AMB_ERR_DRIVER;
  }
  return AMB_OK;
}

// Per-(kernel, device) opt-in to > 48 KB of dynamic shared memory (the attribute is a per-device setting).
int ensure_smem_optin_impl(const void* kern, int bytes) {
  constexpr int MAXK = 64, MAXD = 16;
  static const void* keys[MAXK] = {};
  static bool done[MAXK][MAXD] = {};
  static std::mutex mu;
  int dev = 0;
  AMB_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  int slot = -1;
  for (int i = 0; i < MAXK; ++i) {
    if (keys[i] == kern) { slot = i; break; }
    if (keys[i] == nullptr) { keys[i] = kern; slot = i; break; }
  }
  if (slot >= 0 && dev < MAXD && done[slot][dev]) return AMB_OK;
  AMB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  if (slot >= 0 && dev < MAXD) done[slot][dev] = true;
  return AMB_OK;
}

// SM count of the CURRENT device (cached per device).
int num_sms() {
  static int n[16] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev < 16 && n[dev]) return n[dev];
  int v = 0;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 132;
  if (dev < 16) n[dev] = v;
  return v;
}

}  // namespace amb

extern "C" {

const char* amb_last_error(void) { return amb::g_err; }

int amb_abi_version(void) { return AMB_ABI_VERSION; }

int amb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  AMB_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  AMB_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return amb::AMB_OK;
}

}  // extern "C"
