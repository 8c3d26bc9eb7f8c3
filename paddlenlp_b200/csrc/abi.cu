// C-ABI plumbing: error string, version, device checks, tensor-map encoding.
#include <string.h>

#include <mutex>

#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {

static thread_local char tls_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_err, sizeof(tls_err), fmt, ap);
  va_end(ap);
}
int fail_arg(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_err, sizeof(tls_err), fmt, ap);
  va_end(ap);
  return -1;
}
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: %s", what, cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  return 0;
}

static int g_pdl = 0;
bool pdl_enabled() { return g_pdl != 0; }
// attention kernels (fa_fwd.cu, fa_bwd.cu): b200_set_fa_fwd_impl / b200_set_fa_bwd_impl, 2 = wgmma, 1 = mma.sync
static int g_fa_fwd_impl = 2;
int fa_fwd_impl() { return g_fa_fwd_impl; }
static int g_fa_bwd_impl = 2;
int fa_bwd_impl() { return g_fa_bwd_impl; }

int sm_count() {
  static int cached[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides, const uint32_t* box);

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box) {
  return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides, box);
}
int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                    const uint32_t* box) {
  return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides, box);
}
int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                   const uint32_t* box) {
  return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides, box);
}

static int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides, const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail_arg("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i < rank - 1) gstr[i] = strides[i];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail_arg("tensor map base %p not 16-byte aligned", base);
  for (int i = 0; i < rank - 1; ++i)
    if (gstr[i] % 16 != 0) return fail_arg("tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)gstr[i]);
  CUresult r = fn(out, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail_arg("cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu] box=[%u,%u]", (int)r, rank,
                    (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                    rank > 1 ? box[1] : 0);
  return 0;
}

}  // namespace b200

extern "C" {

const char* b200_last_error(void) { return b200::tls_err; }

int b200_abi_version(void) { return B200NLP_ABI_VERSION; }

int b200_set_pdl(int enable) {
  int old = b200::g_pdl;
  b200::g_pdl = enable ? 1 : 0;
  return old;
}

int b200_set_fa_fwd_impl(int impl) {
  int old = b200::g_fa_fwd_impl;
  b200::g_fa_fwd_impl = impl == 1 ? 1 : 2;
  return old;
}

int b200_set_fa_bwd_impl(int impl) {
  int old = b200::g_fa_bwd_impl;
  b200::g_fa_bwd_impl = impl == 1 ? 1 : 2;
  return old;
}

int b200_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    b200::set_last_error("cudaGetDevice: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) return b200::fail_arg("device %d is sm_%d%d; this library is built for sm_90a only", dev, major, minor);
  return 0;
}

}  // extern "C"
