// Host-side helpers shared by the C-ABI translation units: thread-local error string, CUtensorMap encoding
// through the driver entry point (no link-time dependency on libcuda), device attribute cache.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

// Error convention of the C-ABI (include/b200nlp.h): 0 ok, <0 argument error, >0 cudaError_t.
void set_last_error(const char* fmt, ...);
int fail_arg(const char* fmt, ...);   // records message, returns -1
int check_launch(const char* what);  // cudaGetLastError() -> return code

int sm_count();  // multiprocessors of the current device (cached per device)
int fa_fwd_impl();         // b200_set_fa_fwd_impl(): 2 = wgmma kernel, 1 = mma.sync kernel (cross-check)
int fa_bwd_impl();         // b200_set_fa_bwd_impl(): 2 = wgmma kernel, 1 = mma.sync kernel (cross-check)
// Attention launchers over a KV cache view (kv_cache.cuh: KvCache holds bf16, KvCacheC8 uint8 with per-head scales); the
// prefill one serves b200_append_attention
template <typename T>
struct KvCacheT;
using KvCache = KvCacheT<__nv_bfloat16>;
using KvCacheC8 = KvCacheT<uint8_t>;
template <typename T>
int launch_fa_prefill_paged(const KvCacheT<T>& kv, const void* qkv, void* out, const int32_t* cu_seqlens_q,
                            const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time,
                            int64_t B, int64_t max_q_len, int64_t num_heads, int64_t ldq, int64_t ldo, float softmax_scale,
                            cudaStream_t stream);   // fa_fwd.cu, instantiated for both element types
// decode_attn_tc.cu, dense or paged view: the checks (message names `what`), then the launch of checked arguments
template <typename T>
int check_decode_attention(const char* what, const KvCacheT<T>& kv, const void* qkv, const int32_t* seq_lens, const void* out,
                           const void* workspace, int64_t B, int64_t num_heads, int64_t ld, int64_t num_splits);
template <typename T>
int launch_decode_attention(const KvCacheT<T>& kv, const void* qkv, const int32_t* seq_lens, void* out, void* workspace, int64_t B,
                            int64_t num_heads, int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream);
bool pdl_enabled();   // b200_set_pdl(): launch GEMMs with programmatic dependent launch (decode-step kernel chains)

// Launch `kern` on `stream`; when PDL is enabled the launch carries the programmatic-stream-serialization attribute, so the
// grid may become resident while its predecessor is still running.  Such kernels MUST call pdl_wait() (common.cuh) before
// touching memory the predecessor writes.  Returns the cudaLaunchKernelEx status (recorded by check_launch()).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Encode a 2-D or 3-D bf16 (2-byte element) tiled tensor map with 128-byte swizzle.
//   dims[i]    extent of dimension i in elements (dimension 0 is contiguous)
//   strides[i] byte stride of dimension i+1 (i < rank-1); must be multiples of 16
//   box[i]     box extent in elements; box[0]*2 must be <= 128 for SWIZZLE_128B
// Returns 0 on success, <0 on failure (message recorded).
int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box);
// Same for fp32 elements (box[0] * 4 must be <= 128); used for TMA reduce-add into fp32 accumulation buffers.
int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                    const uint32_t* box);
// Same for 1-byte elements (int8 weights of the weight-only GEMM; box[0] must be <= 128).
int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                   const uint32_t* box);
// out[m, n] = bf16(ws[m, n] + bias[n]) for the split-K GEMMs (N % 8 == 0, ws [M, N] contiguous); re-zeroes ws
// (gemm_wgmma.cu).
int splitk_finish(float* ws, const float* bias, void* out, int64_t M, int64_t N, int64_t ldc, cudaStream_t stream);
// Attention operand [B, S, heads, D] bf16 with token stride ld (elements), box {64 d, 1 head, rows, 1}: one 128-byte swizzled
// block of `rows` rows.  Rows past S read as zeros, so a box never reaches into the next batch row.
inline int make_bf16_map(CUtensorMap* tm, const void* base, int64_t B, int64_t S, int64_t heads, int64_t D, int64_t ld,
                         uint32_t rows) {
  const uint64_t dims[4] = {static_cast<uint64_t>(D), static_cast<uint64_t>(heads), static_cast<uint64_t>(S), static_cast<uint64_t>(B)};
  const uint64_t strides[3] = {static_cast<uint64_t>(D) * 2, static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(S * ld) * 2};
  const uint32_t box[4] = {64, 1, rows, 1};
  return encode_tmap_bf16(tm, base, 4, dims, strides, box);
}

}  // namespace b200

#define B200_CHECK_ARG(cond, ...)                  \
  do {                                             \
    if (!(cond)) return b200::fail_arg(__VA_ARGS__); \
  } while (0)
