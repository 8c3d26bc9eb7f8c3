// The KV cache layouts of generation, and the only code that knows them: every kernel that reads or writes the cache addresses
// a (sequence, kv head, position) row through KvCache, and every C entry point builds its view with dense_kv_cache() or
// paged_kv_cache() (paged_kv_cache_c8() for the uint8 form).
//   dense: k and v are the two halves of one [2, B, kvh, max_len, d] bf16 buffer
//   paged: k and v are [num_blocks, kvh, block_size, d] each, and position pos of sequence b lives in physical block
//          block_tables[b * max_blocks + pos / block_size] (FusedBlockMultiTransformer, fused_transformer_layers.py:2192;
//          cache writes: csrc/gpu/append_attn/decoder_write_cache_with_rope_kernel.cu, encoder_write_cache_with_rope_kernel.cu)
// The paged cache holds bf16 (KvCache) or uint8 (KvCacheC8, cachekv_int8_type="static"): the same shape with 1-byte elements,
// so an element offset is the same number in either, and every writer stores through store8() below.
#pragma once
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// ---- int8 cache numerics (static per-kv-head scales: s quantises, o = 1 / s dequantises; both bf16 [kvh]) ----
// u = clamp(rne(bf16(s * x)), -127, 127) + 128, stored as uint8; x is the post-RoPE bf16 value the bf16 cache would hold.
// s * x is exact in fp32 (two 8-bit significands), so one bf16 rounding and one integer rounding (ties to even) follow, as in
// the reference's decoder-side write (decoder_write_cache_with_rope_impl.cuh:666-682, quant_round_type 0).  The offset is
// +128 for every row: the reference's encoder-side write stores +127 (encoder_write_cache_with_rope_impl.cuh:839) while its
// dequantise subtracts 128, which reads prompt rows back one step low; that is not reproduced here.
__device__ __forceinline__ uint32_t quant_c8(float x, float s) {
  const float r = fminf(fmaxf(rintf(bf16_round(s * x)), -127.f), 127.f);
  return static_cast<uint32_t>(static_cast<int>(r) + 128);
}
// Eight bf16 values (one 16-byte chunk) -> eight cache bytes.
__device__ __forceinline__ uint2 quant_c8x8(const uint4& x, float s) {
  const uint32_t* xi = reinterpret_cast<const uint32_t*>(&x);
  uint32_t w[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float2 a = unpack_bf16x2(xi[2 * h]), b = unpack_bf16x2(xi[2 * h + 1]);
    w[h] = quant_c8(a.x, s) | (quant_c8(a.y, s) << 8) | (quant_c8(b.x, s) << 16) | (quant_c8(b.y, s) << 24);
  }
  return make_uint2(w[0], w[1]);
}
// Byte i of a cache word -> the exact fp32 u - 128: the byte goes into the low mantissa byte of 2^23 (8388608 + u), and
// 8388608 + 128 is subtracted exactly.  The dequantised value is (u - 128) * o; the kernels apply o once per CTA (K: on the
// query scale, V: on the output), never per element.
template <int I>
__device__ __forceinline__ float dequant_c8(uint32_t w) {
  return __fsub_rn(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540 + I)), 8388736.f);
}

template <typename T>
struct KvCacheT {
  // Writable because the cache writers share the view; the attention entry points take const caches and only read through it.
  T* k;
  T* v;
  // uint8 cache only (null for bf16): quantise scales s (writers) and dequantise scales o (readers), bf16 [kvh] each
  const bf16* k_scale;
  const bf16* v_scale;
  const bf16* k_out_scale;
  const bf16* v_out_scale;
  const int* block_tables;   // null for the dense layout
  int max_blocks, block_size;
  int kvh, max_len, d;       // max_len: positions per sequence (max_blocks * block_size when paged)

  // Element offset of row (b, head, pos) in k, and the same in v.  D > 0 is head_dim known at compile time.
  template <bool PAGED, int D = 0>
  __device__ __forceinline__ size_t offset(int b, int head, int pos) const {
    const size_t row_d = D > 0 ? D : d;
    if constexpr (PAGED) {
      const int page = __ldg(block_tables + static_cast<size_t>(b) * max_blocks + pos / block_size);
      return ((static_cast<size_t>(page) * kvh + head) * block_size + pos % block_size) * row_d;
    } else {
      return dense_row(b, head, pos, kvh, max_len) * row_d;
    }
  }
  // Dense layout: row index of (b, head, pos), for a kernel that takes the view's geometry as scalars.
  __device__ __forceinline__ static size_t dense_row(int b, int head, int pos, int kvh, int max_len) {
    return (static_cast<size_t>(b) * kvh + head) * max_len + pos;
  }
  // For kernels that serve both layouts with one instantiation.
  __device__ __forceinline__ size_t offset(int b, int head, int pos) const {
    return block_tables != nullptr ? offset<true>(b, head, pos) : offset<false>(b, head, pos);
  }
  // Store the 16-byte chunk x of eight bf16 values at element `off` of k (which == 0) or v of kv head `head`: as they are in a
  // bf16 cache, quantised with that head's scale in a uint8 cache.
  __device__ __forceinline__ void store8(int which, int head, size_t off, const uint4& x) const {
    T* dst = (which != 0 ? v : k) + off;
    if constexpr (sizeof(T) == 1) {
      *reinterpret_cast<uint2*>(dst) = quant_c8x8(x, __bfloat162float((which != 0 ? v_scale : k_scale)[head]));
    } else {
      *reinterpret_cast<uint4*>(dst) = x;
    }
  }
};
using KvCache = KvCacheT<bf16>;
using KvCacheC8 = KvCacheT<uint8_t>;

// View of a dense cache [2, B, kvh, max_len, head_dim].  Returns 0, or the C-ABI argument error with a message naming `what`.
inline int dense_kv_cache(KvCache* kv, const void* cache, int64_t B, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                          const char* what) {
  if (cache == nullptr) return fail_arg("%s: null cache", what);
  if (!(B > 0 && num_kv_heads > 0 && max_len > 0 && head_dim > 0 && head_dim % 8 == 0))
    return fail_arg("%s: bad cache shape B=%lld kvh=%lld max_len=%lld head_dim=%lld", what, (long long)B, (long long)num_kv_heads,
                    (long long)max_len, (long long)head_dim);
  *kv = {};
  kv->k = static_cast<bf16*>(const_cast<void*>(cache));
  kv->v = kv->k + static_cast<size_t>(B) * num_kv_heads * max_len * head_dim;
  kv->kvh = static_cast<int>(num_kv_heads);
  kv->max_len = static_cast<int>(max_len);
  kv->d = static_cast<int>(head_dim);
  return 0;
}

// View of paged caches [num_blocks, kvh, block_size, head_dim] with block_tables [B, max_blocks_per_seq].  block_size 32, 64 or
// 128: the decode-attention producer moves whole 32-row chunks within a page and 64-row chunks over up to two pages.
template <typename T>
inline int paged_kv_cache(KvCacheT<T>* kv, const void* key_cache, const void* value_cache, const int32_t* block_tables,
                          int64_t num_kv_heads, int64_t head_dim, int64_t block_size, int64_t max_blocks_per_seq, const char* what) {
  if (!(key_cache && value_cache && block_tables)) return fail_arg("%s: null cache or block table", what);
  if (!(block_size == 32 || block_size == 64 || block_size == 128))
    return fail_arg("%s: block_size must be 32, 64 or 128 (got %lld)", what, (long long)block_size);
  if (!(max_blocks_per_seq > 0 && num_kv_heads > 0 && head_dim > 0 && head_dim % 8 == 0))
    return fail_arg("%s: bad cache shape max_blocks_per_seq=%lld kvh=%lld head_dim=%lld", what, (long long)max_blocks_per_seq,
                    (long long)num_kv_heads, (long long)head_dim);
  *kv = {};
  kv->k = static_cast<T*>(const_cast<void*>(key_cache));
  kv->v = static_cast<T*>(const_cast<void*>(value_cache));
  kv->block_tables = block_tables;
  kv->max_blocks = static_cast<int>(max_blocks_per_seq);
  kv->block_size = static_cast<int>(block_size);
  kv->kvh = static_cast<int>(num_kv_heads);
  kv->max_len = static_cast<int>(max_blocks_per_seq * block_size);
  kv->d = static_cast<int>(head_dim);
  return 0;
}

// The uint8 form: the paged view plus the four per-head scale arrays (bf16 [kvh]).  A writer passes only k_scale / v_scale,
// a reader only the out scales; `need_quant` / `need_dequant` say which must be non-null.
inline int paged_kv_cache_c8(KvCacheC8* kv, const void* key_cache, const void* value_cache, const int32_t* block_tables,
                             const void* k_scale, const void* v_scale, const void* k_out_scale, const void* v_out_scale,
                             bool need_quant, bool need_dequant, int64_t num_kv_heads, int64_t head_dim, int64_t block_size,
                             int64_t max_blocks_per_seq, const char* what) {
  if (need_quant && !(k_scale && v_scale)) return fail_arg("%s: null cache_k_scale / cache_v_scale", what);
  if (need_dequant && !(k_out_scale && v_out_scale)) return fail_arg("%s: null cache_k_out_scale / cache_v_out_scale", what);
  if (int rc = paged_kv_cache(kv, key_cache, value_cache, block_tables, num_kv_heads, head_dim, block_size, max_blocks_per_seq, what))
    return rc;
  if (head_dim % 16 != 0) return fail_arg("%s: head_dim must be a multiple of 16 (got %lld)", what, (long long)head_dim);
  kv->k_scale = static_cast<const bf16*>(k_scale);
  kv->v_scale = static_cast<const bf16*>(v_scale);
  kv->k_out_scale = static_cast<const bf16*>(k_out_scale);
  kv->v_out_scale = static_cast<const bf16*>(v_out_scale);
  return 0;
}

}  // namespace b200
