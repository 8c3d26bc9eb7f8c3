// The KV cache layouts of generation, and the only code that knows them: every kernel that reads or writes the cache addresses
// a (sequence, kv head, position) row through KvCache, and every C entry point builds its view with dense_kv_cache() or
// paged_kv_cache().
//   dense: k and v are the two halves of one [2, B, kvh, max_len, d] bf16 buffer
//   paged: k and v are [num_blocks, kvh, block_size, d] each, and position pos of sequence b lives in physical block
//          block_tables[b * max_blocks + pos / block_size] (FusedBlockMultiTransformer, fused_transformer_layers.py:2192;
//          cache writes: csrc/gpu/append_attn/decoder_write_cache_with_rope_kernel.cu, encoder_write_cache_with_rope_kernel.cu)
#pragma once
#include "common.cuh"
#include "host_util.h"

namespace b200 {

struct KvCache {
  // Writable because the cache writers share the view; the attention entry points take const caches and only read through it.
  bf16* k;
  bf16* v;
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
};

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
inline int paged_kv_cache(KvCache* kv, const void* key_cache, const void* value_cache, const int32_t* block_tables,
                          int64_t num_kv_heads, int64_t head_dim, int64_t block_size, int64_t max_blocks_per_seq, const char* what) {
  if (!(key_cache && value_cache && block_tables)) return fail_arg("%s: null cache or block table", what);
  if (!(block_size == 32 || block_size == 64 || block_size == 128))
    return fail_arg("%s: block_size must be 32, 64 or 128 (got %lld)", what, (long long)block_size);
  if (!(max_blocks_per_seq > 0 && num_kv_heads > 0 && head_dim > 0 && head_dim % 8 == 0))
    return fail_arg("%s: bad cache shape max_blocks_per_seq=%lld kvh=%lld head_dim=%lld", what, (long long)max_blocks_per_seq,
                    (long long)num_kv_heads, (long long)head_dim);
  *kv = {};
  kv->k = static_cast<bf16*>(const_cast<void*>(key_cache));
  kv->v = static_cast<bf16*>(const_cast<void*>(value_cache));
  kv->block_tables = block_tables;
  kv->max_blocks = static_cast<int>(max_blocks_per_seq);
  kv->block_size = static_cast<int>(block_size);
  kv->kvh = static_cast<int>(num_kv_heads);
  kv->max_len = static_cast<int>(max_blocks_per_seq * block_size);
  kv->d = static_cast<int>(head_dim);
  return 0;
}

}  // namespace b200
