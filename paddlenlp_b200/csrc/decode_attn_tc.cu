// Decode attention over the dense and the paged KV cache on Hopper: one query token per sequence, GQA, head_dim 128.
//
//   out[b, h, :] = softmax(q[b, h, :] K[b, kv(h), 0:len_b, :]^T / sqrt(d)) V[b, kv(h), 0:len_b, :]
//
// Replaces the attention half of masked_multihead_attention / the decode branch of append_attention
// (paddlenlp/experimental/transformers/fused_transformer_layers.py:884-893;
//  csrc/gpu/append_attn/append_attention_c16_impl.cuh:377-744, split-KV :826-1000).
//
// The op is a pure stream of the cache through the SM (2*len*d*2 bytes per (b, kv head), ~4 flop/byte, far below the
// tensor-core ridge point), so the design goal is bytes in flight:
//   * one producer warp moves 32-row K and V chunks (8 KB each, contiguous in both cache layouts: a page holds 32, 64 or 128
//     rows) with the bulk-copy engine (cp.async.bulk) into a 4-stage shared-memory ring, completion on mbarriers; with two
//     CTAs per SM (GQA groups up to 4) that is 128 KB of cache in flight per SM, independent of the math;
//   * four consumer warps: a half-warp per cache row (16 lanes x 8 dims), the GQA group's G heads share every K/V row,
//     online softmax in fp32 (exp2), the 8 half-warp partials merged through shared memory at the end;
//   * split-KV partials ([B*nh, nsplit, 132] fp32: unnormalised o, running max, sum) are merged by
//     decode_attention_merge_kernel (generation.cu).
// b200_decode_attention (generation.cu, plain global loads) computes the same function and is the cross-check.
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
// generation.cu
int launch_decode_attention_merge(const float* partial, void* out, int rows, int nsplit, cudaStream_t stream);

namespace dab {

constexpr int D = 128;
constexpr int ROWS = 32;                       // cache rows per chunk
constexpr int NST = 4;                         // ring stages
constexpr int CHUNK_BYTES = ROWS * D * 2;      // 8 KB of K (and as much of V) per stage
constexpr int SMEM_BYTES = NST * 2 * CHUNK_BYTES;
constexpr int NUM_THREADS = 160;               // 4 consumer warps + 1 producer warp

struct Params {
  const bf16* qkv;
  const bf16* kc;
  const bf16* vc;
  const int* seq_lens;
  bf16* out;          // [B, nh*128]
  float* partial;     // [B*nh, nsplit, 132] or null
  int B, nh, kvh, max_len;
  int64_t ld;
  float scale_log2;
  // paged cache (block_tables != nullptr): [num_blocks, kvh, block_size, 128], sequence b's logical block i in physical block
  // block_tables[b * max_blocks + i]; dense: [B, kvh, max_len, 128]
  const int* block_tables;
  int max_blocks, block_size;
};

template <int G, bool PAGED>
__global__ void __launch_bounds__(NUM_THREADS, (G <= 4 ? 2 : 1)) decode_attention_bulk_kernel(const Params p) {
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ uint64_t full_bar[NST], empty_bar[NST];
  __shared__ float s_m[8][G], s_l[8][G];
  __shared__ float s_o[8][G][D];
  const int b = blockIdx.x / p.kvh, kh = blockIdx.x % p.kvh;
  const int total_len = min(p.seq_lens[b] + 1, p.max_len);   // the new token was appended at index seq_lens[b]
  const int nsplit = gridDim.y, split = blockIdx.y;
  const int chunk = (((max(total_len, 0) + nsplit - 1) / nsplit) + ROWS - 1) / ROWS * ROWS;
  const int t_begin = split * chunk;
  const int len = min(total_len, t_begin + chunk);
  const int nchunks = len > t_begin ? (len - t_begin + ROWS - 1) / ROWS : 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == 4) {
    // ------------------------------- producer -------------------------------
    if (lane == 0) {
      for (int c = 0; c < nchunks; ++c) {
        const int st = c % NST;
        mbar_wait(&empty_bar[st], ((c / NST) & 1) ^ 1);
        const int t0 = t_begin + c * ROWS;
        const uint32_t bytes = static_cast<uint32_t>(min(ROWS, len - t0)) * D * 2;
        size_t off;
        if constexpr (PAGED) {
          const int page = __ldg(p.block_tables + static_cast<size_t>(b) * p.max_blocks + t0 / p.block_size);
          off = ((static_cast<size_t>(page) * p.kvh + kh) * p.block_size + t0 % p.block_size) * D;
        } else {
          off = ((static_cast<size_t>(b) * p.kvh + kh) * p.max_len + t0) * D;
        }
        mbar_arrive_expect_tx(&full_bar[st], 2 * bytes);
        bulk_load(ring + st * 2 * CHUNK_BYTES, p.kc + off, bytes, &full_bar[st]);
        bulk_load(ring + st * 2 * CHUNK_BYTES + CHUNK_BYTES, p.vc + off, bytes, &full_bar[st]);
      }
    }
    return;
  }

  // ------------------------------- consumers -------------------------------
  const int hw = warp * 2 + (lane >> 4);               // half-warp id 0..7
  const int sub = lane & 15;                           // which 8 dims of the row
  const unsigned hmask = (lane < 16) ? 0x0000ffffu : 0xffff0000u;
  float q[G][8], o[G][8], m[G], l[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 qv = *reinterpret_cast<const uint4*>(p.qkv + static_cast<size_t>(b) * p.ld + (kh * G + g) * D + sub * 8);
    const uint32_t* qi = reinterpret_cast<const uint32_t*>(&qv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(qi[j]);
      q[g][2 * j] = f.x * p.scale_log2; q[g][2 * j + 1] = f.y * p.scale_log2;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[g][j] = 0.f;
    m[g] = -INFINITY; l[g] = 0.f;
  }
  constexpr int U = ROWS / 8;                          // rows per half-warp and chunk
  const uint32_t ring_s = smem_u32(ring);
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NST;
    const int rows = min(ROWS, len - (t_begin + c * ROWS));
    mbar_wait(&full_bar[st], (c / NST) & 1);
    const uint32_t kb = ring_s + st * 2 * CHUNK_BYTES, vb = kb + CHUNK_BYTES;
    uint4 kv[U], vv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = hw + 8 * u;
      if (r < rows) {
        kv[u] = ld_shared_v4(kb + r * (D * 2) + sub * 16);
        vv[u] = ld_shared_v4(vb + r * (D * 2) + sub * 16);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[st]);        // this warp's reads of the stage are in registers
    float sc[U][G];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t* ki = reinterpret_cast<const uint32_t*>(&kv[u]);
      float kf[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 a = unpack_bf16x2(ki[j]); kf[2 * j] = a.x; kf[2 * j + 1] = a.y; }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float sdot = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) sdot += q[g][j] * kf[j];
        sc[u][g] = sdot;
      }
    }
#pragma unroll
    for (int off = 8; off > 0; off >>= 1)
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int g = 0; g < G; ++g) sc[u][g] += __shfl_xor_sync(hmask, sc[u][g], off);
#pragma unroll
    for (int g = 0; g < G; ++g) {
      float mn = m[g];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (hw + 8 * u < rows) mn = fmaxf(mn, sc[u][g]);
      // m = -inf before this half-warp's first valid row -> corr = 0 (o and l are still 0); a chunk may hold no row of this
      // half-warp at all (mn = -inf): exp2(-inf - -inf) must not be evaluated
      const float corr = (mn == -INFINITY) ? 1.f : fast_exp2(m[g] - mn);
      m[g] = mn;
      l[g] *= corr;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[g][j] *= corr;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (hw + 8 * u < rows) {                         // uniform within the half-warp
        const uint32_t* vi = reinterpret_cast<const uint32_t*>(&vv[u]);
        float vf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 cc = unpack_bf16x2(vi[j]); vf[2 * j] = cc.x; vf[2 * j + 1] = cc.y; }
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float pr = fast_exp2(sc[u][g] - m[g]);
          l[g] += pr;
#pragma unroll
          for (int j = 0; j < 8; ++j) o[g][j] += pr * vf[j];
        }
      }
    }
  }
  // merge the 8 half-warp partials (consumer warps only: the producer warp has left)
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (sub == 0) { s_m[hw][g] = m[g]; s_l[hw][g] = l[g]; }
#pragma unroll
    for (int j = 0; j < 8; ++j) s_o[hw][g][sub * 8 + j] = o[g][j];
  }
  named_bar_sync(1, 128);
  for (int idx = threadIdx.x; idx < G * D; idx += 128) {
    const int g = idx / D, dd = idx % D;
    float mm = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) mm = fmaxf(mm, s_m[w][g]);
    float acc = 0.f, lt = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float f = (s_m[w][g] == -INFINITY) ? 0.f : exp2f(s_m[w][g] - mm);
      acc += s_o[w][g][dd] * f;
      lt += s_l[w][g] * f;
    }
    if (nsplit == 1) {
      p.out[static_cast<size_t>(b) * p.nh * D + (kh * G + g) * D + dd] = __float2bfloat16_rn(lt > 0.f ? acc / lt : 0.f);
    } else {
      float* dst = p.partial + ((static_cast<size_t>(b) * p.nh + kh * G + g) * nsplit + split) * (D + 4);
      dst[dd] = acc;
      if (dd == 0) { dst[D] = mm; dst[D + 1] = lt; }
    }
  }
}

template <bool PAGED>
static int launch(const Params& p, int G, int64_t num_splits, cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>(p.B * p.kvh), static_cast<unsigned>(num_splits));
#define B200_DAB(GG)                                                                                                 \
  case GG: {                                                                                                         \
    static bool attr_set = false;                                                                                    \
    if (!attr_set) {                                                                                                 \
      cudaError_t e = cudaFuncSetAttribute(decode_attention_bulk_kernel<GG, PAGED>,                                  \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);                \
      if (e != cudaSuccess) {                                                                                        \
        set_last_error("decode_attention smem attr: %s", cudaGetErrorString(e));                                     \
        return static_cast<int>(e);                                                                                  \
      }                                                                                                              \
      attr_set = true;                                                                                               \
    }                                                                                                                \
    launch_pdl(decode_attention_bulk_kernel<GG, PAGED>, grid, dim3(NUM_THREADS), SMEM_BYTES, stream, p);             \
  } break;
  switch (G) {
    B200_DAB(1) B200_DAB(2) B200_DAB(3) B200_DAB(4) B200_DAB(5) B200_DAB(6) B200_DAB(7) B200_DAB(8)
    default:
      return fail_arg("decode_attention_tc: GQA group size %d not instantiated (1 to 8)", G);
  }
#undef B200_DAB
  int rc = check_launch("decode_attention_tc");
  if (rc || num_splits == 1) return rc;
  return launch_decode_attention_merge(p.partial, p.out, p.B * p.nh, static_cast<int>(num_splits), stream);
}

}  // namespace dab
}  // namespace b200

extern "C" int b200_decode_attention_tc(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace,
                                        int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                                        int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  B200_CHECK_ARG(qkv && cache && seq_lens && out, "decode_attention_tc: null pointer");
  B200_CHECK_ARG(num_splits >= 1 && num_splits <= 64 && (num_splits == 1 || workspace),
                 "decode_attention_tc: bad num_splits / workspace");
  B200_CHECK_ARG(head_dim == 128, "decode_attention_tc: head_dim must be 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0 && max_len > 0 && ld % 8 == 0,
                 "decode_attention_tc: bad shape");
  using namespace b200;
  dab::Params p = {};
  p.qkv = static_cast<const bf16*>(qkv);
  p.kc = static_cast<const bf16*>(cache);
  p.vc = p.kc + static_cast<size_t>(B) * num_kv_heads * max_len * 128;
  p.seq_lens = seq_lens;
  p.out = static_cast<bf16*>(out);
  p.partial = static_cast<float*>(workspace);
  p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads); p.kvh = static_cast<int>(num_kv_heads);
  p.max_len = static_cast<int>(max_len); p.ld = ld;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  return dab::launch<false>(p, static_cast<int>(num_heads / num_kv_heads), num_splits, stream);
}

extern "C" int b200_decode_attention_paged(const void* qkv, const void* key_cache, const void* value_cache,
                                           const int32_t* block_tables, const int32_t* seq_lens, void* out, void* workspace,
                                           int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                           int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                           float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  B200_CHECK_ARG(qkv && key_cache && value_cache && block_tables && seq_lens && out, "decode_attention_paged: null pointer");
  B200_CHECK_ARG(num_splits >= 1 && num_splits <= 64 && (num_splits == 1 || workspace),
                 "decode_attention_paged: bad num_splits / workspace");
  B200_CHECK_ARG(head_dim == 128, "decode_attention_paged: head_dim must be 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(block_size == 32 || block_size == 64 || block_size == 128,
                 "decode_attention_paged: block_size must be 32, 64 or 128 (got %lld)", (long long)block_size);
  B200_CHECK_ARG(B > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0 && num_blocks > 0 && max_blocks_per_seq > 0 &&
                     ld % 8 == 0,
                 "decode_attention_paged: bad shape");
  using namespace b200;
  dab::Params p = {};
  p.qkv = static_cast<const bf16*>(qkv);
  p.kc = static_cast<const bf16*>(key_cache);
  p.vc = static_cast<const bf16*>(value_cache);
  p.seq_lens = seq_lens;
  p.out = static_cast<bf16*>(out);
  p.partial = static_cast<float*>(workspace);
  p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads); p.kvh = static_cast<int>(num_kv_heads);
  p.max_len = static_cast<int>(max_blocks_per_seq * block_size); p.ld = ld;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.block_tables = block_tables;
  p.max_blocks = static_cast<int>(max_blocks_per_seq); p.block_size = static_cast<int>(block_size);
  return dab::launch<true>(p, static_cast<int>(num_heads / num_kv_heads), num_splits, stream);
}
