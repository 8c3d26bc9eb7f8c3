// Decode attention over the dense and the paged KV cache on Hopper: one query token per sequence, GQA, head_dim 64 or 128.
//
//   out[b, h, :] = softmax(q[b, h, :] K[b, kv(h), 0:len_b, :]^T / sqrt(d)) V[b, kv(h), 0:len_b, :]
//
// Replaces the attention half of masked_multihead_attention / the decode branch of append_attention
// (paddlenlp/experimental/transformers/fused_transformer_layers.py:884-893;
//  csrc/gpu/append_attn/append_attention_c16_impl.cuh:377-744, split-KV :826-1000).
//
// The op is a pure stream of the cache through the SM (2*len*d*2 bytes per (b, kv head), ~4 flop/byte, far below the
// tensor-core ridge point), so the design goal is bytes in flight:
//   * one producer warp moves 8 KB K and V chunks (32 rows at d = 128, 64 rows at d = 64) with the bulk-copy engine
//     (cp.async.bulk) into a 4-stage shared-memory ring, completion on mbarriers; with two CTAs per SM (GQA groups up to 4)
//     that is 128 KB of cache in flight per SM at either d, independent of the math.  A chunk is contiguous in the dense
//     cache and within a page (32, 64 or 128 rows); a 64-row chunk over 32-row pages is two bulk copies per tensor;
//   * four consumer warps: a row group of D / 8 lanes x 8 dims per cache row (half-warps at d = 128, quarter-warps at
//     d = 64), the GQA group's G heads share every K/V row, online softmax in fp32 (exp2), the row-group partials merged
//     through shared memory at the end;
//   * split-KV partials ([B*nh, nsplit, 132] fp32: unnormalised o in the first d columns, running max and sum at columns 128
//     and 129, whatever d is) are merged by decode_attention_merge_kernel (generation.cu).
// b200_decode_attention (generation.cu, plain global loads) computes the same function and is the cross-check.
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
// generation.cu
int launch_decode_attention_merge(const float* partial, void* out, int rows, int nsplit, int head_dim, cudaStream_t stream);

namespace dab {

constexpr int CHUNK_BYTES = 8192;              // K (and as much V) per stage: 32 rows at d = 128, 64 rows at d = 64
constexpr int NST = 4;                         // ring stages
constexpr int SMEM_BYTES = NST * 2 * CHUNK_BYTES;
constexpr int NUM_THREADS = 160;               // 4 consumer warps + 1 producer warp

struct Params {
  const bf16* qkv;
  const bf16* kc;
  const bf16* vc;
  const int* seq_lens;
  bf16* out;          // [B, nh*d]
  float* partial;     // [B*nh, nsplit, 132] or null
  int B, nh, kvh, max_len;
  int64_t ld;
  float scale_log2;
  // paged cache (block_tables != nullptr): [num_blocks, kvh, block_size, d], sequence b's logical block i in physical block
  // block_tables[b * max_blocks + i]; dense: [B, kvh, max_len, d]
  const int* block_tables;
  int max_blocks, block_size;
};

template <int D, int G, bool PAGED>
__global__ void __launch_bounds__(NUM_THREADS, (G <= 4 ? 2 : 1)) decode_attention_bulk_kernel(const Params p) {
  constexpr int ROWS = CHUNK_BYTES / (D * 2);                // cache rows per chunk
  constexpr int LPR = D / 8, LPR_LOG2 = D == 128 ? 4 : 3;   // lanes per cache row
  constexpr int NG = 128 / LPR;                              // row groups of the four consumer warps
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ uint64_t full_bar[NST], empty_bar[NST];
  __shared__ float s_m[NG][G], s_l[NG][G];
  __shared__ float s_o[NG][G][D];
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
        if constexpr (PAGED && ROWS > 32) {
          // t0 is a multiple of ROWS, so the chunk starts on a page and spans ROWS / block_size pages when those are shorter
          mbar_arrive_expect_tx(&full_bar[st], 2 * bytes);
          const int n = min(ROWS, len - t0);
          for (int r0 = 0; r0 < n; r0 += p.block_size) {
            const int t = t0 + r0;
            const int page = __ldg(p.block_tables + static_cast<size_t>(b) * p.max_blocks + t / p.block_size);
            const size_t off = ((static_cast<size_t>(page) * p.kvh + kh) * p.block_size + t % p.block_size) * D;
            const uint32_t piece = static_cast<uint32_t>(min(p.block_size, n - r0)) * D * 2;
            bulk_load(ring + st * 2 * CHUNK_BYTES + r0 * D * 2, p.kc + off, piece, &full_bar[st]);
            bulk_load(ring + st * 2 * CHUNK_BYTES + CHUNK_BYTES + r0 * D * 2, p.vc + off, piece, &full_bar[st]);
          }
          continue;
        }
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
  const int hw = warp * (32 / LPR) + (lane >> LPR_LOG2);   // row group id 0..NG-1
  const int sub = lane & (LPR - 1);                         // which 8 dims of the row
  unsigned hmask;
  if constexpr (D == 128) hmask = (lane < 16) ? 0x0000ffffu : 0xffff0000u;
  else hmask = 0xffu << (lane & 24);
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
  constexpr int U = ROWS / NG;                         // rows per row group and chunk
  const uint32_t ring_s = smem_u32(ring);
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NST;
    const int rows = min(ROWS, len - (t_begin + c * ROWS));
    mbar_wait(&full_bar[st], (c / NST) & 1);
    const uint32_t kb = ring_s + st * 2 * CHUNK_BYTES, vb = kb + CHUNK_BYTES;
    uint4 kv[U], vv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = hw + NG * u;
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
    for (int off = LPR / 2; off > 0; off >>= 1)
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int g = 0; g < G; ++g) sc[u][g] += __shfl_xor_sync(hmask, sc[u][g], off);
#pragma unroll
    for (int g = 0; g < G; ++g) {
      float mn = m[g];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (hw + NG * u < rows) mn = fmaxf(mn, sc[u][g]);
      // m = -inf before this row group's first valid row -> corr = 0 (o and l are still 0); a chunk may hold no row of this
      // row group at all (mn = -inf): exp2(-inf - -inf) must not be evaluated
      const float corr = (mn == -INFINITY) ? 1.f : fast_exp2(m[g] - mn);
      m[g] = mn;
      l[g] *= corr;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[g][j] *= corr;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (hw + NG * u < rows) {                        // uniform within the row group
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
  // merge the NG row-group partials (consumer warps only: the producer warp has left)
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
    for (int w = 0; w < NG; ++w) mm = fmaxf(mm, s_m[w][g]);
    float acc = 0.f, lt = 0.f;
#pragma unroll
    for (int w = 0; w < NG; ++w) {
      const float f = (s_m[w][g] == -INFINITY) ? 0.f : exp2f(s_m[w][g] - mm);
      acc += s_o[w][g][dd] * f;
      lt += s_l[w][g] * f;
    }
    if (nsplit == 1) {
      p.out[static_cast<size_t>(b) * p.nh * D + (kh * G + g) * D + dd] = __float2bfloat16_rn(lt > 0.f ? acc / lt : 0.f);
    } else {
      float* dst = p.partial + ((static_cast<size_t>(b) * p.nh + kh * G + g) * nsplit + split) * DECODE_PART_ROW;
      dst[dd] = acc;
      if (dd == 0) { dst[DECODE_PART_M] = mm; dst[DECODE_PART_M + 1] = lt; }
    }
  }
}

template <int D, bool PAGED>
static int launch(const Params& p, int G, int64_t num_splits, cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>(p.B * p.kvh), static_cast<unsigned>(num_splits));
#define B200_DAB(GG)                                                                                                 \
  case GG: {                                                                                                         \
    static bool attr_set = false;                                                                                    \
    if (!attr_set) {                                                                                                 \
      cudaError_t e = cudaFuncSetAttribute(decode_attention_bulk_kernel<D, GG, PAGED>,                               \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);                \
      if (e != cudaSuccess) {                                                                                        \
        set_last_error("decode_attention smem attr: %s", cudaGetErrorString(e));                                     \
        return static_cast<int>(e);                                                                                  \
      }                                                                                                              \
      attr_set = true;                                                                                               \
    }                                                                                                                \
    launch_pdl(decode_attention_bulk_kernel<D, GG, PAGED>, grid, dim3(NUM_THREADS), SMEM_BYTES, stream, p);             \
  } break;
  switch (G) {
    B200_DAB(1) B200_DAB(2) B200_DAB(3) B200_DAB(4) B200_DAB(5) B200_DAB(6) B200_DAB(7) B200_DAB(8)
    default:
      return fail_arg("decode_attention_tc: GQA group size %d not instantiated (1 to 8)", G);
  }
#undef B200_DAB
  int rc = check_launch("decode_attention_tc");
  if (rc || num_splits == 1) return rc;
  return launch_decode_attention_merge(p.partial, p.out, p.B * p.nh, static_cast<int>(num_splits), D, stream);
}

}  // namespace dab
}  // namespace b200

extern "C" int b200_decode_attention_tc(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace,
                                        int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                                        int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  B200_CHECK_ARG(qkv && cache && seq_lens && out, "decode_attention_tc: null pointer");
  B200_CHECK_ARG(num_splits >= 1 && num_splits <= 64 && (num_splits == 1 || workspace),
                 "decode_attention_tc: bad num_splits / workspace");
  B200_CHECK_ARG(head_dim == 64 || head_dim == 128, "decode_attention_tc: head_dim must be 64 or 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0 && max_len > 0 && ld % 8 == 0,
                 "decode_attention_tc: bad shape");
  using namespace b200;
  dab::Params p = {};
  p.qkv = static_cast<const bf16*>(qkv);
  p.kc = static_cast<const bf16*>(cache);
  p.vc = p.kc + static_cast<size_t>(B) * num_kv_heads * max_len * head_dim;
  p.seq_lens = seq_lens;
  p.out = static_cast<bf16*>(out);
  p.partial = static_cast<float*>(workspace);
  p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads); p.kvh = static_cast<int>(num_kv_heads);
  p.max_len = static_cast<int>(max_len); p.ld = ld;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  const int G = static_cast<int>(num_heads / num_kv_heads);
  return head_dim == 64 ? dab::launch<64, false>(p, G, num_splits, stream) : dab::launch<128, false>(p, G, num_splits, stream);
}

extern "C" int b200_decode_attention_paged(const void* qkv, const void* key_cache, const void* value_cache,
                                           const int32_t* block_tables, const int32_t* seq_lens, void* out, void* workspace,
                                           int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                           int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                           float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  B200_CHECK_ARG(qkv && key_cache && value_cache && block_tables && seq_lens && out, "decode_attention_paged: null pointer");
  B200_CHECK_ARG(num_splits >= 1 && num_splits <= 64 && (num_splits == 1 || workspace),
                 "decode_attention_paged: bad num_splits / workspace");
  B200_CHECK_ARG(head_dim == 64 || head_dim == 128, "decode_attention_paged: head_dim must be 64 or 128 (got %lld)",
                 (long long)head_dim);
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
  const int G = static_cast<int>(num_heads / num_kv_heads);
  return head_dim == 64 ? dab::launch<64, true>(p, G, num_splits, stream) : dab::launch<128, true>(p, G, num_splits, stream);
}
