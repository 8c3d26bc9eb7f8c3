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
//     and 129, whatever d is) are merged by decode_attention_merge_kernel.
// The int8 paged cache (KvCacheC8, cachekv_int8_type="static") runs the same kernel with 1-byte elements: a chunk keeps its
// row count (so a lane's rows x G scores, where the registers grow, are the bf16 kernel's) and is 4 KB, and the ring has 8
// stages instead of 4, so the bytes in flight per SM are unchanged.  Each lane turns its 8 bytes of a row into the exact fp32
// u - 128 (dequant_c8); the per-head dequantise scales are applied once: o_k on the query scale, o_v on the merged output
// before the normalisation and before a split-KV partial is written.
// b200_decode_attention (decode_attention_kernel below, plain global loads, dense cache) computes the same function and is the
// cross-check.  Cache rows are addressed through KvCache (kv_cache.cuh).
#include <type_traits>

#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"
#include "kv_cache.cuh"

namespace b200 {
namespace dab {

constexpr int SMEM_BYTES = 65536;              // the ring: NST stages of a K and a V chunk
constexpr int NUM_THREADS = 160;               // 4 consumer warps + 1 producer warp
// K (and as much V) per stage: 32 rows at d = 128, 64 rows at d = 64, whatever the element type: 8 KB in 4 stages (bf16),
// 4 KB in 8 stages (uint8)
template <typename T>
constexpr int CHUNK_BYTES = 4096 * static_cast<int>(sizeof(T));
template <typename T>
constexpr int NST = SMEM_BYTES / (2 * CHUNK_BYTES<T>);

__device__ __forceinline__ uint2 ld_shared_v2(uint32_t saddr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(saddr));
  return v;
}

template <typename T>
struct Params {
  const bf16* qkv;
  KvCacheT<T> kv;     // dense or paged, as the PAGED instantiation says; uint8 only paged
  const int* seq_lens;
  bf16* out;          // [B, nh*d]
  float* partial;     // [B*nh, nsplit, 132] or null
  int B, nh;
  int64_t ld;
  float scale_log2;
};

// A lane's 8 cache elements of one row -> fp32: bf16 as they are, uint8 as the exact u - 128 (kv_cache.cuh)
__device__ __forceinline__ void row8_to_f32(const uint4& x, float (&f)[8]) {
  const uint32_t* xi = reinterpret_cast<const uint32_t*>(&x);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float2 a = unpack_bf16x2(xi[j]); f[2 * j] = a.x; f[2 * j + 1] = a.y; }
}
__device__ __forceinline__ void row8_to_f32(const uint2& x, float (&f)[8]) {
  f[0] = dequant_c8<0>(x.x); f[1] = dequant_c8<1>(x.x); f[2] = dequant_c8<2>(x.x); f[3] = dequant_c8<3>(x.x);
  f[4] = dequant_c8<0>(x.y); f[5] = dequant_c8<1>(x.y); f[6] = dequant_c8<2>(x.y); f[7] = dequant_c8<3>(x.y);
}

template <int D, int G, bool PAGED, typename T>
__global__ void __launch_bounds__(NUM_THREADS, (G <= 4 ? 2 : 1)) decode_attention_bulk_kernel(const Params<T> p) {
  constexpr bool C8 = sizeof(T) == 1;
  constexpr int ES = static_cast<int>(sizeof(T));            // bytes per cache element
  constexpr int CHUNK = CHUNK_BYTES<T>, NSTAGE = NST<T>;
  constexpr int ROWS = CHUNK / (D * ES);                     // cache rows per chunk
  constexpr int LPR = D / 8, LPR_LOG2 = D == 128 ? 4 : 3;   // lanes per cache row
  constexpr int NG = 128 / LPR;                              // row groups of the four consumer warps
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ uint64_t full_bar[NSTAGE], empty_bar[NSTAGE];
  __shared__ float s_m[NG][G], s_l[NG][G];
  __shared__ float s_o[NG][G][D];
  const int b = blockIdx.x / p.kv.kvh, kh = blockIdx.x % p.kv.kvh;
  const int total_len = min(p.seq_lens[b] + 1, p.kv.max_len);   // the new token was appended at index seq_lens[b]
  const int nsplit = gridDim.y, split = blockIdx.y;
  const int chunk = (((max(total_len, 0) + nsplit - 1) / nsplit) + ROWS - 1) / ROWS * ROWS;
  const int t_begin = split * chunk;
  const int len = min(total_len, t_begin + chunk);
  const int nchunks = len > t_begin ? (len - t_begin + ROWS - 1) / ROWS : 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NSTAGE; ++i) {
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
        const int st = c % NSTAGE;
        mbar_wait(&empty_bar[st], ((c / NSTAGE) & 1) ^ 1);
        const int t0 = t_begin + c * ROWS;
        const uint32_t bytes = static_cast<uint32_t>(min(ROWS, len - t0)) * D * ES;
        if constexpr (PAGED && ROWS > 32) {
          // t0 is a multiple of ROWS, so the chunk starts on a page and spans ROWS / block_size pages when those are shorter
          mbar_arrive_expect_tx(&full_bar[st], 2 * bytes);
          const int n = min(ROWS, len - t0);
          for (int r0 = 0; r0 < n; r0 += p.kv.block_size) {
            const size_t off = p.kv.template offset<true, D>(b, kh, t0 + r0);
            const uint32_t piece = static_cast<uint32_t>(min(p.kv.block_size, n - r0)) * D * ES;
            bulk_load(ring + st * 2 * CHUNK + r0 * D * ES, p.kv.k + off, piece, &full_bar[st]);
            bulk_load(ring + st * 2 * CHUNK + CHUNK + r0 * D * ES, p.kv.v + off, piece, &full_bar[st]);
          }
          continue;
        }
        const size_t off = p.kv.template offset<PAGED, D>(b, kh, t0);
        mbar_arrive_expect_tx(&full_bar[st], 2 * bytes);
        bulk_load(ring + st * 2 * CHUNK, p.kv.k + off, bytes, &full_bar[st]);
        bulk_load(ring + st * 2 * CHUNK + CHUNK, p.kv.v + off, bytes, &full_bar[st]);
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
  float q_scale = p.scale_log2;
  if constexpr (C8) q_scale *= __bfloat162float(p.kv.k_out_scale[kh]);   // K = (u - 128) o_k: o_k folds into the query scale
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 qv = *reinterpret_cast<const uint4*>(p.qkv + static_cast<size_t>(b) * p.ld + (kh * G + g) * D + sub * 8);
    const uint32_t* qi = reinterpret_cast<const uint32_t*>(&qv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(qi[j]);
      q[g][2 * j] = f.x * q_scale; q[g][2 * j + 1] = f.y * q_scale;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[g][j] = 0.f;
    m[g] = -INFINITY; l[g] = 0.f;
  }
  constexpr int U = ROWS / NG;                         // rows per row group and chunk
  const uint32_t ring_s = smem_u32(ring);
  // a lane's 8 elements of a row: one 16-byte word of bf16, or the first half of one of uint8
  using Row8 = typename std::conditional<C8, uint2, uint4>::type;
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NSTAGE;
    const int rows = min(ROWS, len - (t_begin + c * ROWS));
    mbar_wait(&full_bar[st], (c / NSTAGE) & 1);
    const uint32_t kb = ring_s + st * 2 * CHUNK, vb = kb + CHUNK;
    Row8 kv[U], vv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = hw + NG * u;
      if (r < rows) {
        if constexpr (C8) {
          kv[u] = ld_shared_v2(kb + r * D + sub * 8);
          vv[u] = ld_shared_v2(vb + r * D + sub * 8);
        } else {
          kv[u] = ld_shared_v4(kb + r * (D * 2) + sub * 16);
          vv[u] = ld_shared_v4(vb + r * (D * 2) + sub * 16);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[st]);        // this warp's reads of the stage are in registers
    float sc[U][G];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float kf[8];
      row8_to_f32(kv[u], kf);
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
        float vf[8];
        row8_to_f32(vv[u], vf);
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
  float v_scale = 1.f;
  if constexpr (C8) v_scale = __bfloat162float(p.kv.v_out_scale[kh]);      // V = (u - 128) o_v
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
    if constexpr (C8) acc *= v_scale;
    if (nsplit == 1) {
      p.out[static_cast<size_t>(b) * p.nh * D + (kh * G + g) * D + dd] = __float2bfloat16_rn(lt > 0.f ? acc / lt : 0.f);
    } else {
      float* dst = p.partial + ((static_cast<size_t>(b) * p.nh + kh * G + g) * nsplit + split) * DECODE_PART_ROW;
      dst[dd] = acc;
      if (dd == 0) { dst[DECODE_PART_M] = mm; dst[DECODE_PART_M + 1] = lt; }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The cross-check: one query token per sequence over the dense cache, GQA group shares each K/V row read.
//   CTA = (batch, kv head); 4 warps; a row group of D / 8 lanes x 16 B reads one K row (a half-warp at d = 128, a quarter
//   at d = 64), so a warp covers 2 (4) cache rows per load; every lane keeps its 8 dims of q / o for the G q-heads of the
//   group in registers; online softmax (exp2, fp32) per row group, merged across the 8 (16) row groups through shared memory.
// HBM roofline: 2 * len * d * 2 bytes per (b, kv head).
// Split-KV partials: DECODE_PART_ROW-float rows (common.cuh).
// ------------------------------------------------------------------------------------------------

template <int D, int G>
__global__ void __launch_bounds__(128, (G <= 4 ? 4 : 2)) decode_attention_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ kc,
                                                               const bf16* __restrict__ vc, const int* __restrict__ seq_lens,
                                                               bf16* __restrict__ out, float* __restrict__ partial, int nh,
                                                               int kvh, int max_len, int64_t ld, float scale_log2) {
  constexpr int LPR = D / 8, LPR_LOG2 = D == 128 ? 4 : 3;   // lanes per cache row
  constexpr int NG = 128 / LPR;                              // row groups per CTA
  __shared__ float s_m[NG][G], s_l[NG][G];
  __shared__ float s_o[NG][G][D];
  pdl_launch_dependents();
  const int b = blockIdx.x / kvh, kh = blockIdx.x % kvh;
  const int total_len = min(seq_lens[b] + 1, max_len);  // the new token was appended at index seq_lens[b]
  // split-KV: gridDim.y CTAs share one (b, kv head); each takes a contiguous range of the cache
  const int nsplit = gridDim.y, split = blockIdx.y;
  const int chunk = (total_len + nsplit - 1) / nsplit;
  const int t_begin = split * chunk;
  const int len = min(total_len, t_begin + chunk);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int hw = warp * (32 / LPR) + (lane >> LPR_LOG2);   // row group id 0..NG-1
  const int sub = lane & (LPR - 1);                         // which 8 dims of the row
  unsigned hmask;
  if constexpr (D == 128) hmask = (lane < 16) ? 0x0000ffffu : 0xffff0000u;
  else hmask = 0xffu << (lane & 24);
  float q[G][8], o[G][8], m[G], l[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 qv = *reinterpret_cast<const uint4*>(qkv + static_cast<size_t>(b) * ld + (kh * G + g) * D + sub * 8);
    const uint32_t* qi = reinterpret_cast<const uint32_t*>(&qv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(qi[j]);
      q[g][2 * j] = f.x * scale_log2; q[g][2 * j + 1] = f.y * scale_log2;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[g][j] = 0.f;
    m[g] = -INFINITY; l[g] = 0.f;
  }
  const size_t head_off = KvCache::dense_row(b, kh, 0, kvh, max_len) * D;   // the rows of one (sequence, head) are consecutive
  const bf16* kbase = kc + head_off;
  const bf16* vbase = vc + head_off;
  constexpr int U = 4;      // rows in flight per row group: 8 x 16-byte loads issued before any math (memory-level parallelism)
  for (int t0 = t_begin + hw; t0 < len; t0 += NG * U) {
    uint4 kv[U], vv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int t = t0 + NG * u;
      if (t < len) {
        kv[u] = ld_nc_v4(reinterpret_cast<const uint4*>(kbase + static_cast<size_t>(t) * D) + sub);
        vv[u] = ld_nc_v4(reinterpret_cast<const uint4*>(vbase + static_cast<size_t>(t) * D) + sub);
      }
    }
    // Blockwise online softmax over the U rows of this iteration: all U*G dot products and their half-warp reductions are
    // independent (instruction-level parallelism instead of one dependent chain per row), then one max / one rescale per
    // head and iteration.
    float sc[U][G];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t* ki = reinterpret_cast<const uint32_t*>(&kv[u]);
      float kf[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 a = unpack_bf16x2(ki[j]); kf[2 * j] = a.x; kf[2 * j + 1] = a.y; }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s += q[g][j] * kf[j];
        sc[u][g] = s;
      }
    }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) {
      // the row groups of a warp can have different trip counts: shuffle within the row group only
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int g = 0; g < G; ++g) sc[u][g] += __shfl_xor_sync(hmask, sc[u][g], off);
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      float mn = m[g];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (t0 + NG * u < len) mn = fmaxf(mn, sc[u][g]);
      const float corr = fast_exp2(m[g] - mn);      // m = -inf on the first block -> corr = 0, o and l are still 0
      m[g] = mn;
      l[g] *= corr;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[g][j] *= corr;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (t0 + NG * u < len) {                     // uniform within the row group
        const uint32_t* vi = reinterpret_cast<const uint32_t*>(&vv[u]);
        float vf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 c = unpack_bf16x2(vi[j]); vf[2 * j] = c.x; vf[2 * j + 1] = c.y; }
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float p = fast_exp2(sc[u][g] - m[g]);
          l[g] += p;
#pragma unroll
          for (int j = 0; j < 8; ++j) o[g][j] += p * vf[j];
        }
      }
    }
  }
  // merge the NG row-group partials
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (sub == 0) { s_m[hw][g] = m[g]; s_l[hw][g] = l[g]; }
#pragma unroll
    for (int j = 0; j < 8; ++j) s_o[hw][g][sub * 8 + j] = o[g][j];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < G * D; idx += blockDim.x) {
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
      out[static_cast<size_t>(b) * nh * D + (kh * G + g) * D + dd] = __float2bfloat16_rn(lt > 0.f ? acc / lt : 0.f);
    } else {
      float* dst = partial + ((static_cast<size_t>(b) * nh + kh * G + g) * nsplit + split) * DECODE_PART_ROW;
      dst[dd] = acc;
      if (dd == 0) { dst[DECODE_PART_M] = mm; dst[DECODE_PART_M + 1] = lt; }
    }
  }
}

// merge the split-KV partials: one warp per (b, head); reads the first D columns of o
template <int D>
__global__ void decode_attention_merge_kernel(const float* __restrict__ partial, bf16* __restrict__ out, int rows, int nsplit) {
  constexpr int W = DECODE_PART_ROW, M = DECODE_PART_M;
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* base = partial + static_cast<size_t>(row) * nsplit * W;
  float mm = -INFINITY;
  for (int s = 0; s < nsplit; ++s) mm = fmaxf(mm, base[s * W + M]);
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, lt = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float ms = base[s * W + M];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
    lt += base[s * W + M + 1] * f;
    if constexpr (D == 128) {
      const float4 o = *reinterpret_cast<const float4*>(base + s * W + lane * 4);
      acc[0] += o.x * f; acc[1] += o.y * f; acc[2] += o.z * f; acc[3] += o.w * f;
    } else {
      const float2 o = *reinterpret_cast<const float2*>(base + s * W + lane * 2);
      acc[0] += o.x * f; acc[1] += o.y * f;
    }
  }
  const float inv = lt > 0.f ? 1.f / lt : 0.f;
  if constexpr (D == 128) {
    uint2 o2;
    o2.x = pack_bf16x2(acc[0] * inv, acc[1] * inv);
    o2.y = pack_bf16x2(acc[2] * inv, acc[3] * inv);
    *reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * D + lane * 4) = o2;
  } else {
    *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(row) * D + lane * 2) = pack_bf16x2(acc[0] * inv, acc[1] * inv);
  }
}

static int launch_merge(const float* partial, bf16* out, int rows, int nsplit, int head_dim, cudaStream_t stream) {
  if (head_dim == 64) launch_pdl(decode_attention_merge_kernel<64>, dim3((rows + 3) / 4), dim3(128), 0, stream, partial, out, rows, nsplit);
  else launch_pdl(decode_attention_merge_kernel<128>, dim3((rows + 3) / 4), dim3(128), 0, stream, partial, out, rows, nsplit);
  return check_launch("decode_attention(merge)");
}

template <int D, bool PAGED, typename T>
static int launch(const Params<T>& p, int G, int64_t num_splits, cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>(p.B * p.kv.kvh), static_cast<unsigned>(num_splits));
#define B200_DAB(GG)                                                                                                 \
  case GG: {                                                                                                         \
    static bool attr_set = false;                                                                                    \
    if (!attr_set) {                                                                                                 \
      cudaError_t e = cudaFuncSetAttribute(decode_attention_bulk_kernel<D, GG, PAGED, T>,                               \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);                \
      if (e != cudaSuccess) {                                                                                        \
        set_last_error("decode_attention smem attr: %s", cudaGetErrorString(e));                                     \
        return static_cast<int>(e);                                                                                  \
      }                                                                                                              \
      attr_set = true;                                                                                               \
    }                                                                                                                \
    launch_pdl(decode_attention_bulk_kernel<D, GG, PAGED, T>, grid, dim3(NUM_THREADS), SMEM_BYTES, stream, p);             \
  } break;
  switch (G) {   // 1 to 8: check_decode_attention()
    B200_DAB(1) B200_DAB(2) B200_DAB(3) B200_DAB(4) B200_DAB(5) B200_DAB(6) B200_DAB(7) B200_DAB(8)
  }
#undef B200_DAB
  int rc = check_launch("decode_attention_tc");
  if (rc || num_splits == 1) return rc;
  return launch_merge(p.partial, p.out, p.B * p.nh, static_cast<int>(num_splits), D, stream);
}

}  // namespace dab

// The checks every decode-attention entry point makes beyond its cache view; `what` names the entry point in the message.
template <typename T>
int check_decode_attention(const char* what, const KvCacheT<T>& kv, const void* qkv, const int32_t* seq_lens, const void* out,
                           const void* workspace, int64_t B, int64_t num_heads, int64_t ld, int64_t num_splits) {
  B200_CHECK_ARG(qkv && seq_lens && out, "%s: null pointer", what);
  B200_CHECK_ARG(num_splits >= 1 && num_splits <= 64 && (num_splits == 1 || workspace), "%s: bad num_splits / workspace", what);
  B200_CHECK_ARG(kv.d == 64 || kv.d == 128, "%s: head_dim must be 64 or 128 (got %d)", what, kv.d);
  B200_CHECK_ARG(B > 0 && num_heads > 0 && num_heads % kv.kvh == 0 && ld % 8 == 0, "%s: bad shape", what);
  B200_CHECK_ARG(num_heads / kv.kvh <= 8, "%s: GQA group size %lld not instantiated (1 to 8)", what,
                 (long long)(num_heads / kv.kvh));
  return 0;
}

// Streaming-kernel decode attention over a dense or paged view whose arguments passed check_decode_attention().  The uint8
// view is paged only.
template <typename T>
int launch_decode_attention(const KvCacheT<T>& kv, const void* qkv, const int32_t* seq_lens, void* out, void* workspace, int64_t B,
                            int64_t num_heads, int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  dab::Params<T> p = {};
  p.qkv = static_cast<const bf16*>(qkv);
  p.kv = kv;
  p.seq_lens = seq_lens;
  p.out = static_cast<bf16*>(out);
  p.partial = static_cast<float*>(workspace);
  p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads);
  p.ld = ld;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  const int G = static_cast<int>(num_heads / kv.kvh);
  if constexpr (sizeof(T) == 1) {
    return kv.d == 64 ? dab::launch<64, true>(p, G, num_splits, stream) : dab::launch<128, true>(p, G, num_splits, stream);
  } else {
    if (kv.block_tables != nullptr)
      return kv.d == 64 ? dab::launch<64, true>(p, G, num_splits, stream) : dab::launch<128, true>(p, G, num_splits, stream);
    return kv.d == 64 ? dab::launch<64, false>(p, G, num_splits, stream) : dab::launch<128, false>(p, G, num_splits, stream);
  }
}
template int check_decode_attention(const char*, const KvCache&, const void*, const int32_t*, const void*, const void*, int64_t,
                                    int64_t, int64_t, int64_t);
template int check_decode_attention(const char*, const KvCacheC8&, const void*, const int32_t*, const void*, const void*, int64_t,
                                    int64_t, int64_t, int64_t);
template int launch_decode_attention(const KvCache&, const void*, const int32_t*, void*, void*, int64_t, int64_t, int64_t, float,
                                     int64_t, cudaStream_t);
template int launch_decode_attention(const KvCacheC8&, const void*, const int32_t*, void*, void*, int64_t, int64_t, int64_t, float,
                                     int64_t, cudaStream_t);

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_decode_attention_workspace_bytes(int64_t B, int64_t num_heads, int64_t num_splits) {
  return num_splits > 1 ? B * num_heads * num_splits * DECODE_PART_ROW * 4 : 0;
}

extern "C" int b200_decode_attention(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace,
                                     int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                                     int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  KvCache kv;
  if (int rc = dense_kv_cache(&kv, cache, B, num_kv_heads, head_dim, max_len, "decode_attention")) return rc;
  if (int rc = check_decode_attention("decode_attention", kv, qkv, seq_lens, out, workspace, B, num_heads, ld, num_splits))
    return rc;
  const int G = static_cast<int>(num_heads / num_kv_heads);
  const float sl2 = softmax_scale * 1.4426950408889634f;
  const dim3 grid(static_cast<unsigned>(B * num_kv_heads), static_cast<unsigned>(num_splits)), block(128);
  const bf16* q = static_cast<const bf16*>(qkv);
  bf16* o = static_cast<bf16*>(out);
  float* part = static_cast<float*>(workspace);
#define B200_DA(DD, GG)                                                                                              \
  case GG:                                                                                                           \
    dab::decode_attention_kernel<DD, GG><<<grid, block, 0, stream>>>(q, kv.k, kv.v, seq_lens, o, part, (int)num_heads, \
                                                                     kv.kvh, kv.max_len, ld, sl2);                  \
    break;
#define B200_DA_G(DD)                                                                                                \
  switch (G) { /* 1 to 8: check_decode_attention() */                                                               \
    B200_DA(DD, 1) B200_DA(DD, 2) B200_DA(DD, 3) B200_DA(DD, 4) B200_DA(DD, 5) B200_DA(DD, 6) B200_DA(DD, 7)          \
    B200_DA(DD, 8)                                                                                                   \
  }
  if (head_dim == 64) {
    B200_DA_G(64)
  } else {
    B200_DA_G(128)
  }
#undef B200_DA_G
#undef B200_DA
  int rc = check_launch("decode_attention");
  if (rc || num_splits == 1) return rc;
  return dab::launch_merge(part, o, static_cast<int>(B * num_heads), static_cast<int>(num_splits), (int)head_dim, stream);
}

extern "C" int b200_decode_attention_tc(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace,
                                        int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                                        int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  KvCache kv;
  if (int rc = dense_kv_cache(&kv, cache, B, num_kv_heads, head_dim, max_len, "decode_attention_tc")) return rc;
  if (int rc = check_decode_attention("decode_attention_tc", kv, qkv, seq_lens, out, workspace, B, num_heads, ld, num_splits))
    return rc;
  return launch_decode_attention(kv, qkv, seq_lens, out, workspace, B, num_heads, ld, softmax_scale, num_splits, stream);
}

extern "C" int b200_decode_attention_paged(const void* qkv, const void* key_cache, const void* value_cache,
                                           const int32_t* block_tables, const int32_t* seq_lens, void* out, void* workspace,
                                           int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                           int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                           float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  KvCache kv;
  if (int rc = paged_kv_cache(&kv, key_cache, value_cache, block_tables, num_kv_heads, head_dim, block_size, max_blocks_per_seq,
                              "decode_attention_paged"))
    return rc;
  B200_CHECK_ARG(num_blocks > 0, "decode_attention_paged: bad shape");
  if (int rc = check_decode_attention("decode_attention_paged", kv, qkv, seq_lens, out, workspace, B, num_heads, ld, num_splits))
    return rc;
  return launch_decode_attention(kv, qkv, seq_lens, out, workspace, B, num_heads, ld, softmax_scale, num_splits, stream);
}

extern "C" int b200_decode_attention_paged_c8(const void* qkv, const void* key_cache, const void* value_cache,
                                              const int32_t* block_tables, const void* cache_k_out_scale,
                                              const void* cache_v_out_scale, const int32_t* seq_lens, void* out, void* workspace,
                                              int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                              int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                              float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  KvCacheC8 kv;
  if (int rc = paged_kv_cache_c8(&kv, key_cache, value_cache, block_tables, nullptr, nullptr, cache_k_out_scale, cache_v_out_scale,
                                 false, true, num_kv_heads, head_dim, block_size, max_blocks_per_seq, "decode_attention_paged_c8"))
    return rc;
  B200_CHECK_ARG(num_blocks > 0, "decode_attention_paged_c8: bad shape");
  if (int rc = check_decode_attention("decode_attention_paged_c8", kv, qkv, seq_lens, out, workspace, B, num_heads, ld, num_splits))
    return rc;
  return launch_decode_attention(kv, qkv, seq_lens, out, workspace, B, num_heads, ld, softmax_scale, num_splits, stream);
}
