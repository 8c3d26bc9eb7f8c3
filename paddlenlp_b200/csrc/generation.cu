// Generation (KV-cache decode) hot path and per-step bookkeeping ops — the bf16, non-quantised subset of the
// reference's `paddlenlp_ops` (csrc/gpu/*.cu) plus the Paddle-core ops FusedMultiTransformer calls
// (paddlenlp/experimental/transformers/fused_transformer_layers.py).  All of it is HBM-/latency-bound integer and
// elementwise work: coalesced 128-bit accesses, no tensor cores, no host synchronisation (the decode step is
// CUDA-graph capturable: every data-dependent quantity — sequence lengths, stop flags — is read from device memory).
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"
#include "kv_cache.cuh"

namespace b200 {
namespace gen {

// ------------------------------------------------------------------------------------------------
// fused residual-add + RMSNorm -> (normed, new_residual)
// Reference: fused_rms_norm(x, norm_weight, ..., residual=residual) -> (out, residual_out)
// (fused_transformer_layers.py:937-949 compute_ffn_layernorm, :976-999 compute_bias_residual_layernorm).
//   r = bf16(x + residual) ; out = bf16( bf16(r * rstd) * w )   — same rounding points as the training path.
// ------------------------------------------------------------------------------------------------
// x_f32 != nullptr: x is the fp32 split-K accumulation of the producing GEMM; it is rounded to bf16 here (the Linear
// output rounding) and the workspace is handed back zeroed — this fuses the split-K "finish" pass into the norm.
// WPR = warps per row: 1 -> four rows per CTA (many rows, prefill); 4 -> one row per CTA (the 64-row decode step, where one
// warp per row leaves the op latency-bound on 16 SMs).
template <int MAXV, int WPR>
__global__ void __launch_bounds__(128) add_rmsnorm_kernel(const bf16* __restrict__ x, float* __restrict__ x_f32,
                                                          const bf16* __restrict__ res,
                                                          const bf16* __restrict__ w, bf16* __restrict__ normed,
                                                          bf16* __restrict__ res_out, int rows, int h, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int TPR = 32 * WPR;                     // threads per row
  __shared__ float s_part[4];
  const int warp = threadIdx.x >> 5;
  const int lane = (WPR == 1) ? (threadIdx.x & 31) : static_cast<int>(threadIdx.x);   // position within the row
  const int row = (WPR == 1) ? blockIdx.x * 4 + warp : static_cast<int>(blockIdx.x);
  if (row >= rows) return;
  const int nchunk = h >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * h);
  float4* xf = x_f32 ? reinterpret_cast<float4*>(x_f32 + static_cast<size_t>(row) * h) : nullptr;
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + static_cast<size_t>(row) * h) : nullptr;
  // Phase 1: issue every load of the row before anything else (branch-free: out-of-range chunks re-read the last valid
  // chunk and are masked later), so the whole row is one memory round trip instead of one per chunk.
  uint4 v[MAXV], rv[MAXV];
  float4 fa[MAXV], fb[MAXV];
  const int last = nchunk - 1;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = min(lane + TPR * i, last);
    if (xf) { fa[i] = xf[2 * c]; fb[i] = xf[2 * c + 1]; }
    else v[i] = ld_nc_v4(xr + c);
    if (rr) rv[i] = ld_nc_v4(rr + c);
  }
  // (one row per CTA: also fetch the norm weight now, so that the row costs one memory round trip, not two)
  uint4 wv_pre[WPR > 1 ? MAXV : 1];
  if constexpr (WPR > 1) {
    if (normed != nullptr) {
#pragma unroll
      for (int i = 0; i < MAXV; ++i) wv_pre[i] = __ldg(reinterpret_cast<const uint4*>(w) + min(lane + TPR * i, last));
    }
  }
  // Phase 2: round the fp32 input (if any), add the residual, accumulate the sum of squares
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const bool ok = (lane + TPR * i) < nchunk;
    if (xf) v[i] = make_uint4(pack_bf16x2(fa[i].x, fa[i].y), pack_bf16x2(fa[i].z, fa[i].w), pack_bf16x2(fb[i].x, fb[i].y),
                              pack_bf16x2(fb[i].z, fb[i].w));
    uint32_t* vi = reinterpret_cast<uint32_t*>(&v[i]);
    if (rr) {
      const uint32_t* ri = reinterpret_cast<const uint32_t*>(&rv[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = unpack_bf16x2(vi[j]), b = unpack_bf16x2(ri[j]);
        vi[j] = pack_bf16x2(a.x + b.x, a.y + b.y);
      }
    }
    float part = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 a = unpack_bf16x2(vi[j]); part += a.x * a.x + a.y * a.y; }
    ss += ok ? part : 0.f;
  }
  // Phase 3: hand the fp32 workspace back zeroed, write the new residual
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = lane + TPR * i;
    if (c < nchunk) {
      if (xf) { xf[2 * c] = make_float4(0.f, 0.f, 0.f, 0.f); xf[2 * c + 1] = make_float4(0.f, 0.f, 0.f, 0.f); }
      if (res_out) st_na_v4(reinterpret_cast<uint4*>(res_out + static_cast<size_t>(row) * h) + c, v[i]);
    }
  }
  ss = warp_sum(ss);
  if constexpr (WPR > 1) {
    if ((threadIdx.x & 31) == 0) s_part[warp] = ss;
    __syncthreads();
    ss = s_part[0] + s_part[1] + s_part[2] + s_part[3];
  }
  const float rstd = rsqrtf(ss / static_cast<float>(h) + eps);
  if (normed == nullptr) return;
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(normed + static_cast<size_t>(row) * h);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = lane + TPR * i;
    if (c < nchunk) {
      uint4 wv;
      if constexpr (WPR > 1) wv = wv_pre[i]; else wv = __ldg(wr + c);
      uint4 o;
      const uint32_t* xi = reinterpret_cast<const uint32_t*>(&v[i]);
      const uint32_t* wi = reinterpret_cast<const uint32_t*>(&wv);
      uint32_t* oi = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(xi[j]), wf = unpack_bf16x2(wi[j]);
        oi[j] = pack_bf16x2(bf16_round(xf.x * rstd) * wf.x, bf16_round(xf.y * rstd) * wf.y);
      }
      st_na_v4(yr + c, o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Prefill: copy the (already rotated) K and the V rows of the packed QKV projection into the dense or paged cache
// (kv_cache.cuh; reference: write_cache_kv, csrc/gpu/write_cache_kv.cu:23-99; here K keeps the plain [max_len, d] row
// layout — the transposed x=8 layout there is private to Paddle's MMHA kernel).  Every cache writer stores through
// KvCacheT::store8, which quantises the same bf16 values into a uint8 cache.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void write_cache_kv_kernel(const bf16* __restrict__ qkv, const KvCacheT<T> cv, const int* __restrict__ seq_lens,
                                      int S, int nh, int64_t ld) {
  const int tok = blockIdx.x;          // b * S + s
  const int b = tok / S, s = tok % S;
  const int kvh = cv.kvh, d = cv.d;
  if (seq_lens != nullptr && s >= seq_lens[b]) return;
  if (s >= cv.max_len) return;
  const int chunks = (kvh * d) >> 3;   // 16-byte chunks per K (or V) row group
  for (int c = threadIdx.x; c < 2 * chunks; c += blockDim.x) {
    const int which = c / chunks;      // 0: K, 1: V
    const int cc = c % chunks;
    const int head = (cc * 8) / d, off = (cc * 8) % d;
    const uint4 v = *reinterpret_cast<const uint4*>(qkv + static_cast<size_t>(tok) * ld + (nh + which * kvh) * d + cc * 8);
    cv.store8(which, head, cv.offset(b, head, s) + off, v);
  }
}

// ------------------------------------------------------------------------------------------------
// Decode: RoPE (rotate-half, fp32 math, one rounding) on the new token's q and k at position seq_lens[b], in place in
// the packed [B, ld] projection, and append k, v to the cache at that position.
// Reference: masked_multihead_attention(x=qkv, cache_kv, sequence_lengths, rotary_tensor, rotary_emb_dims=1,
// use_neox_rotary_style=True) — neox == rotate-half in csrc (encode_rotary_qk.cu:18-56);
// fused variant: append_attn/decoder_write_cache_with_rope_kernel.cu:47-390.
// ------------------------------------------------------------------------------------------------
// acc_f32 != nullptr: the packed projection arrives as the fp32 split-K accumulation (+ optional fp32 bias); it is rounded
// to bf16 here (the Linear output rounding), written to qkv, and the workspace is handed back zeroed.
__device__ __forceinline__ uint4 take_f32_chunk(float* acc, const float* bias, int col) {
  float4* p = reinterpret_cast<float4*>(acc + col);
  float4 a = p[0], b = p[1];
  p[0] = make_float4(0.f, 0.f, 0.f, 0.f);
  p[1] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias != nullptr) {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + col)), b1 = __ldg(reinterpret_cast<const float4*>(bias + col) + 1);
    a.x += b0.x; a.y += b0.y; a.z += b0.z; a.w += b0.w; b.x += b1.x; b.y += b1.y; b.z += b1.z; b.w += b1.w;
  }
  return make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
}

template <typename T>
__global__ void decode_rope_append_kernel(bf16* __restrict__ qkv, float* __restrict__ acc_f32, const float* __restrict__ bias,
                                          const KvCacheT<T> cv, const float* __restrict__ cos_t,
                                          const float* __restrict__ sin_t, const int* __restrict__ seq_lens, int nh,
                                          int64_t ld) {
  // ONE pass, no block barrier: thread = one (head, 8-column chunk pair) of q / k, or one 8-column chunk of v.  Each thread takes
  // its inputs from the fp32 split-K accumulation (rounded to bf16 first: the Linear output rounding) or from the bf16 projection,
  // rotates in registers and writes the projection row and the cache once.  (The first version materialised the bf16 row, hit a
  // __syncthreads and read it back: two dependent global round trips per launch — 11.6 us for 64 rows in the decode chain.)
  const int kvh = cv.kvh, d = cv.d, max_len = cv.max_len;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const int pos = seq_lens[b];
  const bool pos_ok = pos >= 0 && pos < max_len;
  const int half = d >> 1;
  const int per_head = half >> 3;
  const int n_rope = (nh + kvh) * per_head;
  const int idx = threadIdx.x;
  bf16* row = qkv + static_cast<size_t>(b) * ld;
  float* arow = acc_f32 ? acc_f32 + static_cast<size_t>(b) * (nh + 2 * kvh) * d : nullptr;
  if (idx < n_rope) {
    const int head = idx / per_head;
    const int j8 = (idx % per_head) * 8;
    bf16* base = row + head * d;
    uint4 a, bb;
    if (arow != nullptr) {
      a = take_f32_chunk(arow, bias, head * d + j8);
      bb = take_f32_chunk(arow, bias, head * d + half + j8);
    } else {
      if (!pos_ok) return;
      a = *reinterpret_cast<const uint4*>(base + j8);
      bb = *reinterpret_cast<const uint4*>(base + half + j8);
    }
    if (pos_ok) rope_rotate_chunk(a, bb, cos_t, sin_t, pos, half, j8);
    *reinterpret_cast<uint4*>(base + j8) = a;
    *reinterpret_cast<uint4*>(base + half + j8) = bb;
    if (pos_ok && head >= nh) {   // rotated k -> cache
      const size_t dst = cv.offset(b, head - nh, pos);
      cv.store8(0, head - nh, dst + j8, a);
      cv.store8(0, head - nh, dst + half + j8, bb);
    }
  } else {
    // v -> projection row (fp32 path) and cache (16-byte chunks)
    const int c = idx - n_rope;
    if (c >= (kvh * d) >> 3) return;
    const int col = (nh + kvh) * d + c * 8;
    uint4 v;
    if (arow != nullptr) {
      v = take_f32_chunk(arow, bias, col);
      *reinterpret_cast<uint4*>(row + col) = v;
    } else {
      if (!pos_ok) return;
      v = *reinterpret_cast<const uint4*>(row + col);
    }
    if (pos_ok) {
      const int head = (c * 8) / d, off = (c * 8) % d;
      cv.store8(1, head, cv.offset(b, head, pos) + off, v);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Bookkeeping ops (integer work; semantics follow the cited kernels line by line)
// ------------------------------------------------------------------------------------------------
// get_padding_offset_v2 (csrc/gpu/get_padding_offset_v2.cu:17-53)
__global__ void padding_offset_kernel(const int64_t* __restrict__ input_ids, const int* __restrict__ cum_offsets,
                                      const int* __restrict__ seq_lens, int64_t* __restrict__ x_remove_padding,
                                      int* __restrict__ padding_offset, int* __restrict__ cum_offsets_out,
                                      int* __restrict__ cu_seqlens_q, int* __restrict__ cu_seqlens_k, int max_seq_len) {
  const int bi = blockIdx.x, ti = threadIdx.x;
  const int cum_offset = bi == 0 ? 0 : cum_offsets[bi - 1];
  for (int i = ti; i < seq_lens[bi]; i += blockDim.x) {
    padding_offset[bi * max_seq_len - cum_offset + i] = cum_offset;
    x_remove_padding[bi * max_seq_len - cum_offset + i] = input_ids[bi * max_seq_len + i];   // RemovePaddingV2 (:80-85)
  }
  if (ti == 0) {
    cum_offsets_out[bi] = cum_offset;
    const int cum_seq_len = (bi + 1) * max_seq_len - cum_offsets[bi];
    cu_seqlens_q[bi + 1] = cum_seq_len;
    cu_seqlens_k[bi + 1] = cum_seq_len;
    if (bi == 0) { cu_seqlens_q[0] = 0; cu_seqlens_k[0] = 0; }
  }
}

// rebuild_padding_v2 (csrc/gpu/rebuild_padding_v2.cu:18-69): one output row per sequence = its last valid token
// (prefill: token seq_len_encoder-1 of the sequence; decode: its single token).
__global__ void rebuild_padding_kernel(const bf16* __restrict__ tmp_out, const int* __restrict__ cum_offsets,
                                       const int* __restrict__ seq_lens_decoder, const int* __restrict__ seq_lens_encoder,
                                       bf16* __restrict__ out, int max_len, int dim) {
  const int bi = blockIdx.x;
  int seq_id = 0;
  if (seq_lens_decoder[bi] == 0 && seq_lens_encoder[bi] == 0) return;
  if (seq_lens_decoder[bi] == 0) seq_id = seq_lens_encoder[bi] - 1;
  const int ori_token_idx = bi * max_len - cum_offsets[bi] + seq_id;
  for (int i = threadIdx.x; i < dim; i += blockDim.x)
    out[static_cast<size_t>(bi) * dim + i] = tmp_out[static_cast<size_t>(ori_token_idx) * dim + i];
}

// set_value_by_flags_and_idx (v1: csrc/gpu/set_value_by_flags.cu:17-25; v2: set_value_by_flags_v2.cu)
__global__ void set_value_by_flags_kernel(const bool* __restrict__ stop_flags, int64_t* __restrict__ pre_ids_all,
                                          const int64_t* __restrict__ pre_ids, const int64_t* __restrict__ step_idx, int bs,
                                          int length) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < bs && !stop_flags[tid]) {
    if (step_idx[tid] >= 0) pre_ids_all[static_cast<size_t>(tid) * length + step_idx[tid]] = pre_ids[tid];
  }
}
__global__ void set_value_by_flags_v2_kernel(const bool* __restrict__ stop_flags, int64_t* __restrict__ pre_ids_all,
                                             const int64_t* __restrict__ input_ids, const int* __restrict__ seq_lens_encoder,
                                             const int* __restrict__ seq_lens_decoder, const int64_t* __restrict__ step_idx,
                                             int bs, int length, int length_input_ids) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < bs && !stop_flags[tid]) {
    int64_t* pre = pre_ids_all + static_cast<size_t>(tid) * length;
    const int64_t* ids = input_ids + static_cast<size_t>(tid) * length_input_ids;
    const int dec = seq_lens_decoder[tid], enc = seq_lens_encoder[tid];
    if (dec == 0 && enc == 0) return;
    if (step_idx[tid] >= 0) pre[step_idx[tid]] = (dec == 0) ? ids[enc - 1] : ids[0];
  }
}

// get_token_penalty_multi_scores(_v2) (csrc/gpu/token_penalty_multi_scores_v2.cu:19-139; CPU twin
// csrc/cpu/src/token_penalty_multi_scores.cc:18-85).  One CTA per sequence; repeat counts in a caller workspace.
// Precondition: each row of pre_ids is its history as a prefix of ids >= 0 followed only by -1 padding.  The count stops at
// the first negative entry, so a row whose entry 0 is -1 has an empty history whatever follows it (the callers write the
// last prompt token into entry 0 before the first token is chosen).
__global__ void penalty_count_kernel(const int64_t* __restrict__ pre_ids, const int64_t* __restrict__ cur_len,
                                     int* __restrict__ repeat_times, int64_t length, int64_t length_id) {
  const int bi = blockIdx.x;
  if (cur_len[bi] < 0) return;
  const int64_t* ids = pre_ids + static_cast<size_t>(bi) * length_id;
  int* rt = repeat_times + static_cast<size_t>(bi) * length;
  // the reference breaks at the first negative id PER THREAD stride; under the precondition above, scanning until the
  // first negative entry is equivalent.
  for (int64_t i = threadIdx.x; i < length_id; i += blockDim.x) {
    const int64_t id = ids[i];
    if (id < 0) break;
    if (id < length) atomicAdd(&rt[id], 1);
  }
}
__global__ void penalty_apply_kernel(float* __restrict__ logits, const int* __restrict__ repeat_times,
                                     const float* __restrict__ penalty, const float* __restrict__ frequency,
                                     const float* __restrict__ presence, const float* __restrict__ temperatures,
                                     const int64_t* __restrict__ cur_len, const int64_t* __restrict__ min_len,
                                     const int64_t* __restrict__ eos_ids, int64_t eos_len,
                                     const int64_t* __restrict__ bad_tokens, int64_t bad_len, int64_t length) {
  const int bi = blockIdx.x;
  float* lg = logits + static_cast<size_t>(bi) * length;
  const int* rt = repeat_times + static_cast<size_t>(bi) * length;
  const bool min_len_mask = cur_len[bi] >= 0 && cur_len[bi] < min_len[bi];
  const float alpha = penalty[bi], beta = frequency[bi], gamma = presence[bi];
  const float temp = temperatures ? temperatures[bi] : 1.f;
  for (int64_t i = threadIdx.x; i < length; i += blockDim.x) {
    float v = lg[i];
    if (min_len_mask) {
      for (int64_t e = 0; e < eos_len; ++e)
        if (eos_ids[e] == i) v = -1e10f;
    }
    const int times = rt[i];
    if (times != 0) {
      v = v < 0 ? v * alpha : v / alpha;
      v = v - times * beta - gamma;
    }
    v = v / temp;
    for (int64_t k = 0; k < bad_len; ++k)
      if (bad_tokens[k] == i) v = -1e10f;
    lg[i] = v;
  }
}

// set_stop_value_multi_ends: v1 mode 2 (csrc/gpu/stop_generation_multi_ends.cu:45-56), v2 (…_v2.cu:35-59)
__device__ __forceinline__ bool in_end(int64_t id, const int64_t* end_ids, int n) {
  for (int i = 0; i < n; ++i)
    if (id == end_ids[i]) return true;
  return false;
}
__global__ void stop_value_kernel(bool* __restrict__ stop_flags, int64_t* __restrict__ topk_ids,
                                  int64_t* __restrict__ next_tokens, const int64_t* __restrict__ end_ids,
                                  const int* __restrict__ seq_lens, int bs, int end_length, int v2) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= bs) return;
  if (v2) {
    if (stop_flags[tid]) {
      if (seq_lens[tid] == 0) topk_ids[tid] = -1;
      else { topk_ids[tid] = end_ids[0]; next_tokens[tid] = end_ids[0]; }
    } else {
      next_tokens[tid] = topk_ids[tid];
    }
  } else {
    topk_ids[tid] = stop_flags[tid] ? end_ids[0] : topk_ids[tid];
  }
  if (in_end(topk_ids[tid], end_ids, end_length)) stop_flags[tid] = true;
}

// update_inputs (csrc/gpu/update_inputs.cu:18-66), single CTA of 1024 threads
__global__ void update_inputs_kernel(bool* not_need_stop, int* seq_lens_this_time, int* seq_lens_encoder,
                                     int* seq_lens_decoder, int64_t* input_ids, const int64_t* stop_nums,
                                     const bool* stop_flags, const bool* is_block_step, const int64_t* next_tokens, int bsz,
                                     int max_bsz, int input_ids_stride) {
  __shared__ int red[32];
  const int t = threadIdx.x;
  bool stop_now = false;
  int stop_int = 0;
  if (t < max_bsz) {
    if (t < bsz) {
      stop_now = stop_flags[t];
      stop_int = is_block_step[t] ? 0 : static_cast<int>(stop_now);
    } else {
      stop_int = 1;
    }
  }
  if (t < bsz) {
    const int enc = seq_lens_encoder[t], dec = seq_lens_decoder[t];
    seq_lens_decoder[t] = stop_now ? 0 : (dec == 0 ? enc : dec + 1);
    seq_lens_this_time[t] = stop_now ? 0 : 1;
    seq_lens_encoder[t] = 0;
    input_ids[static_cast<size_t>(t) * input_ids_stride] = next_tokens[t];
  }
  int s = stop_int;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((t & 31) == 0) red[t >> 5] = s;
  __syncthreads();
  if (t < 32) {
    s = red[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (t == 0) not_need_stop[0] = static_cast<int64_t>(s) < stop_nums[0];
  }
}

// One fused per-step state update for the dense-cache generate loop
// (GenerationInferenceModel.update_model_kwargs_for_generation, experimental/transformers/generation_utils.py:185-260).
// `was` is the stop flag on entry:
//   step_idx += !was ; next = was ? eos[0] : next ; stop = was || step_idx >= max_dec_len || next in eos ;
//   if !was: pre_ids[b, step_idx] = next (set_value_by_flags_and_idx of the following step) ; seq_len_decoder += !stop ;
//   tgt_ids = next ; out_tokens[b, col] = next ; stop_count = sum(stop)
// Only a row stopped before this call emits eos[0].  A row whose step reaches max_dec_len here keeps (and records) the token it
// chose: the last generated token is a real one, as in oracle/generation_ref.greedy_generate.  This differs on purpose from
// the reference, which sets the max_dec_len flag first (generation_utils.py:185-205) and then substitutes eos for every flagged
// row (stop_generation_multi_ends.cu:48).
__global__ void generate_step_update_kernel(int64_t* next_tokens, bool* stop_flags, int64_t* step_idx,
                                            const int64_t* max_dec_len, int* seq_len_decoder, int64_t* pre_ids,
                                            int64_t pre_len, const int64_t* eos_ids, int eos_len, int64_t* out_tokens,
                                            int64_t out_stride, int64_t out_col, const int64_t* out_col_dev,
                                            int* stop_count, int bs) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (out_col_dev != nullptr) out_col = out_col_dev[0];
  if (b < bs) {
    bool stop = stop_flags[b];
    int64_t step = step_idx[b];
    if (!stop) step += 1;
    if (step >= max_dec_len[b]) stop = true;
    int64_t tok = stop_flags[b] ? eos_ids[0] : next_tokens[b];
    if (in_end(tok, eos_ids, eos_len)) stop = true;
    if (!stop_flags[b] && step >= 0 && step < pre_len) pre_ids[static_cast<size_t>(b) * pre_len + step] = tok;
    if (!stop) seq_len_decoder[b] += 1;
    next_tokens[b] = tok;
    step_idx[b] = step;
    stop_flags[b] = stop;
    if (out_tokens != nullptr && out_col >= 0 && out_col < out_stride)
      out_tokens[static_cast<size_t>(b) * out_stride + out_col] = tok;
    if (stop) atomicAdd(stop_count, 1);
  }
}

__global__ void increment_i64_kernel(int64_t* p) { p[0] += 1; }

__global__ void argmax_f32_kernel(const float* __restrict__ logits, int64_t* __restrict__ out, int vocab, int64_t ld) {
  __shared__ float sv[8];
  __shared__ int si[8];
  const float* lr = logits + static_cast<size_t>(blockIdx.x) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < vocab; i += blockDim.x) {
    const float f = lr[i];
    if (f > best || (f == best && i < bi)) { best = f; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (blockDim.x >> 5); ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
    out[blockIdx.x] = bi;
  }
}

__global__ void bf16_rows_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, int64_t rows, int64_t cols,
                                        int64_t ld) {
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = __bfloat162float(src[(i / cols) * ld + (i % cols)]);
}

// ------------------------------------------------------------------------------------------------
// Sampling: softmax over fp32 logits and rejection top-p sampling.
// Reference: `probs = F.softmax(logits)` then top_p_sampling_reject(probs, top_p, seed)
// (experimental/transformers/generation_utils.py:326-336; csrc/gpu/sample_kernels/top_p_sampling_reject.cu:18-60,
//  kernel sample_kernels/sampling.cuh:286-376, inverse-CDF step :197-280).  The uniform draws are an INPUT here (the
// reference draws [32, bs] of them from Paddle's generator), so the op is a deterministic function of its arguments.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce_1024(float v, float* s_w, bool is_max) {
  // all 1024 threads call; s_w has 32 floats; result broadcast to every thread
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  __syncthreads();                       // s_w free from the previous use
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = s_w[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, r, o);
    r = is_max ? fmaxf(r, t) : r + t;
  }
  return r;
}

// in place: logits[row, :] -> softmax probabilities (fp32)
__global__ void __launch_bounds__(1024) softmax_f32_kernel(float* __restrict__ x, int vocab, int64_t ld) {
  __shared__ float s_w[32];
  float* row = x + static_cast<size_t>(blockIdx.x) * ld;
  const int n4 = vocab >> 2;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n4; i += 1024) {
    const float4 v = reinterpret_cast<const float4*>(row)[i];
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  m = block_reduce_1024(m, s_w, true);
  float sum = 0.f;
  for (int i = threadIdx.x; i < n4; i += 1024) {
    const float4 v = reinterpret_cast<const float4*>(row)[i];
    sum += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
  }
  sum = block_reduce_1024(sum, s_w, false);
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < n4; i += 1024) {
    float4 v = reinterpret_cast<float4*>(row)[i];
    v.x = expf(v.x - m) * inv; v.y = expf(v.y - m) * inv; v.z = expf(v.z - m) * inv; v.w = expf(v.w - m) * inv;
    reinterpret_cast<float4*>(row)[i] = v;
  }
}

// One CTA (1024 threads) per row.  Round r: u = uniform[r, b] * q; sampled = first index whose inclusive CDF over
// {p_j > pivot} exceeds u; pivot = max(pivot, p[sampled]); (q, count) = mass / number of {p_j > pivot};
// stop when 0 < q < top_p, or when count == 0 (covers top_p == 0 -> arg max).
// When no CDF value exceeds u (the row's fp32 total is at most u: a softmax row sums to 1 only within rounding, and u can be
// as large as 1 - 2^-24), sampled is the largest index with p > pivot, the last token the CDF reaches.  The reference falls
// back to vocab - 1 (sampling.cuh:313), which can emit a token of probability zero (e.g. an EOS banned by min_length).
__global__ void __launch_bounds__(1024) top_p_sampling_reject_kernel(const float* __restrict__ probs, const float* __restrict__ top_p,
                                                                     const float* __restrict__ uniform, int64_t* __restrict__ out,
                                                                     int vocab, int64_t ld, int bs, int max_rounds) {
  __shared__ float s_w[32];
  __shared__ int s_sampled;
  __shared__ int s_cnt[32];
  const int b = blockIdx.x, tx = threadIdx.x, lane = tx & 31, warp = tx >> 5;
  const float* row = probs + static_cast<size_t>(b) * ld;
  const float tp = top_p[b];
  const int n4 = vocab >> 2;
  const int iters = (n4 + 1023) / 1024;
  float q = 1.f, pivot = 0.f;
  int sampled = vocab - 1;
  for (int round = 0; round < max_rounds; ++round) {
    if (tx == 0) s_sampled = vocab;                  // "no index found"
    const float u = uniform[static_cast<size_t>(round) * bs + b] * q;
    float aggregate = 0.f;
    for (int it = 0; it < iters; ++it) {
      const int i4 = it * 1024 + tx;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i4 < n4) v = reinterpret_cast<const float4*>(row)[i4];
      const float f0 = v.x > pivot ? v.x : 0.f, f1 = v.y > pivot ? v.y : 0.f, f2 = v.z > pivot ? v.z : 0.f,
                  f3 = v.w > pivot ? v.w : 0.f;
      const float c0 = f0, c1 = c0 + f1, c2 = c1 + f2, c3 = c2 + f3;     // thread-local inclusive sums
      // block-wide exclusive prefix of the thread totals
      float incl = c3;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      __syncthreads();                               // s_w / s_sampled settled from the previous iteration
      if (lane == 31) s_w[warp] = incl;
      __syncthreads();
      float wsum = s_w[lane];
      float wincl = wsum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, wincl, o);
        if (lane >= o) wincl += t;
      }
      const float total = __shfl_sync(0xffffffffu, wincl, 31);
      const float warp_excl = __shfl_sync(0xffffffffu, wincl - wsum, warp);
      const float base = aggregate + warp_excl + (incl - c3);              // mass strictly before this thread's 4 elements
      if (aggregate + total > u) {
        // first (lowest-index) valid element whose inclusive CDF exceeds u; the block scan is only monotone up to fp32
        // rounding, so every candidate thread votes and the minimum wins (sampling.cuh:267-270)
        if (base + c3 > u) {
          int j = -1;
          if (base + c0 > u && f0 > 0.f) j = 0;
          else if (base + c1 > u && f1 > 0.f) j = 1;
          else if (base + c2 > u && f2 > 0.f) j = 2;
          else if (f3 > 0.f) j = 3;
          if (j >= 0) atomicMin(&s_sampled, i4 * 4 + j);
        }
        aggregate += total;
        break;
      }
      aggregate += total;
    }
    __syncthreads();
    sampled = s_sampled;
    if (sampled == vocab) {                          // block-uniform: every thread read the same s_sampled
      int last = -1;                                 // this thread's largest index with p > pivot (its i4 only grow)
      for (int i4 = tx; i4 < n4; i4 += 1024) {
        const float4 v = reinterpret_cast<const float4*>(row)[i4];
        if (v.w > pivot) last = i4 * 4 + 3;
        else if (v.z > pivot) last = i4 * 4 + 2;
        else if (v.y > pivot) last = i4 * 4 + 1;
        else if (v.x > pivot) last = i4 * 4;
      }
      last = __reduce_max_sync(0xffffffffu, last);
      if (lane == 0) s_cnt[warp] = last;
      __syncthreads();
      last = __reduce_max_sync(0xffffffffu, s_cnt[lane]);
      sampled = last >= 0 ? last : vocab - 1;        // nothing above the pivot: only a row without positive mass
    }
    pivot = fmaxf(pivot, row[sampled]);
    float mass = 0.f;
    int cnt = 0;
    for (int i4 = tx; i4 < n4; i4 += 1024) {
      const float4 v = reinterpret_cast<const float4*>(row)[i4];
      if (v.x > pivot) { mass += v.x; ++cnt; }
      if (v.y > pivot) { mass += v.y; ++cnt; }
      if (v.z > pivot) { mass += v.z; ++cnt; }
      if (v.w > pivot) { mass += v.w; ++cnt; }
    }
    q = block_reduce_1024(mass, s_w, false);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_cnt[warp] = cnt;
    __syncthreads();
    int total_cnt = s_cnt[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total_cnt += __shfl_xor_sync(0xffffffffu, total_cnt, o);
    if (q > 0.f && q < tp) break;
    if (total_cnt < 1) break;
  }
  if (tx == 0) out[b] = sampled;
}

}  // namespace gen
}  // namespace b200

using namespace b200;
using namespace b200::gen;

static int add_rmsnorm_launch(const void* x, float* x_f32, const void* residual, const void* w, void* normed,
                              void* residual_out, int64_t rows, int64_t h, float eps, cudaStream_t stream);
template <typename T>
static int rope_append_launch(void* qkv, float* acc_f32_ws, const float* bias, const KvCacheT<T>& cv, const float* cos_table,
                              const float* sin_table, const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t ld,
                              cudaStream_t stream);

extern "C" int b200_add_rmsnorm(const void* x, const void* residual, const void* w, void* normed, void* residual_out,
                                int64_t rows, int64_t h, float eps, cudaStream_t stream) {
  B200_CHECK_ARG(x, "add_rmsnorm: null pointer");
  return add_rmsnorm_launch(x, nullptr, residual, w, normed, residual_out, rows, h, eps, stream);
}

extern "C" int b200_add_rmsnorm_f32(float* x_f32_ws, const void* residual, const void* w, void* normed, void* residual_out,
                                    int64_t rows, int64_t h, float eps, cudaStream_t stream) {
  B200_CHECK_ARG(x_f32_ws, "add_rmsnorm_f32: null pointer");
  return add_rmsnorm_launch(nullptr, x_f32_ws, residual, w, normed, residual_out, rows, h, eps, stream);
}

static int add_rmsnorm_launch(const void* x, float* x_f32, const void* residual, const void* w, void* normed,
                              void* residual_out, int64_t rows, int64_t h, float eps, cudaStream_t stream) {
  B200_CHECK_ARG((w || !normed), "add_rmsnorm: null pointer");
  B200_CHECK_ARG(rows > 0 && h > 0 && h % 8 == 0 && h <= 8192, "add_rmsnorm: need 0 < h <= 8192, h %% 8 == 0");
  const int nchunk = static_cast<int>(h / 8);
  const dim3 block(128);
  const bf16 *xp = static_cast<const bf16*>(x), *rp = static_cast<const bf16*>(residual), *wp = static_cast<const bf16*>(w);
  bf16 *np = static_cast<bf16*>(normed), *ro = static_cast<bf16*>(residual_out);
  if (rows <= 1024) {            // few rows (decode step): one CTA per row
    const dim3 grid(static_cast<unsigned>(rows));
    if (nchunk <= 256) launch_pdl(add_rmsnorm_kernel<2, 4>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
    else if (nchunk <= 512) launch_pdl(add_rmsnorm_kernel<4, 4>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
    else launch_pdl(add_rmsnorm_kernel<8, 4>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
  } else {
    const dim3 grid(static_cast<unsigned>((rows + 3) / 4));
    if (nchunk <= 128) launch_pdl(add_rmsnorm_kernel<4, 1>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
    else if (nchunk <= 512) launch_pdl(add_rmsnorm_kernel<16, 1>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
    else launch_pdl(add_rmsnorm_kernel<32, 1>, grid, block, 0, stream, xp, x_f32, rp, wp, np, ro, (int)rows, (int)h, eps);
  }
  return check_launch("add_rmsnorm");
}

extern "C" int b200_write_cache_kv(const void* qkv, void* cache, const int32_t* seq_lens, int64_t B, int64_t S,
                                   int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len, int64_t ld,
                                   cudaStream_t stream) {
  KvCache cv;
  if (int rc = dense_kv_cache(&cv, cache, B, num_kv_heads, head_dim, max_len, "write_cache_kv")) return rc;
  B200_CHECK_ARG(qkv && ld % 8 == 0 && S > 0 && S <= max_len, "write_cache_kv: bad sizes");
  write_cache_kv_kernel<<<static_cast<unsigned>(B * S), 128, 0, stream>>>(static_cast<const bf16*>(qkv), cv, seq_lens, (int)S,
                                                                          (int)num_heads, ld);
  return check_launch("write_cache_kv");
}

extern "C" int b200_write_cache_kv_paged(const void* qkv, void* key_cache, void* value_cache, const int32_t* block_tables,
                                         const int32_t* seq_lens, int64_t B, int64_t S, int64_t num_heads,
                                         int64_t num_kv_heads, int64_t head_dim, int64_t block_size,
                                         int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream) {
  KvCache cv;
  if (int rc = paged_kv_cache(&cv, key_cache, value_cache, block_tables, num_kv_heads, head_dim, block_size, max_blocks_per_seq,
                              "write_cache_kv_paged"))
    return rc;
  B200_CHECK_ARG(qkv && ld % 8 == 0 && B > 0 && S > 0 && S <= cv.max_len, "write_cache_kv_paged: bad sizes");
  write_cache_kv_kernel<<<static_cast<unsigned>(B * S), 128, 0, stream>>>(static_cast<const bf16*>(qkv), cv, seq_lens, (int)S,
                                                                          (int)num_heads, ld);
  return check_launch("write_cache_kv_paged");
}

extern "C" int b200_write_cache_kv_paged_c8(const void* qkv, void* key_cache, void* value_cache, const int32_t* block_tables,
                                            const void* cache_k_scale, const void* cache_v_scale, const int32_t* seq_lens,
                                            int64_t B, int64_t S, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                            int64_t block_size, int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream) {
  KvCacheC8 cv;
  if (int rc = paged_kv_cache_c8(&cv, key_cache, value_cache, block_tables, cache_k_scale, cache_v_scale, nullptr, nullptr, true,
                                 false, num_kv_heads, head_dim, block_size, max_blocks_per_seq, "write_cache_kv_paged_c8"))
    return rc;
  B200_CHECK_ARG(qkv && ld % 8 == 0 && B > 0 && S > 0 && S <= cv.max_len, "write_cache_kv_paged_c8: bad sizes");
  write_cache_kv_kernel<<<static_cast<unsigned>(B * S), 128, 0, stream>>>(static_cast<const bf16*>(qkv), cv, seq_lens, (int)S,
                                                                          (int)num_heads, ld);
  return check_launch("write_cache_kv_paged_c8");
}

extern "C" int b200_decode_rope_append_f32(void* qkv, float* acc_f32_ws, const float* bias, void* cache,
                                           const float* cos_table, const float* sin_table, const int32_t* seq_lens,
                                           int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                           int64_t max_len, int64_t ld, cudaStream_t stream);

extern "C" int b200_decode_rope_append(void* qkv, void* cache, const float* cos_table, const float* sin_table,
                                       const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t num_kv_heads,
                                       int64_t head_dim, int64_t max_len, int64_t ld, cudaStream_t stream) {
  return b200_decode_rope_append_f32(qkv, nullptr, nullptr, cache, cos_table, sin_table, seq_lens, B, num_heads,
                                     num_kv_heads, head_dim, max_len, ld, stream);
}

extern "C" int b200_decode_rope_append_f32(void* qkv, float* acc_f32_ws, const float* bias, void* cache,
                                           const float* cos_table, const float* sin_table, const int32_t* seq_lens,
                                           int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                           int64_t max_len, int64_t ld, cudaStream_t stream) {
  KvCache cv;
  if (int rc = dense_kv_cache(&cv, cache, B, num_kv_heads, head_dim, max_len, "decode_rope_append")) return rc;
  B200_CHECK_ARG(qkv && cos_table && sin_table && seq_lens, "decode_rope_append: null pointer");
  return rope_append_launch(qkv, acc_f32_ws, bias, cv, cos_table, sin_table, seq_lens, B, num_heads, ld, stream);
}

template <typename T>
static int rope_append_launch(void* qkv, float* acc_f32_ws, const float* bias, const KvCacheT<T>& cv, const float* cos_table,
                              const float* sin_table, const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t ld,
                              cudaStream_t stream) {
  B200_CHECK_ARG(cv.d % 16 == 0 && ld % 8 == 0, "decode_rope_append: head_dim %% 16, ld %% 8");
  const int threads_needed = static_cast<int>((num_heads + cv.kvh) * (cv.d / 16) + (cv.kvh * cv.d) / 8);   // rope pairs + v chunks
  B200_CHECK_ARG(threads_needed <= 1024, "decode_rope_append: too many heads");
  const int threads = (threads_needed + 31) / 32 * 32;
  launch_pdl(decode_rope_append_kernel<T>, dim3(static_cast<unsigned>(B)), dim3(threads), 0, stream, static_cast<bf16*>(qkv),
             acc_f32_ws, bias, cv, cos_table, sin_table, seq_lens, (int)num_heads, ld);
  return check_launch("decode_rope_append");
}

extern "C" int b200_decode_rope_append_paged(void* qkv, float* acc_f32_ws, const float* bias, void* key_cache, void* value_cache,
                                             const int32_t* block_tables, const float* cos_table, const float* sin_table,
                                             const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t num_kv_heads,
                                             int64_t head_dim, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                             cudaStream_t stream) {
  KvCache cv;
  if (int rc = paged_kv_cache(&cv, key_cache, value_cache, block_tables, num_kv_heads, head_dim, block_size, max_blocks_per_seq,
                              "decode_rope_append_paged"))
    return rc;
  B200_CHECK_ARG(qkv && cos_table && sin_table && seq_lens, "decode_rope_append_paged: null pointer");
  return rope_append_launch(qkv, acc_f32_ws, bias, cv, cos_table, sin_table, seq_lens, B, num_heads, ld, stream);
}

extern "C" int b200_decode_rope_append_paged_c8(void* qkv, float* acc_f32_ws, const float* bias, void* key_cache,
                                                void* value_cache, const int32_t* block_tables, const void* cache_k_scale,
                                                const void* cache_v_scale, const float* cos_table, const float* sin_table,
                                                const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t num_kv_heads,
                                                int64_t head_dim, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld,
                                                cudaStream_t stream) {
  KvCacheC8 cv;
  if (int rc = paged_kv_cache_c8(&cv, key_cache, value_cache, block_tables, cache_k_scale, cache_v_scale, nullptr, nullptr, true,
                                 false, num_kv_heads, head_dim, block_size, max_blocks_per_seq, "decode_rope_append_paged_c8"))
    return rc;
  B200_CHECK_ARG(qkv && cos_table && sin_table && seq_lens, "decode_rope_append_paged_c8: null pointer");
  return rope_append_launch(qkv, acc_f32_ws, bias, cv, cos_table, sin_table, seq_lens, B, num_heads, ld, stream);
}

extern "C" int b200_get_padding_offset(const int64_t* input_ids, const int32_t* cum_offsets, const int32_t* seq_lens,
                                       int64_t* x_remove_padding, int32_t* padding_offset, int32_t* cum_offsets_out,
                                       int32_t* cu_seqlens_q, int32_t* cu_seqlens_k, int64_t bsz, int64_t max_seq_len,
                                       cudaStream_t stream) {
  B200_CHECK_ARG(input_ids && cum_offsets && seq_lens && x_remove_padding && padding_offset && cum_offsets_out &&
                     cu_seqlens_q && cu_seqlens_k && bsz > 0,
                 "get_padding_offset: bad arguments");
  padding_offset_kernel<<<static_cast<unsigned>(bsz), 128, 0, stream>>>(input_ids, cum_offsets, seq_lens, x_remove_padding,
                                                                       padding_offset, cum_offsets_out, cu_seqlens_q,
                                                                       cu_seqlens_k, (int)max_seq_len);
  return check_launch("get_padding_offset");
}

extern "C" int b200_rebuild_padding(const void* tmp_out, const int32_t* cum_offsets, const int32_t* seq_lens_decoder,
                                    const int32_t* seq_lens_encoder, void* out, int64_t bsz, int64_t max_len, int64_t dim,
                                    cudaStream_t stream) {
  B200_CHECK_ARG(tmp_out && cum_offsets && seq_lens_decoder && seq_lens_encoder && out && bsz > 0, "rebuild_padding: bad arguments");
  rebuild_padding_kernel<<<static_cast<unsigned>(bsz), 256, 0, stream>>>(static_cast<const bf16*>(tmp_out), cum_offsets,
                                                                        seq_lens_decoder, seq_lens_encoder,
                                                                        static_cast<bf16*>(out), (int)max_len, (int)dim);
  return check_launch("rebuild_padding");
}

extern "C" int b200_set_value_by_flags_and_idx(const bool* stop_flags, int64_t* pre_ids_all, const int64_t* pre_ids_now,
                                               const int64_t* step_idx, int64_t bs, int64_t length, cudaStream_t stream) {
  B200_CHECK_ARG(stop_flags && pre_ids_all && pre_ids_now && step_idx && bs > 0, "set_value_by_flags_and_idx: bad arguments");
  set_value_by_flags_kernel<<<static_cast<unsigned>((bs + 127) / 128), 128, 0, stream>>>(stop_flags, pre_ids_all, pre_ids_now,
                                                                                        step_idx, (int)bs, (int)length);
  return check_launch("set_value_by_flags_and_idx");
}

extern "C" int b200_set_value_by_flags_and_idx_v2(const bool* stop_flags, int64_t* pre_ids_all, const int64_t* input_ids,
                                                  const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder,
                                                  const int64_t* step_idx, int64_t bs, int64_t length,
                                                  int64_t length_input_ids, cudaStream_t stream) {
  B200_CHECK_ARG(stop_flags && pre_ids_all && input_ids && seq_lens_encoder && seq_lens_decoder && step_idx && bs > 0,
                 "set_value_by_flags_and_idx_v2: bad arguments");
  set_value_by_flags_v2_kernel<<<static_cast<unsigned>((bs + 127) / 128), 128, 0, stream>>>(
      stop_flags, pre_ids_all, input_ids, seq_lens_encoder, seq_lens_decoder, step_idx, (int)bs, (int)length,
      (int)length_input_ids);
  return check_launch("set_value_by_flags_and_idx_v2");
}

extern "C" int b200_token_penalty_multi_scores(const int64_t* pre_ids, float* logits, const float* penalty_scores,
                                               const float* frequency_scores, const float* presence_scores,
                                               const float* temperatures, const int64_t* bad_tokens, const int64_t* cur_len,
                                               const int64_t* min_len, const int64_t* eos_token_id, int32_t* workspace,
                                               int64_t bs, int64_t length, int64_t length_id, int64_t bad_len,
                                               int64_t eos_len, cudaStream_t stream) {
  B200_CHECK_ARG(pre_ids && logits && penalty_scores && frequency_scores && presence_scores && cur_len && min_len &&
                     eos_token_id && workspace && bs > 0 && length > 0,
                 "token_penalty_multi_scores: bad arguments");
  cudaError_t e = cudaMemsetAsync(workspace, 0, static_cast<size_t>(bs) * length * sizeof(int32_t), stream);
  if (e != cudaSuccess) {
    set_last_error("token_penalty memset: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  penalty_count_kernel<<<static_cast<unsigned>(bs), 1, 0, stream>>>(pre_ids, cur_len, workspace, length, length_id);
  int rc = check_launch("token_penalty(count)");
  if (rc) return rc;
  penalty_apply_kernel<<<static_cast<unsigned>(bs), 512, 0, stream>>>(logits, workspace, penalty_scores, frequency_scores,
                                                                     presence_scores, temperatures, cur_len, min_len,
                                                                     eos_token_id, eos_len, bad_tokens, bad_len, length);
  return check_launch("token_penalty(apply)");
}

extern "C" int b200_set_stop_value_multi_ends(bool* stop_flags, int64_t* topk_ids, int64_t* next_tokens,
                                              const int64_t* end_ids, const int32_t* seq_lens, int64_t bs, int64_t end_length,
                                              int v2, cudaStream_t stream) {
  B200_CHECK_ARG(stop_flags && topk_ids && end_ids && bs > 0 && end_length > 0, "set_stop_value_multi_ends: bad arguments");
  B200_CHECK_ARG(!v2 || (next_tokens && seq_lens), "set_stop_value_multi_ends(v2): next_tokens and seq_lens required");
  stop_value_kernel<<<static_cast<unsigned>((bs + 127) / 128), 128, 0, stream>>>(stop_flags, topk_ids, next_tokens, end_ids,
                                                                                seq_lens, (int)bs, (int)end_length, v2);
  return check_launch("set_stop_value_multi_ends");
}

extern "C" int b200_update_inputs(bool* not_need_stop, int32_t* seq_lens_this_time, int32_t* seq_lens_encoder,
                                  int32_t* seq_lens_decoder, int64_t* input_ids, const int64_t* stop_nums,
                                  const bool* stop_flags, const bool* is_block_step, const int64_t* next_tokens, int64_t bsz,
                                  int64_t max_bsz, int64_t input_ids_stride, cudaStream_t stream) {
  B200_CHECK_ARG(not_need_stop && seq_lens_this_time && seq_lens_encoder && seq_lens_decoder && input_ids && stop_nums &&
                     stop_flags && is_block_step && next_tokens,
                 "update_inputs: null pointer");
  B200_CHECK_ARG(bsz > 0 && bsz <= max_bsz && max_bsz <= 1024, "update_inputs: need 0 < bsz <= max_bsz <= 1024");
  update_inputs_kernel<<<1, 1024, 0, stream>>>(not_need_stop, seq_lens_this_time, seq_lens_encoder, seq_lens_decoder,
                                              input_ids, stop_nums, stop_flags, is_block_step, next_tokens, (int)bsz,
                                              (int)max_bsz, (int)input_ids_stride);
  return check_launch("update_inputs");
}

extern "C" int b200_generate_step_update(int64_t* next_tokens, bool* stop_flags, int64_t* step_idx, const int64_t* max_dec_len,
                                         int32_t* seq_len_decoder, int64_t* pre_ids, int64_t pre_len, const int64_t* eos_ids,
                                         int64_t eos_len, int64_t* out_tokens, int64_t out_stride, int64_t out_col,
                                         int64_t* out_col_dev, int32_t* stop_count, int64_t bs, cudaStream_t stream) {
  B200_CHECK_ARG(next_tokens && stop_flags && step_idx && max_dec_len && seq_len_decoder && pre_ids && eos_ids && stop_count &&
                     bs > 0 && eos_len > 0,
                 "generate_step_update: bad arguments");
  cudaError_t e = cudaMemsetAsync(stop_count, 0, sizeof(int32_t), stream);
  if (e != cudaSuccess) {
    set_last_error("generate_step_update memset: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  generate_step_update_kernel<<<static_cast<unsigned>((bs + 127) / 128), 128, 0, stream>>>(
      next_tokens, stop_flags, step_idx, max_dec_len, seq_len_decoder, pre_ids, pre_len, eos_ids, (int)eos_len, out_tokens,
      out_stride, out_col, out_col_dev, stop_count, (int)bs);
  int rc = check_launch("generate_step_update");
  if (rc) return rc;
  if (out_col_dev != nullptr) {
    increment_i64_kernel<<<1, 1, 0, stream>>>(out_col_dev);
    rc = check_launch("generate_step_update(counter)");
  }
  return rc;
}

extern "C" int b200_argmax_f32(const float* logits, int64_t* out, int64_t rows, int64_t vocab, int64_t ld,
                               cudaStream_t stream) {
  B200_CHECK_ARG(logits && out && rows > 0 && vocab > 0, "argmax_f32: bad arguments");
  argmax_f32_kernel<<<static_cast<unsigned>(rows), 256, 0, stream>>>(logits, out, (int)vocab, ld);
  return check_launch("argmax_f32");
}

extern "C" int b200_bf16_rows_to_f32(const void* src, float* dst, int64_t rows, int64_t cols, int64_t ld,
                                     cudaStream_t stream) {
  B200_CHECK_ARG(src && dst && rows > 0 && cols > 0, "bf16_rows_to_f32: bad arguments");
  bf16_rows_to_f32_kernel<<<sm_count() * 4, 256, 0, stream>>>(static_cast<const bf16*>(src), dst, rows, cols, ld);
  return check_launch("bf16_rows_to_f32");
}

extern "C" int b200_softmax_f32(float* logits, int64_t rows, int64_t vocab, int64_t ld, cudaStream_t stream) {
  B200_CHECK_ARG(logits && rows > 0 && vocab > 0 && vocab % 4 == 0 && ld % 4 == 0, "softmax_f32: vocab and ld must be multiples of 4");
  softmax_f32_kernel<<<static_cast<unsigned>(rows), 1024, 0, stream>>>(logits, (int)vocab, ld);
  return check_launch("softmax_f32");
}

extern "C" int b200_top_p_sampling_reject(const float* probs, const float* top_p, const float* uniform, int64_t* out,
                                          int64_t bs, int64_t vocab, int64_t ld, int64_t max_rounds, cudaStream_t stream) {
  B200_CHECK_ARG(probs && top_p && uniform && out, "top_p_sampling_reject: null pointer");
  B200_CHECK_ARG(bs > 0 && vocab > 0 && vocab % 4 == 0 && ld % 4 == 0 && max_rounds > 0,
                 "top_p_sampling_reject: vocab and ld must be multiples of 4");
  top_p_sampling_reject_kernel<<<static_cast<unsigned>(bs), 1024, 0, stream>>>(probs, top_p, uniform, out, (int)vocab, ld,
                                                                               (int)bs, (int)max_rounds);
  return check_launch("top_p_sampling_reject");
}

// ------------------------------------------------------------------------------------------------------------------
// fused_get_rotary_embedding (csrc/gpu/fused_get_rope.cu:40-223): position ids -> fp32 cos / sin tables
//   out [2, bsz, 1, seq, head_dim]:  out[0] = cos, out[1] = sin of  position_ids[b, s + prompt_num] * theta^(-2j/head_dim)
//   use_neox != 0 ("neox" in csrc naming == rotate-half, the Llama / Qwen2 convention, SURVEY.md §8 naming trap):
//       value j is stored at columns j and j + head_dim/2;   use_neox == 0: at columns 2j and 2j+1 (interleaved pairs).
// One thread per (b, s, j): powf / cosf / sinf in fp32 like the reference kernel; the two copies of each value are written as
// one 8-byte store in the interleaved layout and as two coalesced 4-byte stores in the half-split layout.
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace gen {
__global__ void __launch_bounds__(256) fused_get_rope_kernel(const int64_t* __restrict__ position_ids, float* __restrict__ out,
                                                            int bsz, int seq, int pos_stride, int head_dim, int prompt_num,
                                                            float inv_head_dim, float theta, int use_neox) {
  const int half = head_dim >> 1;
  const int64_t total = static_cast<int64_t>(bsz) * seq * half;
  const int64_t sin_base = static_cast<int64_t>(bsz) * seq * head_dim;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t bs_idx = idx / half;
    const int j = static_cast<int>(idx - bs_idx * half);
    const int b = static_cast<int>(bs_idx / seq), s_ = static_cast<int>(bs_idx - static_cast<int64_t>(b) * seq);
    const float exponent = -static_cast<float>(2 * j) * inv_head_dim;
    const float inv_freq = powf(theta, exponent);
    const float f = static_cast<float>(position_ids[static_cast<int64_t>(b) * pos_stride + s_ + prompt_num]) * inv_freq;
    const float c = cosf(f), sn = sinf(f);
    const int64_t row = bs_idx * head_dim;
    if (use_neox) {
      out[row + j] = c; out[row + j + half] = c;
      out[sin_base + row + j] = sn; out[sin_base + row + j + half] = sn;
    } else {
      *reinterpret_cast<float2*>(out + row + 2 * j) = make_float2(c, c);
      *reinterpret_cast<float2*>(out + sin_base + row + 2 * j) = make_float2(sn, sn);
    }
  }
}
}  // namespace gen
}  // namespace b200

extern "C" int b200_fused_get_rotary_embedding(const int64_t* position_ids, float* rope_embedding, int64_t bsz,
                                               int64_t max_seq_length, int64_t max_position_seq_length, int64_t head_dim,
                                               int64_t prompt_num, float theta, int use_neox, cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(position_ids && rope_embedding, "fused_get_rotary_embedding: null pointer");
  B200_CHECK_ARG(bsz > 0 && max_seq_length > 0 && head_dim > 0 && head_dim % 2 == 0 && prompt_num >= 0 &&
                     max_seq_length + prompt_num <= max_position_seq_length,
                 "fused_get_rotary_embedding: need even head_dim and seq + prompt_num <= position_ids row length "
                 "(bsz=%lld seq=%lld pos_len=%lld head_dim=%lld prompt_num=%lld)",
                 (long long)bsz, (long long)max_seq_length, (long long)max_position_seq_length, (long long)head_dim,
                 (long long)prompt_num);
  const int64_t total = bsz * max_seq_length * (head_dim / 2);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  gen::fused_get_rope_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      position_ids, rope_embedding, (int)bsz, (int)max_seq_length, (int)max_position_seq_length, (int)head_dim, (int)prompt_num,
      1.0f / static_cast<float>(head_dim), theta, use_neox);
  return check_launch("fused_get_rotary_embedding");
}

// ------------------------------------------------------------------------------------------------------------------
// step_paddle (csrc/gpu/step.cu:19-283): continuous-batching block bookkeeping of the paged KV cache, one call per decode step.
//   1. finished sequences hand their decoder blocks back to the free list; running sequences whose next token falls into an
//      unallocated block register a request                                              (free_and_dispatch_block :41-67)
//   2. while requests outnumber free blocks, the running sequence holding the most decoder blocks is pre-empted ("block
//      step"): its decoder blocks are freed and it is parked in step_block_list            (:73-103)
//   3. every surviving request receives one block from the tail of the free list            (:105-117)
//   4. parked sequences are recovered, last-parked first, while the free list can hold their decoder blocks plus one (:119-150)
//   5. a recovered sequence is re-armed for a fresh prefill over prompt + generated tokens: lengths, stop flag, input ids
//      rebuilt from pre_ids, its decoder blocks re-attached                                 (recover_block :154-214)
// The reference runs 1-4 in one 512-thread CTA with atomicAdd/atomicSub on the list lengths (so the ORDER of blocks in the
// free list depends on thread timing), copies recover_len to the host, and launches step 5 with that grid.  Here everything is
// ONE launch of one CTA: list positions come from block-wide prefix sums in sequence-index order (deterministic, and one of the
// orders the reference's atomics can produce), the arg-max is a shuffle reduction (ties -> lowest index, as cub::ArgMax), and
// step 5 loops over the recovered sequences inside the same CTA — no host round trip.
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace gen {

constexpr int STEP_THREADS = 1024;

// exclusive prefix sum over the CTA (value per thread) + total; all STEP_THREADS threads must call
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();                       // s_warp may still be read from a previous call
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  if (w == 0) {
    int x = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += n;
    }
    s_warp[lane] = x;                    // inclusive over warps
  }
  __syncthreads();
  const int base = w == 0 ? 0 : s_warp[w - 1];
  *total = s_warp[31];
  return base + inc - v;
}

__global__ void __launch_bounds__(STEP_THREADS, 1)
step_paddle_kernel(bool* stop_flags, int* seq_lens_this_time, const int* ori_seq_lens_encoder, int* seq_lens_encoder,
                   int* seq_lens_decoder, int* block_tables, int* encoder_block_lens, bool* is_block_step, int* step_block_list,
                   int* step_len, int* recover_block_list, int* recover_len, int* need_block_list, int* need_block_len,
                   int* used_list_len, int* free_list, int* free_list_len, int64_t* input_ids, const int64_t* pre_ids,
                   const int64_t* step_idx, const int64_t* next_tokens, int bsz, int block_size, int block_num_per_seq, int length,
                   int pre_id_length, int64_t first_token_id) {
  __shared__ int s_warp[32];
  __shared__ int s_key[32], s_val[32];
  __shared__ int s_free_len, s_need_len, s_best_key, s_best_val;
  const int tid = threadIdx.x;
  const int max_decoder_block_num = length / block_size;
  int* tbl = block_tables + static_cast<int64_t>(tid < bsz ? tid : 0) * block_num_per_seq;

  // ---- 1. free finished sequences / collect block requests (positions by prefix sum, in sequence order) ----
  int n_free = 0, need = 0, enc_len = 0;
  if (tid < bsz) {
    if (stop_flags[tid] && !is_block_step[tid]) {
      n_free = used_list_len[tid];
      enc_len = encoder_block_lens[tid];
    } else if (seq_lens_decoder[tid] != 0 && tbl[seq_lens_decoder[tid] / block_size] == -1) {
      need = 1;
    }
  }
  int total_free, total_need;
  const int free_pos = block_exclusive_scan(n_free, s_warp, &total_free);
  const int need_pos = block_exclusive_scan(need, s_warp, &total_need);
  const int free0 = *free_list_len, need0 = *need_block_len;
  if (n_free > 0) {
    for (int i = 0; i < n_free; ++i) {
      free_list[free0 + free_pos + i] = tbl[enc_len + i];
      tbl[enc_len + i] = -1;
    }
    encoder_block_lens[tid] = 0;
    used_list_len[tid] = 0;
  }
  if (need) need_block_list[need0 + need_pos] = tid;
  __syncthreads();
  if (tid == 0) {
    s_free_len = free0 + total_free;
    s_need_len = need0 + total_need;
  }
  __syncthreads();

  // ---- 2. pre-empt the largest holders until the requests fit ----
  while (s_need_len > s_free_len) {
    int key = tid, val = (tid < bsz && !is_block_step[tid]) ? used_list_len[tid] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int k2 = __shfl_xor_sync(0xffffffffu, key, o), v2 = __shfl_xor_sync(0xffffffffu, val, o);
      if (v2 > val || (v2 == val && k2 < key)) { key = k2; val = v2; }
    }
    if ((tid & 31) == 0) { s_key[tid >> 5] = key; s_val[tid >> 5] = val; }
    __syncthreads();
    if (tid < 32) {
      key = s_key[tid]; val = s_val[tid];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const int k2 = __shfl_xor_sync(0xffffffffu, key, o), v2 = __shfl_xor_sync(0xffffffffu, val, o);
        if (v2 > val || (v2 == val && k2 < key)) { key = k2; val = v2; }
      }
      if (tid == 0) { s_best_key = key; s_best_val = val; }
    }
    __syncthreads();
    if (s_best_val <= 0) break;          // nothing left to reclaim (the reference would spin here forever)
    if (tid == 0) {
      const int k = s_best_key, v = s_best_val;
      int* t2 = block_tables + static_cast<int64_t>(k) * block_num_per_seq;
      const int e = encoder_block_lens[k];
      for (int i = 0; i < v; ++i) {
        free_list[s_free_len + i] = t2[e + i];
        t2[e + i] = -1;
      }
      step_block_list[*step_len] = k;
      *step_len += 1;
      s_free_len += v;
      stop_flags[k] = true;
      is_block_step[k] = true;
      seq_lens_this_time[k] = 0;
      seq_lens_decoder[k] = 0;
    }
    __syncthreads();
  }

  // ---- 3. one block per surviving request, taken from the tail of the free list in request order ----
  int req = -1, active = 0;
  if (tid < s_need_len) {
    req = need_block_list[tid];
    active = !stop_flags[req];
  }
  int total_active;
  const int apos = block_exclusive_scan(active, s_warp, &total_active);
  if (active) {
    used_list_len[req] += 1;
    int* t2 = block_tables + static_cast<int64_t>(req) * block_num_per_seq;
    t2[seq_lens_decoder[req] / block_size] = free_list[s_free_len - 1 - apos];
  }
  if (tid < s_need_len) need_block_list[tid] = -1;
  __syncthreads();

  // ---- 4. which parked sequences fit again (last parked first; one spare block each) ----
  if (tid == 0) {
    s_free_len -= total_active;
    int ori_free = s_free_len;
    int ori_step_len = *step_len;
    if (ori_step_len > 0) {
      int sid = step_block_list[ori_step_len - 1];
      int tmp_used = used_list_len[sid];
      int used_len = tmp_used < max_decoder_block_num ? tmp_used + 1 : tmp_used;
      while (ori_step_len > 0 && ori_free >= used_len) {
        recover_block_list[*recover_len] = sid;
        is_block_step[sid] = false;
        used_list_len[sid] = used_len;
        ori_free -= used_len;
        step_block_list[ori_step_len - 1] = -1;
        *step_len -= 1;
        *recover_len += 1;
        ori_step_len = *step_len;
        if (ori_step_len > 0) {
          sid = step_block_list[ori_step_len - 1];
          tmp_used = used_list_len[sid];
          used_len = tmp_used < max_decoder_block_num ? tmp_used + 1 : tmp_used;
        }
      }
    }
    *need_block_len = 0;
  }
  __syncthreads();

  // ---- 5. re-arm the recovered sequences (recover_block), in recover-list order ----
  const int n_rec = *recover_len;
  for (int r = 0; r < n_rec; ++r) {
    const int rid = recover_block_list[r];
    const int ori_enc = ori_seq_lens_encoder[rid];
    const int step_now = static_cast<int>(step_idx[rid]);
    const int seq_len = ori_enc + step_now;
    const int e = encoder_block_lens[rid];
    const int used = used_list_len[rid];
    int* t2 = block_tables + static_cast<int64_t>(rid) * block_num_per_seq;
    int64_t* ids = input_ids + static_cast<int64_t>(rid) * length;
    const int64_t* pre = pre_ids + static_cast<int64_t>(rid) * pre_id_length;
    const int ori_free = s_free_len;
    for (int i = tid; i < used; i += STEP_THREADS) t2[e + i] = free_list[ori_free - i - 1];
    for (int i = tid; i < step_now - 1; i += STEP_THREADS) ids[ori_enc + i] = pre[i + 1];
    __syncthreads();                      // the element writes below overwrite positions of the loops above
    if (tid == 0) {
      seq_lens_this_time[rid] = seq_len;
      seq_lens_encoder[rid] = seq_len;
      stop_flags[rid] = false;
      ids[ori_enc + step_now - 1] = next_tokens[rid];
      ids[0] = first_token_id;
      s_free_len = ori_free - used;
    }
    __syncthreads();
  }
  if (tid == 0) {
    *recover_len = 0;
    *free_list_len = s_free_len;
  }
}
}  // namespace gen
}  // namespace b200

extern "C" int b200_step_paddle(bool* stop_flags, int32_t* seq_lens_this_time, const int32_t* ori_seq_lens_encoder,
                                int32_t* seq_lens_encoder, int32_t* seq_lens_decoder, int32_t* block_tables,
                                int32_t* encoder_block_lens, bool* is_block_step, int32_t* step_block_list, int32_t* step_lens,
                                int32_t* recover_block_list, int32_t* recover_lens, int32_t* need_block_list,
                                int32_t* need_block_len, int32_t* used_list_len, int32_t* free_list, int32_t* free_list_len,
                                int64_t* input_ids, const int64_t* pre_ids, const int64_t* step_idx, const int64_t* next_tokens,
                                int64_t bsz, int64_t block_size, int64_t block_num_per_seq, int64_t length, int64_t pre_id_length,
                                int64_t first_token_id, cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(stop_flags && seq_lens_this_time && ori_seq_lens_encoder && seq_lens_encoder && seq_lens_decoder && block_tables &&
                     encoder_block_lens && is_block_step && step_block_list && step_lens && recover_block_list && recover_lens &&
                     need_block_list && need_block_len && used_list_len && free_list && free_list_len && input_ids && pre_ids &&
                     step_idx && next_tokens,
                 "step_paddle: null pointer");
  B200_CHECK_ARG(bsz > 0 && bsz <= gen::STEP_THREADS && block_size > 0 && block_num_per_seq > 0 && length > 0 && pre_id_length > 0,
                 "step_paddle: need 0 < bsz <= %d and positive sizes", gen::STEP_THREADS);
  gen::step_paddle_kernel<<<1, gen::STEP_THREADS, 0, stream>>>(
      stop_flags, seq_lens_this_time, ori_seq_lens_encoder, seq_lens_encoder, seq_lens_decoder, block_tables, encoder_block_lens,
      is_block_step, step_block_list, step_lens, recover_block_list, recover_lens, need_block_list, need_block_len, used_list_len,
      free_list, free_list_len, input_ids, pre_ids, step_idx, next_tokens, (int)bsz, (int)block_size, (int)block_num_per_seq,
      (int)length, (int)pre_id_length, first_token_id);
  return check_launch("step_paddle");
}

// ------------------------------------------------------------------------------------------------------------------
// retire_admit: the continuous-batching half step_paddle leaves to its caller, run right after it every step.  One CTA, one
// thread per slot, list positions from prefix sums in slot order (deterministic), no host synchronisation.
//   0. a slot recovered by step_paddle this step gets its first prompt token back in input_ids[b, 0] (update_inputs wrote the
//      last generated token there; step_paddle restores one first_token_id for every slot)
//   1. a parked slot (is_block_step) hands its encoder blocks back too and counts them as decoder blocks: step_paddle then
//      recovers it with a fresh table of used + 1 blocks from position 0.  A parked slot so holds no block, and a pool of at
//      least the largest request's pages can always recover the last-parked sequence once nothing else runs.
//   2. a slot that stopped (and is not parked) retires: its tokens pre_ids[b, 1 .. step_idx-1] + next_tokens[b] go to row
//      slot_request[b] of out_ids, its encoder blocks to the free list (step_paddle freed the decoder blocks and zeroed
//      encoder_block_lens, leaving the encoder blocks in the row), the slot empties
//   3. FIFO admission while no sequence is parked: the k-th empty slot takes request cursor + k if the free list holds the
//      blocks of it and of every request before it, and the pool keeps one spare block per resident slot; the blocks are
//      popped from the tail of the free list
//   4. the step header in (pinned, device-mapped) host memory
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace gen {

__global__ void __launch_bounds__(STEP_THREADS, 1)
retire_admit_kernel(bool* stop_flags, bool* is_block_step, int* seq_lens_this_time, int* seq_lens_encoder,
                    int* ori_seq_lens_encoder, int* seq_lens_decoder, int64_t* step_idx, int64_t* pre_ids,
                    const int64_t* next_tokens, int64_t* input_ids, int* block_tables, int* encoder_block_lens, int* used_list_len,
                    int* free_list, int* free_list_len, const int* step_lens, int64_t* max_dec_len, int64_t* min_dec_len,
                    int* slot_request, const int64_t* prompt_ids, const int* prompt_offsets, const int64_t* req_max_dec_len,
                    const int64_t* req_min_dec_len, int* cursor, int64_t* out_ids, int* out_lens, volatile int* header, int bsz,
                    int block_size, int block_num_per_seq, int length, int pre_id_length, int num_requests, int out_stride) {
  __shared__ int s_warp[32];
  __shared__ int s_slot[STEP_THREADS], s_req[STEP_THREADS];
  __shared__ int s_max_q;
  const int tid = threadIdx.x;
  const bool valid = tid < bsz;
  int* tbl = block_tables + static_cast<int64_t>(valid ? tid : 0) * block_num_per_seq;
  if (tid == 0) s_max_q = 0;
  const int req = valid ? slot_request[tid] : -1;

  // ---- 0 / 1 / 2: recovered, parked and retiring slots ----
  const bool parked = valid && is_block_step[tid];
  const bool retire = valid && req >= 0 && stop_flags[tid] && !parked;
  const bool recovered = valid && req >= 0 && !stop_flags[tid] && seq_lens_encoder[tid] > 0 && step_idx[tid] > 0;
  if (recovered) input_ids[static_cast<int64_t>(tid) * length] = prompt_ids[prompt_offsets[req]];
  // the blocks a parked or stopped slot still holds are its encoder blocks, a prefix of its row: step_paddle cleared the
  // decoder entries (and, for a stopped slot, zeroed encoder_block_lens too)
  int n_push = 0;
  if (parked || retire)
    while (n_push < block_num_per_seq && tbl[n_push] >= 0) ++n_push;
  int total_push;
  const int push_pos = block_exclusive_scan(n_push, s_warp, &total_push);
  const int free0 = *free_list_len;
  for (int i = 0; i < n_push; ++i) {
    free_list[free0 + push_pos + i] = tbl[i];
    tbl[i] = -1;
  }
  if (parked || retire) encoder_block_lens[tid] = 0;
  if (parked) used_list_len[tid] += n_push;
  if (retire) slot_request[tid] = -1;
  int n_retire;
  const int rpos = block_exclusive_scan(retire ? 1 : 0, s_warp, &n_retire);
  if (retire) { s_slot[rpos] = tid; s_req[rpos] = req; }
  int n_recovered;
  block_exclusive_scan(recovered ? 1 : 0, s_warp, &n_recovered);
  __syncthreads();
  for (int k = 0; k < n_retire; ++k) {
    const int b = s_slot[k], r = s_req[k];
    int n = static_cast<int>(step_idx[b]);
    n = n < out_stride ? n : out_stride;
    const int64_t* pre = pre_ids + static_cast<int64_t>(b) * pre_id_length;
    int64_t* out = out_ids + static_cast<int64_t>(r) * out_stride;
    for (int i = tid; i < n; i += STEP_THREADS) out[i] = i + 1 < n ? pre[i + 1] : next_tokens[b];
    if (tid == 0) out_lens[r] = n;
  }

  // ---- 3: FIFO admission into the empty slots, in slot order ----
  const int free1 = free0 + total_push;
  const int cur = *cursor;
  const bool empty = valid && (retire || req < 0);
  int n_empty, occupied0, held_dec;
  const int epos = block_exclusive_scan(empty ? 1 : 0, s_warp, &n_empty);
  block_exclusive_scan(valid && !empty ? 1 : 0, s_warp, &occupied0);
  block_exclusive_scan(valid && !empty && !parked ? used_list_len[tid] : 0, s_warp, &held_dec);
  const int r = cur + epos;
  const bool cand = empty && *step_lens == 0 && r < num_requests;
  const int plen = cand ? prompt_offsets[r + 1] - prompt_offsets[r] : 0;
  const int need = (plen + block_size - 1) / block_size;
  int total_need;
  const int excl = block_exclusive_scan(need, s_warp, &total_need);
  // the blocks must be free now, and the pool must keep one block per resident slot beyond every encoder block: step_paddle
  // can only pre-empt decoder blocks, so a step in which each resident asks for one more block is always served.  Needs are
  // >= 1 and the candidates a prefix of the empty slots: the admitted are a prefix too (epos = admissions before this one)
  const bool admit = cand && excl + need <= free1 && excl + need + occupied0 + epos + 1 <= free1 + held_dec;
  int n_admit;
  block_exclusive_scan(admit ? 1 : 0, s_warp, &n_admit);
  int popped;
  block_exclusive_scan(admit ? need : 0, s_warp, &popped);
  if (admit) {
    for (int j = 0; j < need; ++j) tbl[j] = free_list[free1 - 1 - excl - j];
    encoder_block_lens[tid] = need;
    used_list_len[tid] = 0;
    seq_lens_this_time[tid] = plen;
    seq_lens_encoder[tid] = plen;
    ori_seq_lens_encoder[tid] = plen;
    seq_lens_decoder[tid] = 0;
    step_idx[tid] = 0;
    stop_flags[tid] = false;
    max_dec_len[tid] = req_max_dec_len[r];
    min_dec_len[tid] = req_min_dec_len[r];
    slot_request[tid] = r;
    s_slot[epos] = tid;
    s_req[epos] = r;
  }
  __syncthreads();
  for (int k = 0; k < n_admit; ++k) {
    const int b = s_slot[k], rq = s_req[k];
    const int64_t* src = prompt_ids + prompt_offsets[rq];
    const int n = prompt_offsets[rq + 1] - prompt_offsets[rq];
    int64_t* ids = input_ids + static_cast<int64_t>(b) * length;
    for (int i = tid; i < n; i += STEP_THREADS) ids[i] = src[i];
    int64_t* pre = pre_ids + static_cast<int64_t>(b) * pre_id_length;
    for (int i = tid; i < pre_id_length; i += STEP_THREADS) pre[i] = -1;
  }

  // ---- 4: step header ----
  const int this_time = valid ? seq_lens_this_time[tid] : 0;
  if (this_time > 0) atomicMax(&s_max_q, this_time);
  int token_num, running, occupied;
  block_exclusive_scan(this_time, s_warp, &token_num);
  block_exclusive_scan(this_time > 0 ? 1 : 0, s_warp, &running);
  block_exclusive_scan(valid && slot_request[tid] >= 0 ? 1 : 0, s_warp, &occupied);
  __syncthreads();
  if (tid == 0) {
    const int new_cursor = cur + n_admit;
    const int parked_now = *step_lens;
    *cursor = new_cursor;
    *free_list_len = free1 - popped;
    header[B200_RA_PREEMPTIONS] = header[B200_RA_PREEMPTIONS] + parked_now - header[B200_RA_PARKED] + n_recovered;
    header[B200_RA_RECOVERIES] = header[B200_RA_RECOVERIES] + n_recovered;
    header[B200_RA_TOKEN_NUM] = token_num;
    header[B200_RA_MAX_Q_LEN] = s_max_q;
    header[B200_RA_RUNNING] = running;
    header[B200_RA_PENDING] = num_requests - new_cursor;
    header[B200_RA_PARKED] = parked_now;
    header[B200_RA_FREE_BLOCKS] = free1 - popped;
    header[B200_RA_ADMITTED] = n_admit;
    header[B200_RA_RETIRED] = n_retire;
    header[B200_RA_DONE] = (occupied == 0 && new_cursor >= num_requests) ? 1 : 0;
    __threadfence_system();
  }
}
}  // namespace gen
}  // namespace b200

extern "C" int b200_retire_admit(bool* stop_flags, bool* is_block_step, int32_t* seq_lens_this_time, int32_t* seq_lens_encoder,
                                 int32_t* ori_seq_lens_encoder, int32_t* seq_lens_decoder, int64_t* step_idx, int64_t* pre_ids,
                                 const int64_t* next_tokens, int64_t* input_ids, int32_t* block_tables, int32_t* encoder_block_lens,
                                 int32_t* used_list_len, int32_t* free_list, int32_t* free_list_len, const int32_t* step_lens,
                                 int64_t* max_dec_len, int64_t* min_dec_len, int32_t* slot_request, const int64_t* prompt_ids,
                                 const int32_t* prompt_offsets, const int64_t* req_max_dec_len, const int64_t* req_min_dec_len,
                                 int32_t* cursor, int64_t* out_ids, int32_t* out_lens, int32_t* header, int64_t bsz,
                                 int64_t block_size, int64_t block_num_per_seq, int64_t length, int64_t pre_id_length,
                                 int64_t num_requests, int64_t out_stride, int64_t max_prompt_len, int64_t max_seq_len,
                                 cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(stop_flags && is_block_step && seq_lens_this_time && seq_lens_encoder && ori_seq_lens_encoder && seq_lens_decoder &&
                     step_idx && pre_ids && next_tokens && input_ids && block_tables && encoder_block_lens && used_list_len &&
                     free_list && free_list_len && step_lens && max_dec_len && min_dec_len && slot_request && prompt_ids &&
                     prompt_offsets && req_max_dec_len && req_min_dec_len && cursor && out_ids && out_lens && header,
                 "retire_admit: null pointer");
  B200_CHECK_ARG(bsz > 0 && bsz <= gen::STEP_THREADS, "retire_admit: need 0 < bsz <= %d (got %lld)", gen::STEP_THREADS,
                 (long long)bsz);
  B200_CHECK_ARG(block_size > 0 && block_num_per_seq > 0 && num_requests > 0 && out_stride > 0 && max_prompt_len > 0 &&
                     max_seq_len >= max_prompt_len && pre_id_length >= out_stride,
                 "retire_admit: need positive sizes, max_seq_len >= max_prompt_len and pre_id_length >= out_stride");
  B200_CHECK_ARG(max_prompt_len <= block_num_per_seq * block_size,
                 "retire_admit: a prompt of %lld tokens does not fit block_num_per_seq %lld x block_size %lld",
                 (long long)max_prompt_len, (long long)block_num_per_seq, (long long)block_size);
  B200_CHECK_ARG(max_seq_len <= length, "retire_admit: input_ids rows of %lld tokens are too narrow for prompt + max length %lld",
                 (long long)length, (long long)max_seq_len);
  gen::retire_admit_kernel<<<1, gen::STEP_THREADS, 0, stream>>>(
      stop_flags, is_block_step, seq_lens_this_time, seq_lens_encoder, ori_seq_lens_encoder, seq_lens_decoder, step_idx, pre_ids,
      next_tokens, input_ids, block_tables, encoder_block_lens, used_list_len, free_list, free_list_len, step_lens, max_dec_len,
      min_dec_len, slot_request, prompt_ids, prompt_offsets, req_max_dec_len, req_min_dec_len, cursor, out_ids, out_lens, header,
      (int)bsz, (int)block_size, (int)block_num_per_seq, (int)length, (int)pre_id_length, (int)num_requests, (int)out_stride);
  return check_launch("retire_admit");
}

// ------------------------------------------------------------------------------------------------------------------
// save_output / get_output replacement (csrc/gpu/save_with_output_msg.cc:28-52, csrc/gpu/get_output.cc:28-60).
// The reference copies the step's tokens to the host synchronously (two blocking D2H copies per decode step) and pushes them
// into a SysV message queue as  int mtext[MAX_BSZ + 2] = {not_need_stop ? 1 : -1, bsz, tokens...}.  Here the decode step's own
// stream writes the same message straight into a ring of slots in PINNED, DEVICE-MAPPED host memory — no copy engine, no host
// synchronisation, CUDA-graph replayable — and publishes it by storing the step's sequence number into the slot header LAST
// (after __threadfence_system()); a host reader thread polls the header (paddlenlp_b200/experimental/transformers/token_stream.py).
//   slot layout (int32):  [0] seq = step + 1 (0 = never written)   [1] flag (1 running / -1 finished)   [2] bsz   [3 ..] tokens
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace gen {
__global__ void __launch_bounds__(512) save_output_stream_kernel(const int64_t* __restrict__ tokens, const int32_t* __restrict__ stop_count,
                                                                 volatile int32_t* ring, int64_t slot_stride, int64_t num_slots,
                                                                 int64_t* step_counter, int64_t last_step, int bs) {
  const int64_t step = *step_counter;
  volatile int32_t* slot = ring + (step % num_slots) * slot_stride;
  for (int i = threadIdx.x; i < bs; i += blockDim.x) slot[3 + i] = static_cast<int32_t>(tokens[i]);
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool finished = (stop_count != nullptr && *stop_count >= bs) || (last_step >= 0 && step >= last_step);
    slot[1] = finished ? -1 : 1;
    slot[2] = bs;
    __threadfence_system();
    slot[0] = static_cast<int32_t>(step + 1);
    __threadfence_system();
    *step_counter = step + 1;
  }
}
}  // namespace gen
}  // namespace b200

extern "C" int b200_save_output_stream(const int64_t* next_tokens, const int32_t* stop_count, int32_t* ring, int64_t slot_stride,
                                       int64_t num_slots, int64_t* step_counter, int64_t last_step, int64_t bs,
                                       cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(next_tokens && ring && step_counter, "save_output_stream: null pointer");
  B200_CHECK_ARG(bs > 0 && num_slots > 0 && slot_stride >= bs + 3, "save_output_stream: need slot_stride >= bs + 3 (bs=%lld stride=%lld)",
                 (long long)bs, (long long)slot_stride);
  gen::save_output_stream_kernel<<<1, 512, 0, stream>>>(next_tokens, stop_count, ring, slot_stride, num_slots, step_counter,
                                                        last_step, (int)bs);
  return check_launch("save_output_stream");
}

// ------------------------------------------------------------------------------------------------------------------
// append_attention (csrc/gpu/append_attention.cu:428-851; encoder / decoder cache writers append_attn/
// encoder_write_cache_with_rope_impl.cuh:22-690, decoder_write_cache_with_rope_kernel.cu; tile planning
// get_block_shape_and_split_kv_block.cu:23-294): ONE entry point for a mixed batch over the paged KV cache.  Sequence b
// contributes seq_lens_this_time[b] token rows of the packed (remove-padding) QKV projection, at absolute positions
// seq_lens_decoder[b] + i:
//     prompt / prompt CHUNK   (seq_lens_encoder[b] > 0, or more than one row): rows attend to the cached prefix + themselves
//     decode                  (one row, seq_lens_encoder[b] == 0)
//     idle slot               (seq_lens_this_time[b] == 0)
//   1. append_rope_write_kernel  RoPE (rotate-half) on q, k of EVERY new row in place + k, v appended to the pages (one launch
//                                for prompt and decode rows alike); decode rows' q are also gathered into a dense [B, ld] buffer
//   2. fa_fwd_kernel<d, 8, PAGED> prompt rows: flash attention, q tiles of 128 rows, K/V rows gathered page by page with
//                                cp.async, causal band offset by the cached prefix (chunked prefill)
//   3. decode_attention_tc<PAGED> decode rows (the decode step's kernel; sequences of the other kinds, idle slots included,
//                                have length -1 = no work)
//   4. scatter of the decode rows' outputs back to their token rows
// No host synchronisation: each kernel decides from the device-resident length arrays which sequences are its own (the
// reference plans tiles on the device too, but copies the plan sizes to the host).
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace gen {

template <typename T>
__global__ void append_rope_write_kernel(bf16* __restrict__ qkv, const KvCacheT<T> cv, const float* __restrict__ cos_t,
                                         const float* __restrict__ sin_t, const int* __restrict__ cu_q,
                                         const int* __restrict__ seq_enc, const int* __restrict__ seq_dec,
                                         const int* __restrict__ seq_this, bf16* __restrict__ q_dec, int* __restrict__ dec_len, int B,
                                         int nh, int max_pos, int64_t ld) {
  const int kvh = cv.kvh, d = cv.d;
  const int tok = blockIdx.x;
  // an idle slot owns no token row, so no block below writes its decode length: mark it here, or the decode kernel and the
  // scatter would act on whatever length the workspace held from an earlier call (and write into the next sequence's row)
  if (tok == 0)
    for (int bb = threadIdx.x; bb < B; bb += blockDim.x)
      if (__ldg(seq_this + bb) <= 0) dec_len[bb] = -1;
  // which sequence owns this token row: the last b with cu_q[b] <= tok
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cu_q + mid) <= tok) lo = mid; else hi = mid;
  }
  const int b = lo;
  const int i = tok - __ldg(cu_q + b);
  const int n = __ldg(seq_this + b);
  if (i >= n) return;                                   // (padding rows between sequences, if the caller left any)
  const int pos = __ldg(seq_dec + b) + i;
  const bool is_decode = (n == 1) && (__ldg(seq_enc + b) <= 0);
  if (threadIdx.x == 0 && i == 0) dec_len[b] = is_decode ? pos : -1;
  if (pos < 0 || pos >= cv.max_len || pos >= max_pos) return;
  const int half = d >> 1;
  const int per_head = half >> 3;
  const int n_rope = (nh + kvh) * per_head;
  const int idx = threadIdx.x;
  bf16* row = qkv + static_cast<size_t>(tok) * ld;
  if (idx < n_rope) {
    const int head = idx / per_head;
    const int j8 = (idx % per_head) * 8;
    bf16* base = row + head * d;
    uint4 a = *reinterpret_cast<const uint4*>(base + j8);
    uint4 bb = *reinterpret_cast<const uint4*>(base + half + j8);
    rope_rotate_chunk(a, bb, cos_t, sin_t, pos, half, j8);
    *reinterpret_cast<uint4*>(base + j8) = a;
    *reinterpret_cast<uint4*>(base + half + j8) = bb;
    if (head >= nh) {
      const size_t dst = cv.offset(b, head - nh, pos);
      cv.store8(0, head - nh, dst + j8, a);
      cv.store8(0, head - nh, dst + half + j8, bb);
    } else if (is_decode) {
      bf16* dst = q_dec + static_cast<size_t>(b) * ld + head * d;
      *reinterpret_cast<uint4*>(dst + j8) = a;
      *reinterpret_cast<uint4*>(dst + half + j8) = bb;
    }
  } else {
    const int c = idx - n_rope;
    if (c >= (kvh * d) >> 3) return;
    const uint4 v = *reinterpret_cast<const uint4*>(row + (nh + kvh) * d + c * 8);
    const int head = (c * 8) / d, off = (c * 8) % d;
    cv.store8(1, head, cv.offset(b, head, pos) + off, v);
  }
}

// out[cu_q[b], :] = out_dec[b, :] for the decode rows
__global__ void append_scatter_decode_kernel(const bf16* __restrict__ out_dec, bf16* __restrict__ out, const int* __restrict__ cu_q,
                                             const int* __restrict__ dec_len, int width, int64_t ldo) {
  const int b = blockIdx.x;
  if (dec_len[b] < 0) return;
  const uint4* src = reinterpret_cast<const uint4*>(out_dec + static_cast<size_t>(b) * width);
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(cu_q[b]) * ldo);
  for (int c = threadIdx.x; c < width / 8; c += blockDim.x) dst[c] = src[c];
}
}  // namespace gen
}  // namespace b200

extern "C" int64_t b200_append_attention_workspace_bytes(int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                                         int64_t num_splits) {
  // dense decode-row q buffer [B, (nh + 2 kvh) d] bf16 | decode outputs [B, nh d] bf16 | decode lengths [B] int32 (padded) |
  // split-KV partials of the decode kernel
  const int64_t ld = (num_heads + 2 * num_kv_heads) * head_dim;
  return B * ld * 2 + B * num_heads * head_dim * 2 + ((B * 4 + 255) / 256) * 256 +
         (num_splits > 1 ? b200_decode_attention_workspace_bytes(B, num_heads, num_splits) : 0);
}

// The steps of append_attention over a checked paged view of either element type.
template <typename T>
static int append_attention_run(const KvCacheT<T>& cv, void* qkv, const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder,
                                const int32_t* seq_lens_this_time, const int32_t* cu_seqlens_q, const float* cos_table,
                                const float* sin_table, void* out, void* workspace, int64_t B, int64_t token_num,
                                int64_t max_q_len, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t num_blocks,
                                int64_t rope_positions, int64_t ldq, int64_t ldo, float softmax_scale, int64_t num_splits,
                                cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(head_dim == 64 || head_dim == 128, "append_attention: head_dim must be 64 or 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && token_num > 0 && max_q_len > 0 && num_heads % num_kv_heads == 0 && num_blocks > 0 && ldq % 8 == 0 &&
                     ldo % 8 == 0 && num_splits >= 1 && num_splits <= 64,
                 "append_attention: bad shape");
  const int64_t ld = (num_heads + 2 * num_kv_heads) * head_dim;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  bf16* q_dec = reinterpret_cast<bf16*>(ws);
  bf16* out_dec = reinterpret_cast<bf16*>(ws + B * ld * 2);
  int32_t* dec_len = reinterpret_cast<int32_t*>(ws + B * ld * 2 + B * num_heads * head_dim * 2);
  void* dec_ws = ws + B * ld * 2 + B * num_heads * head_dim * 2 + ((B * 4 + 255) / 256) * 256;
  const int threads = static_cast<int>(((num_heads + num_kv_heads) * (head_dim / 16) + (num_kv_heads * head_dim) / 8 + 31) / 32 * 32);
  B200_CHECK_ARG(threads <= 1024, "append_attention: too many heads");
  void* dec_part = num_splits > 1 ? dec_ws : nullptr;
  if (int rc = check_decode_attention("append_attention", cv, q_dec, dec_len, out_dec, dec_part, B, num_heads, ld, num_splits))
    return rc;   // before the first launch: a refused call leaves the cache untouched
  gen::append_rope_write_kernel<<<static_cast<unsigned>(token_num), threads, 0, stream>>>(
      static_cast<bf16*>(qkv), cv, cos_table, sin_table, cu_seqlens_q, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, q_dec,
      dec_len, (int)B, (int)num_heads, (int)rope_positions, ldq);
  int rc = check_launch("append_attention(rope + cache write)");
  if (rc) return rc;
  rc = launch_fa_prefill_paged(cv, qkv, out, cu_seqlens_q, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, B, max_q_len,
                               num_heads, ldq, ldo, softmax_scale, stream);
  if (rc) return rc;
  rc = launch_decode_attention(cv, q_dec, dec_len, out_dec, dec_part, B, num_heads, ld, softmax_scale, num_splits, stream);
  if (rc) return rc;
  gen::append_scatter_decode_kernel<<<static_cast<unsigned>(B), 128, 0, stream>>>(out_dec, static_cast<bf16*>(out), cu_seqlens_q,
                                                                                 dec_len, (int)(num_heads * head_dim), ldo);
  return check_launch("append_attention(scatter)");
}

extern "C" int b200_append_attention(void* qkv, void* key_cache, void* value_cache, const int32_t* seq_lens_encoder,
                                     const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time,
                                     const int32_t* cu_seqlens_q, const int32_t* block_tables, const float* cos_table,
                                     const float* sin_table, void* out, void* workspace, int64_t B, int64_t token_num,
                                     int64_t max_q_len, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                     int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t rope_positions,
                                     int64_t ldq, int64_t ldo, float softmax_scale, int64_t num_splits, cudaStream_t stream) {
  B200_CHECK_ARG(qkv && seq_lens_encoder && seq_lens_decoder && seq_lens_this_time && cu_seqlens_q && cos_table && sin_table && out &&
                     workspace,
                 "append_attention: null pointer");
  KvCache cv;
  if (int rc = paged_kv_cache(&cv, key_cache, value_cache, block_tables, num_kv_heads, head_dim, block_size, max_blocks_per_seq,
                              "append_attention"))
    return rc;
  return append_attention_run(cv, qkv, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, cos_table, sin_table,
                              out, workspace, B, token_num, max_q_len, num_heads, num_kv_heads, head_dim, num_blocks,
                              rope_positions, ldq, ldo, softmax_scale, num_splits, stream);
}

extern "C" int b200_append_attention_c8(void* qkv, void* key_cache, void* value_cache, const void* cache_k_scale,
                                        const void* cache_v_scale, const void* cache_k_out_scale, const void* cache_v_out_scale,
                                        const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder,
                                        const int32_t* seq_lens_this_time, const int32_t* cu_seqlens_q, const int32_t* block_tables,
                                        const float* cos_table, const float* sin_table, void* out, void* workspace, int64_t B,
                                        int64_t token_num, int64_t max_q_len, int64_t num_heads, int64_t num_kv_heads,
                                        int64_t head_dim, int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq,
                                        int64_t rope_positions, int64_t ldq, int64_t ldo, float softmax_scale, int64_t num_splits,
                                        cudaStream_t stream) {
  B200_CHECK_ARG(qkv && seq_lens_encoder && seq_lens_decoder && seq_lens_this_time && cu_seqlens_q && cos_table && sin_table && out &&
                     workspace,
                 "append_attention_c8: null pointer");
  KvCacheC8 cv;
  if (int rc = paged_kv_cache_c8(&cv, key_cache, value_cache, block_tables, cache_k_scale, cache_v_scale, cache_k_out_scale,
                                 cache_v_out_scale, true, true, num_kv_heads, head_dim, block_size, max_blocks_per_seq,
                                 "append_attention_c8"))
    return rc;
  return append_attention_run(cv, qkv, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, cos_table, sin_table,
                              out, workspace, B, token_num, max_q_len, num_heads, num_kv_heads, head_dim, num_blocks,
                              rope_positions, ldq, ldo, softmax_scale, num_splits, stream);
}
