// Causal GQA flash-attention forward on Hopper tensor cores (mma.sync m16n8k16, head_dim 64 or 128).
//
//   O = softmax(Q K^T / sqrt(d) + causal) V ,  LSE saved for the backward.
//   q [b, s, nh, d], k/v [b, s, kvh, d] (arbitrary token stride: they are views into the packed QKV projection),
//   o [b, s, nh, d] contiguous, lse [b, nh, s] fp32 (natural log).
//
// Replaces F.scaled_dot_product_attention(is_causal=True) -> vendored FlashAttention-2 in the reference
// (paddlenlp/transformers/llama/fusion_ops.py:240-246; eager math llama/modeling.py:244-301).
// Rounding points: S and softmax in fp32 (scale applied to S), P rounded to bf16 before P@V, O rounded to bf16.
//
// One CTA = one (batch, q-head, BQ-row q tile), NW warps of 16 q rows each (BQ = 16 NW; b200_set_fa_fwd_impl: 2 = 128 rows,
// 1 = 64 rows).  K/V tiles are double-buffered in 128-byte-row-swizzled shared memory with cp.async; Q stays in
// registers as mma A fragments; S, P and the O accumulator never leave the registers of the warp that owns the rows.
// Three modes: plain causal, FlashMask start rows, and the paged-cache prefill of append_attention; each for head_dim D = 128
// and D = 64.  At D = 64 a K/V row is 128 bytes (one swizzle row), and the Q fragments and the O accumulator halve; K/V tiles
// are 64 rows high at D = 128 and 128 rows at D = 64 (KV_ROWS).
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace fa {

// kv rows per tile.  At D = 64 a 128-row tile holds as many S registers as the 64-row tile holds O registers at D = 128, and
// halves the barriers and softmax rescales per kv row: 0.35 against 0.43 ms at (1, 4096, 32 / 8), 0.17 against 0.21 ms at
// (4, 2048, 14 / 2), 0.11 against 0.13 ms at (1, 2048, 32 / 4) (tools/fa_bench.py, H100 80GB HBM3, 700 W; DESIGN.md section 5).
template <int D>
constexpr int KV_ROWS = 64;
template <>
constexpr int KV_ROWS<64> = 128;

enum Mode { DENSE = 0, MASK = 1, PAGED = 2 };

struct Params {
  const bf16* q;
  const bf16* k;
  const bf16* v;
  bf16* o;
  float* lse;         // [B, nh, S] (DENSE / MASK)
  int64_t ldq, ldk, ldv, ldo;
  int S, B, nh, kvh;
  float scale_log2;   // (1/sqrt(d)) * log2(e)
  // FlashMask, causal lower-triangular form (fusion_ops.py:218-231 -> F.flashmask_attention(startend_row_indices, causal=True)):
  // mask_start[b, c] = first query row that may NOT see key column c (the end of c's packed document, llm/utils/data.py:
  // 200-204 + zero_padding_dataset.py:84-86); non-decreasing in c and > c.  Row i sees column c iff c <= i < mask_start[b, c].
  const int* mask_start;
  // PAGED (prefill half of append_attention, csrc/gpu/append_attention.cu:428-851): sequence b contributes seq_this[b] new query
  // rows (token rows cu_q[b] .. of the packed projection) at absolute positions seq_dec[b] + i and attends to cache positions
  // [0, seq_dec[b] + i] of its pages; key/value caches [num_blocks, kvh, block_size, D]
  const int* cu_q;
  const int* seq_dec;
  const int* seq_this;
  const int* seq_enc;
  const int* block_tables;
  int max_blocks, block_size;
};

// byte offset of 16-byte chunk `chunk` of row `row` in a [rows][D] bf16 tile (chunks XOR-swizzled by row & 7: conflict-free
// ldmatrix for both the plain and the transposed reads)
template <int D>
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return static_cast<uint32_t>(row * (D * 2) + ((chunk ^ (row & 7)) << 4)); }

template <int D, int NW, int MODE>
__global__ void __launch_bounds__(NW * 32, 1) fa_fwd_kernel(const Params p) {
  constexpr int BQ = 16 * NW;
  constexpr int CH = D / 8, CH_LOG2 = D == 128 ? 4 : 3;   // 16-byte chunks per row
  constexpr int BKV = KV_ROWS<D>;
  constexpr int KV_TILE_BYTES = BKV * D * 2;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + BQ * D * 2;            // [2] K tiles
  const uint32_t sV = sK + 2 * KV_TILE_BYTES;     // [2] V tiles

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / (p.nh / p.kvh);
  int n_rows = p.S, pos0 = 0, tok0 = batch * p.S;
  if constexpr (MODE == PAGED) {
    n_rows = p.seq_this[batch];
    // decode rows (one new token on top of a cache, no prompt) belong to the decode kernel; idle slots to nobody
    if (n_rows <= 0 || (n_rows == 1 && p.seq_enc[batch] <= 0)) return;
    pos0 = p.seq_dec[batch];
    tok0 = p.cu_q[batch];
  }
  const int qt = (n_rows + BQ - 1) / BQ - 1 - static_cast<int>(blockIdx.x);   // heavy tiles first
  if (qt < 0) return;
  const int q0 = qt * BQ;
  const int kv_total = pos0 + n_rows;                             // kv positions that exist
  const int kv_end = pos0 + min(q0 + BQ, n_rows);                 // kv positions the tile's last row can see
  const int n_kv = (kv_end + BKV - 1) / BKV;
  // With a document mask the leading kv tiles whose every column belongs to a document that ended at or before this q tile
  // are skipped (mask_start is non-decreasing, so they form a prefix; the diagonal tile is never empty).
  int j_lo = 0;
  if constexpr (MODE == MASK) {
    const int* ms = p.mask_start + static_cast<size_t>(batch) * p.S;
    while (j_lo < n_kv - 1 && __ldg(ms + min(j_lo * BKV + BKV - 1, p.S - 1)) <= q0) ++j_lo;
  }

  auto kv_row = [&](const bf16* base, int64_t ld, int c) -> const bf16* {
    if constexpr (MODE == PAGED) {
      const int page = __ldg(p.block_tables + static_cast<size_t>(batch) * p.max_blocks + c / p.block_size);
      return base + ((static_cast<size_t>(page) * p.kvh + kv_head) * p.block_size + c % p.block_size) * D;
    } else {
      return base + static_cast<size_t>(tok0 + c) * ld + kv_head * D;
    }
  };
  auto load_kv = [&](int j, int buf) {
    for (int i = threadIdx.x; i < BKV * CH; i += NW * 32) {
      const int r = i >> CH_LOG2, ch = i & (CH - 1), c = j * BKV + r;
      const bool ok = c < kv_total;
      cp_async_16(sK + buf * KV_TILE_BYTES + swz<D>(r, ch), ok ? kv_row(p.k, p.ldk, c) + ch * 8 : p.k, ok ? 16u : 0u);
      cp_async_16(sV + buf * KV_TILE_BYTES + swz<D>(r, ch), ok ? kv_row(p.v, p.ldv, c) + ch * 8 : p.v, ok ? 16u : 0u);
    }
  };
  for (int i = threadIdx.x; i < BQ * CH; i += NW * 32) {
    const int r = i >> CH_LOG2, ch = i & (CH - 1);
    const bool ok = q0 + r < n_rows;
    cp_async_16(sQ + swz<D>(r, ch), ok ? p.q + static_cast<size_t>(tok0 + q0 + r) * p.ldq + head * D + ch * 8 : p.q, ok ? 16u : 0u);
  }
  load_kv(j_lo, 0);
  cp_async_commit();

  const int g = lane >> 2, tq = lane & 3;
  const int row_a = q0 + warp * 16 + g;                 // tile rows of this thread: row_a and row_a + 8
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  uint32_t qf[D / 16][4];

  for (int j = j_lo; j < n_kv; ++j) {
    const int buf = (j - j_lo) & 1;
    if (j + 1 < n_kv) {
      load_kv(j + 1, buf ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == j_lo) {
#pragma unroll
      for (int kc = 0; kc < D / 16; ++kc) ldsm_x4(sQ + swz<D>(warp * 16 + (lane & 15), kc * 2 + (lane >> 4)), qf[kc]);
    }
    // S = Q K^T   (16 rows x 64 kv columns per warp)
    float s[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const uint32_t kb = sK + buf * KV_TILE_BYTES, vb = sV + buf * KV_TILE_BYTES;
#pragma unroll
    for (int kc = 0; kc < D / 16; ++kc) {
#pragma unroll
      for (int np = 0; np < BKV / 16; ++np) {
        uint32_t b[4];
        ldsm_x4(kb + swz<D>(np * 16 + (lane & 7) + ((lane >> 4) << 3), kc * 2 + ((lane >> 3) & 1)), b);
        mma_bf16_16816(s[2 * np], qf[kc], b[0], b[1]);
        mma_bf16_16816(s[2 * np + 1], qf[kc], b[2], b[3]);
      }
    }
    // masks: causal (kv position > query position), FlashMask (query row >= mask_start of the column)
    const int c_base = j * BKV + 2 * tq;
    const bool need_causal = j * BKV + BKV - 1 > pos0 + q0 + warp * 16;
    bool need_mask = false;
    if constexpr (MODE == MASK) need_mask = __ldg(p.mask_start + static_cast<size_t>(batch) * p.S + j * BKV) <= q0 + BQ - 1;
    if (need_causal || need_mask) {
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = c_base + nt * 8 + (e & 1);
          const int r = row_a + (e >> 1) * 8;
          bool dead = c > pos0 + r;
          if constexpr (MODE == MASK) {
            if (!dead && c < p.S) dead = r >= __ldg(p.mask_start + static_cast<size_t>(batch) * p.S + c);
          }
          if (dead) s[nt][e] = -INFINITY;
        }
    }
    // online softmax (two rows per thread; a row's BKV columns live in the 4 threads of a quad)
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) mx = fmaxf(mx, fmaxf(s[nt][2 * h], s[nt][2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx * p.scale_log2);
      const float corr = (m[h] == -INFINITY) ? 0.f : fast_exp2(m[h] - m_new);
      m[h] = m_new;
      // a row can be fully masked in its first tiles (documents): exp2(-inf - (-inf)) must not be evaluated
      const float neg_m = (m_new == -INFINITY) ? 0.f : -m_new;
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
        const float p0 = fast_exp2(fmaf(s[nt][2 * h], p.scale_log2, neg_m));
        const float p1 = fast_exp2(fmaf(s[nt][2 * h + 1], p.scale_log2, neg_m));
        rs += p0 + p1;
        pa[nt >> 1][(nt & 1) * 2 + h] = pack_bf16x2(p0, p1);
      }
      l[h] = l[h] * corr + rs;
#pragma unroll
      for (int dt = 0; dt < D / 8; ++dt) { o[dt][2 * h] *= corr; o[dt][2 * h + 1] *= corr; }
    }
    // O += P V
#pragma unroll
    for (int kc = 0; kc < BKV / 16; ++kc) {
#pragma unroll
      for (int dp = 0; dp < D / 16; ++dp) {
        uint32_t b[4];
        ldsm_x4_t(vb + swz<D>(kc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4)), b);
        mma_bf16_16816(o[2 * dp], pa[kc], b[0], b[1]);
        mma_bf16_16816(o[2 * dp + 1], pa[kc], b[2], b[3]);
      }
    }
    __syncthreads();   // the buffer is refilled by the next iteration's prefetch
  }
  // epilogue: O / l -> bf16 ; LSE
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const int r = row_a + 8 * h;
    if (r >= n_rows) continue;
    const float inv = 1.f / lt;
    bf16* orow = p.o + static_cast<size_t>(tok0 + r) * p.ldo + head * D;
#pragma unroll
    for (int dt = 0; dt < D / 8; ++dt)
      *reinterpret_cast<uint32_t*>(orow + dt * 8 + 2 * tq) = pack_bf16x2(o[dt][2 * h] * inv, o[dt][2 * h + 1] * inv);
    if constexpr (MODE != PAGED) {
      if (tq == 0) p.lse[(static_cast<size_t>(batch) * p.nh + head) * p.S + r] = (m[h] + log2f(lt)) * 0.6931471805599453f;
    }
  }
}

template <int D, int NW, int MODE>
static int launch(const Params& p, int q_rows, cudaStream_t stream) {
  constexpr int SMEM = 16 * NW * D * 2 + 4 * KV_ROWS<D> * D * 2;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(fa_fwd_kernel<D, NW, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("fa_fwd smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  dim3 grid(static_cast<unsigned>((q_rows + 16 * NW - 1) / (16 * NW)), static_cast<unsigned>(p.nh), static_cast<unsigned>(p.B));
  fa_fwd_kernel<D, NW, MODE><<<grid, NW * 32, SMEM, stream>>>(p);
  return check_launch("fa_fwd");
}

}  // namespace fa

// Prefill half of append_attention: causal attention of the NEW token rows of every prompt / prompt-chunk sequence over its paged
// cache (cached prefix + the rows themselves, already appended).  qkv: packed projection [token_num, ldq] (q heads first, rotated);
// key / value caches [num_blocks, kvh, block_size, head_dim]; out [token_num, ldo].  max_q_len bounds seq_lens_this_time (grid
// size).  head_dim is 64 or 128 (checked by the caller).
int launch_fa_prefill_paged(const void* qkv, const void* key_cache, const void* value_cache, void* out, const int32_t* cu_seqlens_q,
                            const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time,
                            const int32_t* block_tables, int64_t B, int64_t token_num, int64_t max_q_len, int64_t num_heads,
                            int64_t num_kv_heads, int64_t head_dim, int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq, int64_t ldq,
                            int64_t ldo, float softmax_scale, cudaStream_t stream) {
  using namespace fa;
  (void)token_num; (void)num_blocks;
  Params p = {};
  p.q = static_cast<const bf16*>(qkv);
  p.k = static_cast<const bf16*>(key_cache);
  p.v = static_cast<const bf16*>(value_cache);
  p.o = static_cast<bf16*>(out);
  p.ldq = ldq; p.ldo = ldo;
  p.S = static_cast<int>(max_q_len); p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads);
  p.kvh = static_cast<int>(num_kv_heads);
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.cu_q = cu_seqlens_q; p.seq_dec = seq_lens_decoder; p.seq_this = seq_lens_this_time; p.seq_enc = seq_lens_encoder;
  p.block_tables = block_tables;
  p.max_blocks = static_cast<int>(max_blocks_per_seq); p.block_size = static_cast<int>(block_size);
  if (head_dim == 64) return launch<64, 8, PAGED>(p, static_cast<int>(max_q_len), stream);
  return launch<128, 8, PAGED>(p, static_cast<int>(max_q_len), stream);
}

}  // namespace b200

extern "C" int b200_fa_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int64_t B, int64_t S,
                           int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk,
                           int64_t ldv, int64_t ldo, float softmax_scale, cudaStream_t stream) {
  return b200_fa_fwd_flashmask(q, k, v, o, lse, nullptr, B, S, num_heads, num_kv_heads, head_dim, ldq, ldk, ldv, ldo,
                               softmax_scale, stream);
}

extern "C" int b200_fa_fwd_flashmask(const void* q, const void* k, const void* v, void* o, float* lse,
                                     const int32_t* mask_start_rows, int64_t B, int64_t S, int64_t num_heads,
                                     int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv,
                                     int64_t ldo, float softmax_scale, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::fa;
  B200_CHECK_ARG(q && k && v && o && lse, "fa_fwd: null pointer");
  B200_CHECK_ARG(head_dim == 64 || head_dim == 128, "fa_fwd: head_dim must be 64 or 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && S > 0 && num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0,
                 "fa_fwd: bad shape B=%lld S=%lld nh=%lld kvh=%lld", (long long)B, (long long)S, (long long)num_heads,
                 (long long)num_kv_heads);
  B200_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "fa_fwd: token strides must be multiples of 8");
  Params p = {};
  p.q = static_cast<const bf16*>(q);
  p.k = static_cast<const bf16*>(k);
  p.v = static_cast<const bf16*>(v);
  p.o = static_cast<bf16*>(o);
  p.lse = lse;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.S = static_cast<int>(S); p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads);
  p.kvh = static_cast<int>(num_kv_heads);
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.mask_start = mask_start_rows;
  const int rows = static_cast<int>(S);
  if (head_dim == 64) {
    if (fa_fwd_impl() == 1)
      return mask_start_rows ? launch<64, 4, MASK>(p, rows, stream) : launch<64, 4, DENSE>(p, rows, stream);
    return mask_start_rows ? launch<64, 8, MASK>(p, rows, stream) : launch<64, 8, DENSE>(p, rows, stream);
  }
  if (fa_fwd_impl() == 1)
    return mask_start_rows ? launch<128, 4, MASK>(p, rows, stream) : launch<128, 4, DENSE>(p, rows, stream);
  return mask_start_rows ? launch<128, 8, MASK>(p, rows, stream) : launch<128, 8, DENSE>(p, rows, stream);
}
