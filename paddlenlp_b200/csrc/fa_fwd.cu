// Causal GQA flash-attention forward on Hopper tensor cores (head_dim 64 or 128).
//
//   O = softmax(Q K^T / sqrt(d) + causal) V ,  LSE saved for the backward.
//   q [b, s, nh, d], k/v [b, s, kvh, d] (arbitrary token stride: they are views into the packed QKV projection),
//   o [b, s, nh, d] (token stride ldo), lse [b, nh, s] fp32 (natural log).
//
// Replaces F.scaled_dot_product_attention(is_causal=True) -> vendored FlashAttention-2 in the reference
// (paddlenlp/transformers/llama/fusion_ops.py:240-246; eager math llama/modeling.py:244-301).
// Rounding points: S and softmax in fp32 (scale applied to S), P rounded to bf16 before P@V, O rounded to bf16.
//
// Two kernels (b200_set_fa_fwd_impl), both with one CTA per (batch, q-head, 128-row q tile) and 128-row kv tiles (BKV):
//
// impl 2 (default), fa_fwd_wgmma_kernel: two warpgroups of 64 q rows each.
//   TMA (issued by thread 0): Q once, then each kv tile's K and V into a 2-stage ring (4-D tensor maps over the strided views,
//                          128-byte swizzle, rows past S zero-filled), K and V with their own full / empty mbarriers: K of a
//                          stage is free once S = Q K^T has run, V only once P V has, which is one tile later
//   each warpgroup:        S_j = Q K_j^T                 (SS m64n128k16, D / 16 k-steps)
//                          O += P_{j-1} V_{j-1}          (RS m64n{D}k16: the bf16-packed P registers are the A fragment, V the
//                                                         MN-major B operand), issued behind S_j, so that the softmax of tile j
//                                                         runs while the tensor cores work on the previous tile's P V
//                          masks and online softmax on S_j, then O *= corr_j once P_{j-1} V_{j-1} is done
//   The order of operations on (m, l, O) is the mma.sync kernel's: O = O corr_j + P_j V_j per tile.
// impl 1, fa_fwd_kernel: the mma.sync cross-check, and the only kernel of the paged-cache prefill of append_attention.  8 warps
//   of 16 q rows each; K/V tiles double-buffered in 128-byte-row-swizzled shared memory with cp.async; Q stays in registers as
//   mma A fragments; S, P and the O accumulator never leave the registers of the warp that owns the rows.  Four modes: plain
//   causal, FlashMask start rows, and the paged prefill over a bf16 or a uint8 cache.  Over the uint8 cache
//   (cachekv_int8_type="static") the cp.async loads fill a double-buffered staging area of cache bytes, and each tile is
//   converted into the one bf16 K and V tile as the exact integers u - 128, so ldmatrix and mma.sync run unchanged on exact
//   values; the per-head dequantise scales are applied once, o_k on the softmax scale and o_v on O.
#include <climits>

#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"
#include "kv_cache.cuh"

namespace b200 {
namespace fa {

constexpr int NW = 8;          // mma.sync kernel: warps per CTA
constexpr int BQ = 16 * NW;    // q rows per CTA (both kernels)

// kv rows per tile (both kernels).  With equal kv tiles the two kernels see the same running maxima, so P is rounded to bf16
// at the same points, and the paged prefill (mma.sync) agrees with the training forward (wgmma) to summation-order noise.
constexpr int BKV = 128;

enum Mode { DENSE = 0, MASK = 1, PAGED = 2, PAGED_C8 = 3 };

struct Params {
  const bf16* q;
  const bf16* k;
  const bf16* v;
  bf16* o;
  float* lse;         // [B, nh, S] (DENSE / MASK)
  int64_t ldq, ldk, ldv, ldo;
  int S, B, nh, kvh;
  float scale_log2;   // softmax_scale * log2(e)
  // FlashMask, causal lower-triangular form (fusion_ops.py:218-231 -> F.flashmask_attention(startend_row_indices, causal=True)):
  // mask_start[b, c] = first query row that may NOT see key column c (the end of c's packed document, llm/utils/data.py:
  // 200-204 + zero_padding_dataset.py:84-86); non-decreasing in c and > c.  Row i sees column c iff c <= i < mask_start[b, c].
  const int* mask_start;
  // PAGED (prefill half of append_attention, csrc/gpu/append_attention.cu:428-851): sequence b contributes seq_this[b] new query
  // rows (token rows cu_q[b] .. of the packed projection) at absolute positions seq_dec[b] + i and attends to cache positions
  // [0, seq_dec[b] + i] of the paged cache `kv` (k and v above are not used)
  const int* cu_q;
  const int* seq_dec;
  const int* seq_this;
  const int* seq_enc;
  KvCache kv;
  KvCacheC8 kv8;      // PAGED_C8: the uint8 cache and its scales (kv unused)
};

// With a document mask the leading kv tiles whose every column belongs to a document that ended at or before the q tile's
// first row q0 are skipped (mask_start is non-decreasing, so they form a prefix; the diagonal tile is never empty).
__device__ __forceinline__ int first_visible_kv_tile(const int* ms, int S, int q0, int n_kv, int bkv) {
  int j = 0;
  while (j < n_kv - 1 && __ldg(ms + min(j * bkv + bkv - 1, S - 1)) <= q0) ++j;
  return j;
}

// byte offset of 16-byte chunk `chunk` of row `row` in a [rows][D] bf16 tile (chunks XOR-swizzled by row & 7: conflict-free
// ldmatrix for both the plain and the transposed reads)
template <int D>
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return static_cast<uint32_t>(row * (D * 2) + ((chunk ^ (row & 7)) << 4)); }

// Shared memory of fa_fwd_kernel: Q, then two K and two V bf16 tiles; over the uint8 cache one K and one V bf16 tile and the
// staging area [2][K, V] of cache bytes (the same total).
template <int D, int MODE>
constexpr int fa_smem_bytes() {
  return MODE == PAGED_C8 ? BQ * D * 2 + 2 * BKV * D * 2 + 4 * BKV * D : BQ * D * 2 + 4 * BKV * D * 2;
}

// 16 cache bytes -> 16 bf16 (two 16-byte chunks) holding the exact u - 128
__device__ __forceinline__ void c8x16_to_bf16(const uint4& x, uint4& lo, uint4& hi) {
  const uint32_t* xi = reinterpret_cast<const uint32_t*>(&x);
  uint32_t r[8];
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    r[2 * w] = pack_bf16x2(dequant_c8<0>(xi[w]), dequant_c8<1>(xi[w]));
    r[2 * w + 1] = pack_bf16x2(dequant_c8<2>(xi[w]), dequant_c8<3>(xi[w]));
  }
  lo = make_uint4(r[0], r[1], r[2], r[3]);
  hi = make_uint4(r[4], r[5], r[6], r[7]);
}

template <int D, int MODE>
__global__ void __launch_bounds__(NW * 32, 1) fa_fwd_kernel(const Params p) {
  constexpr bool C8 = MODE == PAGED_C8;
  constexpr int CH = D / 8, CH_LOG2 = D == 128 ? 4 : 3;   // 16-byte chunks per row
  constexpr int KV_TILE_BYTES = BKV * D * 2;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + BQ * D * 2;                     // [2] K tiles ([1] over the uint8 cache)
  const uint32_t sV = sK + (C8 ? 1 : 2) * KV_TILE_BYTES;   // [2] V tiles ([1])
  const uint32_t sS = sV + KV_TILE_BYTES;                  // uint8 cache: staging [2][K, V] of BKV * D bytes

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / (p.nh / p.kvh);
  int n_rows = p.S, pos0 = 0, tok0 = batch * p.S;
  if constexpr (MODE == PAGED || MODE == PAGED_C8) {
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
  int j_lo = 0;
  if constexpr (MODE == MASK) j_lo = first_visible_kv_tile(p.mask_start + static_cast<size_t>(batch) * p.S, p.S, q0, n_kv, BKV);

  const bf16* kbase = MODE == PAGED ? p.kv.k : p.k;   // (PAGED_C8: unused)
  const bf16* vbase = MODE == PAGED ? p.kv.v : p.v;
  auto kv_row = [&](const bf16* base, int64_t ld, int c) -> const bf16* {
    if constexpr (MODE == PAGED) return base + p.kv.offset<true, D>(batch, kv_head, c);
    else return base + static_cast<size_t>(tok0 + c) * ld + kv_head * D;
  };
  auto load_kv = [&](int j, int buf) {
    if constexpr (C8) {
      constexpr int CH8 = D / 16, CH8_LOG2 = D == 128 ? 3 : 2;    // 16-byte chunks per cache row
      const uint8_t* kc = p.kv8.k;
      const uint8_t* vc = p.kv8.v;
      const uint32_t st = sS + buf * 2 * BKV * D;
      for (int i = threadIdx.x; i < BKV * CH8; i += NW * 32) {
        const int r = i >> CH8_LOG2, ch = i & (CH8 - 1), c = j * BKV + r;
        const bool ok = c < kv_total;
        const size_t off = ok ? p.kv8.offset<true, D>(batch, kv_head, c) + ch * 16 : 0;
        // rows past the sequence read as u = 0 (-128 after the conversion): masked in S, and P = 0 in P V
        cp_async_16(st + r * D + ch * 16, kc + off, ok ? 16u : 0u);
        cp_async_16(st + BKV * D + r * D + ch * 16, vc + off, ok ? 16u : 0u);
      }
      return;
    }
    for (int i = threadIdx.x; i < BKV * CH; i += NW * 32) {
      const int r = i >> CH_LOG2, ch = i & (CH - 1), c = j * BKV + r;
      const bool ok = c < kv_total;
      cp_async_16(sK + buf * KV_TILE_BYTES + swz<D>(r, ch), ok ? kv_row(kbase, p.ldk, c) + ch * 8 : kbase, ok ? 16u : 0u);
      cp_async_16(sV + buf * KV_TILE_BYTES + swz<D>(r, ch), ok ? kv_row(vbase, p.ldv, c) + ch * 8 : vbase, ok ? 16u : 0u);
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
  float scale_log2 = p.scale_log2;
  if constexpr (C8) scale_log2 *= __bfloat162float(p.kv8.k_out_scale[kv_head]);   // K = (u - 128) o_k

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
    if constexpr (C8) {
      // staging buffer `buf` -> the bf16 K and V tiles (free: the previous tile's readers passed the barrier at the loop's end)
      constexpr int CH8 = D / 16, CH8_LOG2 = D == 128 ? 3 : 2;
      const uint32_t st = sS + buf * 2 * BKV * D;
      for (int i = threadIdx.x; i < 2 * BKV * CH8; i += NW * 32) {
        const int t = i / (BKV * CH8), ii = i % (BKV * CH8);
        const int r = ii >> CH8_LOG2, ch = ii & (CH8 - 1);
        uint4 lo, hi;
        c8x16_to_bf16(ld_shared_v4(st + t * BKV * D + r * D + ch * 16), lo, hi);
        const uint32_t dst = t == 0 ? sK : sV;
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst + swz<D>(r, 2 * ch)), "r"(lo.x), "r"(lo.y), "r"(lo.z),
                     "r"(lo.w) : "memory");
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst + swz<D>(r, 2 * ch + 1)), "r"(hi.x), "r"(hi.y), "r"(hi.z),
                     "r"(hi.w) : "memory");
      }
      __syncthreads();
    }
    if (j == j_lo) {
#pragma unroll
      for (int kc = 0; kc < D / 16; ++kc) ldsm_x4(sQ + swz<D>(warp * 16 + (lane & 15), kc * 2 + (lane >> 4)), qf[kc]);
    }
    // S = Q K^T   (16 rows x BKV kv columns per warp)
    float s[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const uint32_t kb = sK + (C8 ? 0 : buf) * KV_TILE_BYTES, vb = sV + (C8 ? 0 : buf) * KV_TILE_BYTES;
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
      const float m_new = fmaxf(m[h], mx * scale_log2);
      const float corr = (m[h] == -INFINITY) ? 0.f : fast_exp2(m[h] - m_new);
      m[h] = m_new;
      // a row can be fully masked in its first tiles (documents): exp2(-inf - (-inf)) must not be evaluated
      const float neg_m = (m_new == -INFINITY) ? 0.f : -m_new;
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
        const float p0 = fast_exp2(fmaf(s[nt][2 * h], scale_log2, neg_m));
        const float p1 = fast_exp2(fmaf(s[nt][2 * h + 1], scale_log2, neg_m));
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
    float inv = 1.f / lt;
    if constexpr (C8) inv = __bfloat162float(p.kv8.v_out_scale[kv_head]) / lt;   // V = (u - 128) o_v
    bf16* orow = p.o + static_cast<size_t>(tok0 + r) * p.ldo + head * D;
#pragma unroll
    for (int dt = 0; dt < D / 8; ++dt)
      *reinterpret_cast<uint32_t*>(orow + dt * 8 + 2 * tq) = pack_bf16x2(o[dt][2 * h] * inv, o[dt][2 * h + 1] * inv);
    if constexpr (MODE == DENSE || MODE == MASK) {
      if (tq == 0) p.lse[(static_cast<size_t>(batch) * p.nh + head) * p.S + r] = (m[h] + log2f(lt)) * 0.6931471805599453f;
    }
  }
}

template <int D, int MODE>
static int launch(const Params& p, int q_rows, cudaStream_t stream) {
  constexpr int SMEM = fa_smem_bytes<D, MODE>();
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(fa_fwd_kernel<D, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("fa_fwd smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  dim3 grid(static_cast<unsigned>((q_rows + BQ - 1) / BQ), static_cast<unsigned>(p.nh), static_cast<unsigned>(p.B));
  fa_fwd_kernel<D, MODE><<<grid, NW * 32, SMEM, stream>>>(p);
  return check_launch("fa_fwd");
}

// ------------------------------------------------------------------------------------------------------------------------
// impl 2: warp-specialised wgmma kernel
// ------------------------------------------------------------------------------------------------------------------------
namespace wg {
constexpr int STAGES = 2;
constexpr int NUM_THREADS = 256;         // two warpgroups, 64 q rows each
constexpr int BLK = 128 * 64 * 2;        // one swizzled [128 rows][64 d] block of Q, K or V

// shared-memory layout at head_dim D: Q, then the K stages, then the V stages (every tile D / 64 blocks)
template <int D>
struct Layout {
  static constexpr int TILE = 128 * D * 2;
  static constexpr int OFF_Q = 0, OFF_K = TILE, OFF_V = OFF_K + STAGES * TILE, OFF_BAR = OFF_V + STAGES * TILE;
  static constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;   // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 227 * 1024, "fa_fwd_wgmma: shared memory");
};

// Compiler-level fence on registers that wgmma reads or writes asynchronously: no access may be scheduled across it.
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

template <int D, bool MASK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
fa_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const Params p) {
  using L = Layout<D>;
  constexpr int TILE = L::TILE;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* k_full = q_bar + 1;              // [STAGES] each
  uint64_t* k_empty = k_full + STAGES;
  uint64_t* v_full = k_empty + STAGES;
  uint64_t* v_empty = v_full + STAGES;

  // grid (heads, batch, q tiles): the heads of a GQA group run side by side on the same kv tiles (L2 reuse), heavy q tiles first
  const int head = blockIdx.x, batch = blockIdx.y;
  const int kv_head = head / (p.nh / p.kvh);
  const int qt = (p.S + BQ - 1) / BQ - 1 - static_cast<int>(blockIdx.z);
  const int q0 = qt * BQ;
  const int n_kv = (min(q0 + BQ, p.S) + BKV - 1) / BKV;
  int j_lo = 0;
  if constexpr (MASK) j_lo = first_visible_kv_tile(p.mask_start + static_cast<size_t>(batch) * p.S, p.S, q0, n_kv, BKV);

  if (threadIdx.x == 0) {
    mbar_init(q_bar, 1);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 256);
      mbar_init(&v_empty[i], 256);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // Thread 0 also issues the TMA loads (Q once, K_j and V_j into the ring; see the refills in the loop).  A separate producer
  // warp would make ptxas budget the registers of a 384-thread CTA, 168 per thread, and spill: O, S and P alone take 160.
  auto load_k = [&](int it) {
    const int st = it % STAGES;
    mbar_arrive_expect_tx(&k_full[st], TILE);
#pragma unroll
    for (int h = 0; h < D / 64; ++h)
      tma_load_4d(&tmK, &k_full[st], smem + L::OFF_K + st * TILE + h * BLK, h * 64, kv_head, (j_lo + it) * BKV, batch);
  };
  auto load_v = [&](int it) {
    const int st = it % STAGES;
    mbar_arrive_expect_tx(&v_full[st], TILE);
#pragma unroll
    for (int h = 0; h < D / 64; ++h)
      tma_load_4d(&tmV, &v_full[st], smem + L::OFF_V + st * TILE + h * BLK, h * 64, kv_head, (j_lo + it) * BKV, batch);
  };
  const int n_it = n_kv - j_lo;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_arrive_expect_tx(q_bar, TILE);
#pragma unroll
    for (int h = 0; h < D / 64; ++h) tma_load_4d(&tmQ, q_bar, smem + L::OFF_Q + h * BLK, h * 64, head, q0, batch);
    for (int it = 0; it < STAGES && it < n_it; ++it) {
      load_k(it);
      load_v(it);
    }
  }

  const int cw = threadIdx.x >> 7;                          // warpgroup = 64-row half of the q tile
  const int wi = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int row0 = q0 + cw * 64 + wi * 16 + g;              // q row of accumulator rows i = 0 (and + 8 for i = 1)
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sQ = sbase + L::OFF_Q + cw * 64 * 128;
  const int* ms = MASK ? p.mask_start + static_cast<size_t>(batch) * p.S : nullptr;

  // accumulator fragments (64 rows x 8 NJ columns): register 4j + 2i + e = row 16 wi + g + 8i, column 8j + 2 tq + e
  float o[D / 2];
  float s[64];
  uint32_t pa[32];    // P of the previous tile as bf16 A fragments: pa[t] = columns 8 (t / 2) + 2 tq + {0, 1} of row i = t % 2
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, corr[2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;

  auto issue_s = [&](int st) {   // S = Q K^T: both operands K-major (d contiguous)
    const uint32_t sK = sbase + L::OFF_K + st * TILE;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t off = (kk >> 2) * BLK + (kk & 3) * 32;
      wgmma_m64n128k16<0, 0>(s, wgmma_desc_sw128(sQ + off, 16, 1024), wgmma_desc_sw128(sK + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int st) {  // O += P V: B = V, MN-major (d contiguous), k = 16 kv rows = 2048 bytes
    const uint32_t sV = sbase + L::OFF_V + st * TILE;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BKV / 16; ++k) {
      if constexpr (D == 128) wgmma_m64n128k16_rs<1>(o, pa + 4 * k, wgmma_desc_sw128(sV + k * 2048, BLK, 1024), 1u);
      else wgmma_m64n64k16_rs<1>(o, pa + 4 * k, wgmma_desc_sw128(sV + k * 2048, BLK, 1024), 1u);
    }
    wgmma_commit();
  };
  // masks and online softmax of kv tile j: s <- P (fp32), m, l updated, corr = the factor O must be scaled by before P V
  auto softmax = [&](int j) {
    // causal: only the diagonal tile (q tiles and kv tiles are both 128 rows, aligned); FlashMask: only tiles whose first
    // column's document ends inside or before the q tile
    const bool need_causal = j * BKV + BKV - 1 > q0 + cw * 64;
    bool need_mask = false;
    if constexpr (MASK) need_mask = __ldg(ms + j * BKV) <= q0 + BQ - 1;
    if (need_causal || need_mask) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = j * BKV + 8 * jj + 2 * tq + e;
          int start = INT_MAX;
          if constexpr (MASK) {
            if (need_mask && c < p.S) start = __ldg(ms + c);
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int r = row0 + 8 * i;
            if (c > r || r >= start) s[4 * jj + 2 * i + e] = -INFINITY;
          }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[i], mx * p.scale_log2);
      corr[i] = (m[i] == -INFINITY) ? 0.f : fast_exp2(m[i] - m_new);
      m[i] = m_new;
      // a row can be fully masked in its first tiles (documents): exp2(-inf - (-inf)) must not be evaluated
      const float neg_m = (m_new == -INFINITY) ? 0.f : -m_new;
      float rs = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const float p0 = fast_exp2(fmaf(s[4 * jj + 2 * i], p.scale_log2, neg_m));
        const float p1 = fast_exp2(fmaf(s[4 * jj + 2 * i + 1], p.scale_log2, neg_m));
        rs += p0 + p1;
        s[4 * jj + 2 * i] = p0;
        s[4 * jj + 2 * i + 1] = p1;
      }
      l[i] = l[i] * corr[i] + rs;
    }
  };
  auto rescale_and_pack = [&]() {
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        o[4 * jj + 2 * i] *= corr[i];
        o[4 * jj + 2 * i + 1] *= corr[i];
      }
#pragma unroll
    for (int t = 0; t < 32; ++t) pa[t] = pack_bf16x2(s[2 * t], s[2 * t + 1]);
  };

  mbar_wait_nocall(q_bar, 0);
  mbar_wait_nocall(&k_full[0], 0);
  issue_s(0);
  wgmma_wait<0>();
  reg_fence(s);
  mbar_arrive(&k_empty[0]);
  softmax(j_lo);
  rescale_and_pack();
  int it = 0;
  for (int j = j_lo + 1; j < n_kv; ++j) {
    ++it;
    const int st = it % STAGES, ps = (it - 1) % STAGES;
    if (threadIdx.x == 0) {
      // refills: K_{it+1} into the stage of tile it - 1 once both warpgroups have run S_{it-1}; V_it into the stage of tile
      // it - 2 once both have run P_{it-2} V_{it-2} (one iteration ahead of their use either way)
      static_assert(STAGES == 2, "fa_fwd_wgmma: refill schedule");
      if (it + 1 < n_it) {
        mbar_wait_nocall(&k_empty[ps], ((it - 1) / STAGES) & 1);
        load_k(it + 1);
      }
      if (it >= STAGES) {
        mbar_wait_nocall(&v_empty[st], ((it - 2) / STAGES) & 1);
        load_v(it);
      }
    }
    mbar_wait_nocall(&k_full[st], (it / STAGES) & 1);
    issue_s(st);
    mbar_wait_nocall(&v_full[ps], ((it - 1) / STAGES) & 1);
    issue_pv(ps);
    wgmma_wait<1>();               // S_j is done; P_{j-1} V_{j-1} may still run
    reg_fence(s);
    mbar_arrive(&k_empty[st]);
    softmax(j);
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(s);                  // pa is rewritten from s only after the wgmma reading it has finished
    mbar_arrive(&v_empty[ps]);
    rescale_and_pack();
  }
  {
    const int st = it % STAGES;
    mbar_wait_nocall(&v_full[st], (it / STAGES) & 1);
    issue_pv(st);
    wgmma_wait<0>();
    reg_fence(o);
  }

  // epilogue: O / l -> bf16 straight from the accumulator ; LSE
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float lt = l[i];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const int r = row0 + 8 * i;
    if (r >= p.S) continue;
    const float inv = 1.f / lt;
    bf16* orow = p.o + static_cast<size_t>(batch * p.S + r) * p.ldo + head * D;
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj)
      *reinterpret_cast<uint32_t*>(orow + jj * 8 + 2 * tq) = pack_bf16x2(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
    if (tq == 0) p.lse[(static_cast<size_t>(batch) * p.nh + head) * p.S + r] = (m[i] + log2f(lt)) * 0.6931471805599453f;
  }
}

template <int D, bool MASK>
static int launch(const CUtensorMap (&tm)[3], const Params& p, cudaStream_t stream) {
  constexpr int SMEM_BYTES = Layout<D>::SMEM_BYTES;
  auto kern = fa_fwd_wgmma_kernel<D, MASK>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      set_last_error("fa_fwd_wgmma smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  const dim3 grid(static_cast<unsigned>(p.nh), static_cast<unsigned>(p.B), static_cast<unsigned>((p.S + BQ - 1) / BQ));
  kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], p);
  return check_launch("fa_fwd_wgmma");
}
}  // namespace wg

}  // namespace fa

// Prefill half of append_attention: causal attention of the NEW token rows of every prompt / prompt-chunk sequence over its paged
// cache `kv` (cached prefix + the rows themselves, already appended).  qkv: packed projection [token_num, ldq] (q heads first,
// rotated); out [token_num, ldo].  max_q_len bounds seq_lens_this_time (grid size).  kv.d is 64 or 128 (checked by the caller).
template <typename T>
int launch_fa_prefill_paged(const KvCacheT<T>& kv, const void* qkv, void* out, const int32_t* cu_seqlens_q,
                            const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time,
                            int64_t B, int64_t max_q_len, int64_t num_heads, int64_t ldq, int64_t ldo, float softmax_scale,
                            cudaStream_t stream) {
  using namespace fa;
  Params p = {};
  p.q = static_cast<const bf16*>(qkv);
  p.o = static_cast<bf16*>(out);
  p.ldq = ldq; p.ldo = ldo;
  p.S = static_cast<int>(max_q_len); p.B = static_cast<int>(B); p.nh = static_cast<int>(num_heads);
  p.kvh = kv.kvh;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.cu_q = cu_seqlens_q; p.seq_dec = seq_lens_decoder; p.seq_this = seq_lens_this_time; p.seq_enc = seq_lens_encoder;
  if constexpr (sizeof(T) == 1) {
    p.kv8 = kv;
    if (kv.d == 64) return launch<64, PAGED_C8>(p, static_cast<int>(max_q_len), stream);
    return launch<128, PAGED_C8>(p, static_cast<int>(max_q_len), stream);
  } else {
    p.kv = kv;
    if (kv.d == 64) return launch<64, PAGED>(p, static_cast<int>(max_q_len), stream);
    return launch<128, PAGED>(p, static_cast<int>(max_q_len), stream);
  }
}
template int launch_fa_prefill_paged(const KvCache&, const void*, void*, const int32_t*, const int32_t*, const int32_t*,
                                     const int32_t*, int64_t, int64_t, int64_t, int64_t, int64_t, float, cudaStream_t);
template int launch_fa_prefill_paged(const KvCacheC8&, const void*, void*, const int32_t*, const int32_t*, const int32_t*,
                                     const int32_t*, int64_t, int64_t, int64_t, int64_t, int64_t, float, cudaStream_t);

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
  {
    // TMA (impl 2) and cp.async (impl 1) address rows in 16-byte units
    const void* ptrs[4] = {q, k, v, o};
    const char* names[4] = {"q", "k", "v", "o"};
    for (int i = 0; i < 4; ++i)
      B200_CHECK_ARG((reinterpret_cast<uintptr_t>(ptrs[i]) & 15) == 0, "fa_fwd: %s must be 16-byte aligned (got %p)", names[i], ptrs[i]);
  }
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
  if (fa_fwd_impl() == 1) {
    const int rows = static_cast<int>(S);
    if (head_dim == 64) return mask_start_rows ? launch<64, MASK>(p, rows, stream) : launch<64, DENSE>(p, rows, stream);
    return mask_start_rows ? launch<128, MASK>(p, rows, stream) : launch<128, DENSE>(p, rows, stream);
  }
  CUtensorMap tm[3];
  int rc;
  if ((rc = make_bf16_map(&tm[0], q, B, S, num_heads, head_dim, ldq, BQ)) != 0) return rc;
  if ((rc = make_bf16_map(&tm[1], k, B, S, num_kv_heads, head_dim, ldk, BKV)) != 0) return rc;
  if ((rc = make_bf16_map(&tm[2], v, B, S, num_kv_heads, head_dim, ldv, BKV)) != 0) return rc;
  if (head_dim == 64) return mask_start_rows ? wg::launch<64, true>(tm, p, stream) : wg::launch<64, false>(tm, p, stream);
  return mask_start_rows ? wg::launch<128, true>(tm, p, stream) : wg::launch<128, false>(tm, p, stream);
}
