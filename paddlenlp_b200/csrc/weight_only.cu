// Weight-only int8 linear layers for generation (--quant_type weight_only_int8, llm/predict/predictor.py:86,1250;
// weight_quantize / weight_only_linear under FusedMultiTransformerWeightOnly, fused_transformer_layers.py:1221-1440).
//
//   weight_quantize:  scale[n] = bf16(max_k |W[k, n]| / 127),  q[k, n] = clamp(rint(W[k, n] / scale[n]), -127, 127)
//   weight_only GEMM: y[m, n] = scale[n] * sum_k x[m, k] q[k, n] (+ bias[n]),  fp32 sums, one rounding to bf16 (or fp32 out)
//
// int8 -> bf16 is exact, so the weights are never rounded: prefill, mixed continuous-batching steps and decode steps compute
// the same y, whatever the row count and split-K.
//
// GEMM design (one persistent kernel for every M, warp-specialised, 3 warpgroups = 384 threads):
//   The operands are swapped: the weights are the wgmma A operand (64 output channels per consumer warpgroup, 128 per CTA)
//   and the tokens are the wgmma N dimension, NT = 8 ... 128 wide as the row count needs (a batch of 5 runs an n8 tile).
//   warpgroup 0     TMA producer : one thread streams int8 weight tiles (128 channels x 64 k, 8 KB) and the bf16 activation
//                                  tile (NT tokens x 64 k, K-major, 128B-swizzled) through an mbarrier ring; the weight tiles
//                                  of the first stages are requested before the PDL wait (they do not depend on the
//                                  predecessor kernel)
//   warpgroups 1,2  MMA + epilogue: each thread reads its A fragment of a k-step (two 32-bit shared loads), converts the
//                                  int8 values to bf16 in registers and issues wgmma.mma_async in the RS form (A from
//                                  registers, B = activations from shared memory); the epilogue scales each channel's fp32
//                                  sums, adds the bias, transposes [channels, tokens] through shared memory and stores bf16
//                                  [tokens, channels] boxes with TMA, or reduce-adds fp32 boxes into a workspace (split-K and
//                                  the fp32-output form).
//   K is split across CTAs when channel tiles x token tiles do not cover the SMs (every decode shape).
#include "../../include/b200nlp.h"
#include <cstring>

#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace w8 {

constexpr int BC = 128;                       // output channels per CTA (2 consumer warpgroups x 64)
constexpr int BK = 64;                        // k per pipeline stage (one 128-byte swizzle row of bf16 activations)
constexpr int W_BYTES = BC * BK;              // int8 weight tile: 16 channel groups x 4 k-steps x 128 bytes = 8 KB
constexpr int NUM_THREADS = 384;

// Packed weight layout (include/b200nlp.h): unit (g, s) = channels 8g .. 8g+7 x k 16s .. 16s+15, 128 bytes at byte offset
// (g * K/16 + s) * 128; lane l's 4 bytes at 4 l are q[16s + c][8g + l/4], q[16s + c + 1][.], q[16s + c + 8][.], q[16s + c + 9][.]
// with c = 2 (l % 4): the two bf16 pairs of the wgmma / mma.sync A fragment of row l/4.  A weight tile is one 3-D TMA box
// {128 bytes, 4 k-steps, 16 groups}.
template <int NT>
struct Cfg {
  static constexpr int X_BYTES = NT * BK * 2;                      // activation tile
  static constexpr int STAGE_BYTES = W_BYTES + X_BYTES;
  static constexpr int TC = NT < 64 ? NT : 64;                     // tokens per epilogue box
  static constexpr int BOX_BYTES = TC * 128;                       // a box: TC rows of 128 bytes (64 bf16 or 32 fp32 channels)
  static constexpr int EPI_BYTES = 2 * 2 * BOX_BYTES;              // two box buffers per consumer warpgroup
  static constexpr int STAGES_FIT = (200 * 1024 - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT < 8 ? STAGES_FIT : 8;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 256 + 1024;   // + barriers + alignment slack
  static_assert(STAGES >= 3, "pipeline too shallow");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

struct Params {
  int M, N, K;
  int num_c_tiles, num_t_tiles;
  int gm;                  // token tiles per raster group
  int split_k, kb_per_split;
  int f32_out;             // 0: bf16 C = bf16(scale * acc + bias) ; 1: fp32 workspace += scale * acc (TMA reduce-add)
  const bf16* scale;       // [N]
  const float* bias;       // [N] fp32 or nullptr (bf16 output only)
};

// d[64 x 8] (+)= A[64 x 16] * B[16 x 8]; A from registers, B K-major in shared memory (128-byte swizzle).
__device__ __forceinline__ void wgmma_m64n8k16_rs(float (&d)[4], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}
// d[64 x 16] (+)= A[64 x 16] * B[16 x 16]; A from registers, B K-major in shared memory (128-byte swizzle).
__device__ __forceinline__ void wgmma_m64n16k16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}
// d[64 x 32] (+)= A[64 x 16] * B[16 x 32]; A from registers, B K-major in shared memory (128-byte swizzle).
__device__ __forceinline__ void wgmma_m64n32k16_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// Dispatch of the RS-form wgmma on the token width NT (B operand K-major).
template <int NT>
__device__ __forceinline__ void wgmma_rs(float (&d)[NT / 2], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  if constexpr (NT == 8) wgmma_m64n8k16_rs(d, a, desc_b, accumulate);
  else if constexpr (NT == 16) wgmma_m64n16k16_rs(d, a, desc_b, accumulate);
  else if constexpr (NT == 32) wgmma_m64n32k16_rs(d, a, desc_b, accumulate);
  else if constexpr (NT == 64) wgmma_m64n64k16_rs<0>(d, a, desc_b, accumulate);
  else wgmma_m64n128k16_rs<0>(d, a, desc_b, accumulate);
}

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}

// Four int8 (the bytes of w) -> two bf16 pairs, lo = (byte 0, byte 1), hi = (byte 2, byte 3).  x + 128 goes into the low
// mantissa byte of 2^23 (the fp32 8388608 + x + 128, exact), the offset is subtracted exactly, and an integer of at most 127
// in magnitude converts to bf16 exactly.
__device__ __forceinline__ void i8x4_to_bf16(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const uint32_t u = w ^ 0x80808080u;
  const float f0 = __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7540)), 8388736.f);
  const float f1 = __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7541)), 8388736.f);
  const float f2 = __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7542)), 8388736.f);
  const float f3 = __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7543)), 8388736.f);
  lo = pack_bf16x2(f0, f1);
  hi = pack_bf16x2(f2, f3);
}

template <int N>
__device__ __forceinline__ void fence_regs(float (&acc)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

template <int NT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
w8_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
               const __grid_constant__ CUtensorMap tmY, const Params p) {
  using C = Cfg<NT>;
  constexpr int STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES, TC = C::TC, BOX_BYTES = C::BOX_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + C::EPI_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                                          // [STAGES]

  const int num_items = p.num_c_tiles * p.num_t_tiles * p.split_k;
  const int num_kb = (p.K + BK - 1) / BK;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2 * 128);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const int wg = threadIdx.x >> 7;
  if (wg == 0) {
    // ===================================== TMA producer =====================================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // The weights do not depend on the predecessor kernel: the first stages' weight tiles are requested before the PDL
      // wait, their activation tiles after it.
      int t = blockIdx.x, pre = 0;
      if (t < num_items) {
        int c_blk, t_blk;
        tile_coords(t / p.split_k, p.num_t_tiles, p.num_c_tiles, t_blk, c_blk, p.gm);
        const int kb0 = (t % p.split_k) * p.kb_per_split;
        pre = min(STAGES, min(num_kb, kb0 + p.kb_per_split) - kb0);
        for (int i = 0; i < pre; ++i) {
          mbar_arrive_expect_tx(&full_bar[i], STAGE_BYTES);
          tma_load_3d(&tmW, &full_bar[i], smem + i * STAGE_BYTES, 0, (kb0 + i) * (BK / 16), c_blk * (BC / 8));
        }
        pdl_wait();
        for (int i = 0; i < pre; ++i)
          tma_load_2d(&tmX, &full_bar[i], smem + i * STAGE_BYTES + W_BYTES, (kb0 + i) * BK, t_blk * NT);
      } else {
        pdl_wait();
      }
      uint32_t it = 0;
      for (; t < num_items; t += gridDim.x) {
        int c_blk, t_blk;
        tile_coords(t / p.split_k, p.num_t_tiles, p.num_c_tiles, t_blk, c_blk, p.gm);
        const int kb0 = (t % p.split_k) * p.kb_per_split;
        const int kb1 = min(num_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          if (it < static_cast<uint32_t>(pre)) continue;   // issued above
          const int st = static_cast<int>(it % STAGES);
          // no function call in any wait of a wgmma kernel (mbar_wait's printf): ptxas would serialise the wgmmas (C7510)
          mbar_wait_nocall(&empty_bar[st], ((it / STAGES) & 1u) ^ 1u);
          uint8_t* sW = smem + st * STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[st], STAGE_BYTES);
          tma_load_3d(&tmW, &full_bar[st], sW, 0, kb * (BK / 16), c_blk * (BC / 8));
          tma_load_2d(&tmX, &full_bar[st], sW + W_BYTES, kb * BK, t_blk * NT);
        }
      }
    }
    return;
  }

  // ===================================== MMA + epilogue =====================================
  setmaxnreg_inc<232>();
  pdl_wait();                                              // the outputs may still be read or re-zeroed by the predecessor
  const int cw = wg - 1;                                   // 64-channel half of the tile
  const int wi = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool leader = (threadIdx.x & 127) == 0;            // issues the warpgroup's epilogue stores
  const uint32_t ring = smem_u32(smem);
  const uint32_t ebuf = smem_u32(smem + STAGES * STAGE_BYTES) + cw * 2 * BOX_BYTES;
  // This thread's A-fragment words in a weight tile: channel group g = 8 cw + 2 wi + h (h = 0: fragment rows l/4, h = 1: rows
  // l/4 + 8) at k-step kk is tile row R = 4 g + kk; 128-byte swizzle: 16-byte chunk l/4 sits at (l/4) ^ (R % 8), R % 8 = 4 h + kk.
  const uint32_t a_base = (4 * (8 * cw + 2 * wi)) * 128 + 4 * (lane & 3);
  auto a_off = [&](int h, int kk) { return a_base + (4 * h + kk) * 128 + (((lane >> 2) ^ (4 * h + kk)) << 4); };
  const int r_lo = 16 * wi + (lane >> 2);                  // this thread's channels in the warpgroup: r_lo + 8 i
  const int cq = 2 * (lane & 3);                           // and tokens of each 8-column block: cq + e
  uint32_t it = 0;
  float acc[NT / 2];
  for (int t = blockIdx.x; t < num_items; t += gridDim.x) {
    int c_blk, t_blk;
    tile_coords(t / p.split_k, p.num_t_tiles, p.num_c_tiles, t_blk, c_blk, p.gm);
    const int kb0 = (t % p.split_k) * p.kb_per_split;
    const int nkb = min(num_kb, kb0 + p.kb_per_split) - kb0;
    fence_regs(acc);
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    fence_regs(acc);
    for (int i = 0; i < nkb; ++i, ++it) {
      const int st = static_cast<int>(it % STAGES);
      mbar_wait_nocall(&full_bar[st], (it / STAGES) & 1u);
      const uint32_t sW = ring + st * STAGE_BYTES;
      uint32_t a[BK / 16][4];
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        i8x4_to_bf16(ld_shared_u32(sW + a_off(0, kk)), a[kk][0], a[kk][2]);
        i8x4_to_bf16(ld_shared_u32(sW + a_off(1, kk)), a[kk][1], a[kk][3]);
      }
      const uint64_t dX = wgmma_desc_sw128(sW + W_BYTES, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) wgmma_rs<NT>(acc, a[kk], dX + ((kk * 32) >> 4), (i > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
      // The wgmmas read the A fragments from registers: they are overwritten only after these have finished.  The other
      // consumer warpgroup keeps the tensor cores busy meanwhile.
      wgmma_wait<0>();
      fence_regs(acc);
      mbar_arrive(&empty_bar[st]);
    }

    // accumulator fragment: register 4j + 2i + e holds channel r_lo + 8i, token 8j + cq + e of the tile
    const int ch0 = c_blk * BC + cw * 64;                  // first channel of the warpgroup's boxes
    if (ch0 >= p.N) continue;
    float sc[2], bs[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int ch = ch0 + r_lo + 8 * i;
      sc[i] = ch < p.N ? __bfloat162float(p.scale[ch]) : 0.f;
      bs[i] = (ch < p.N && p.bias != nullptr) ? __ldg(p.bias + ch) : 0.f;
    }
#pragma unroll
    for (int s = 0; s < NT / TC; ++s) {
      const int tok0 = t_blk * NT + s * TC;
      if (tok0 >= p.M) break;
      if (leader) tma_store_wait_read<0>();               // the previous stores have finished reading the box buffers
      named_bar_sync(1 + cw, 128);
#pragma unroll
      for (int jj = 0; jj < TC / 8; ++jj)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = s * (TC / 8) + jj, row = 8 * jj + cq + e, c = r_lo + 8 * i;
            const float v = __fmul_rn(acc[4 * j + 2 * i + e], sc[i]);
            if (p.f32_out) {                               // box h holds channels 32 h .. 32 h + 31, 128 bytes per token
              const uint32_t addr = ebuf + (c >> 5) * BOX_BYTES + row * 128 + ((((c & 31) >> 2) ^ (row & 7)) << 4) + 4 * (c & 3);
              asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v));
            } else {                                       // one box: 64 bf16 channels, 128 bytes per token
              const uint32_t addr = ebuf + row * 128 + (((c >> 3) ^ (row & 7)) << 4) + 2 * (c & 7);
              const unsigned short b = __bfloat16_as_ushort(__float2bfloat16_rn(__fadd_rn(v, bs[i])));
              asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(b));
            }
          }
      fence_proxy_async_smem();
      named_bar_sync(1 + cw, 128);
      if (leader) {
        if (p.f32_out) {
          tma_reduce_add_2d(&tmY, ebuf, ch0, tok0);
          tma_reduce_add_2d(&tmY, ebuf + BOX_BYTES, ch0 + 32, tok0);
        } else {
          tma_store_2d(&tmY, ebuf, ch0, tok0);
        }
        tma_store_commit();
      }
    }
  }
  if (leader) tma_store_wait<0>();                         // the box buffers stay allocated until the last store is done
}

// One CTA per 64 columns: column absmax, scales, then the packed bytes of the block's 8 channel groups (one 32-bit word of
// the layout per thread and step: coalesced writes).  Runs once per matrix at load time.
__global__ void __launch_bounds__(256)
quantize_kernel(const bf16* __restrict__ W, uint32_t* __restrict__ Q, bf16* __restrict__ scale, int K, int N, int64_t ldw) {
  __shared__ float red[4][64];
  __shared__ float s_scale[64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int n0 = blockIdx.x * 64;
  float m = 0.f;
  if (n0 + tx < N)
    for (int k = ty; k < K; k += 4) m = fmaxf(m, fabsf(__bfloat162float(W[static_cast<int64_t>(k) * ldw + n0 + tx])));
  red[ty][tx] = m;
  __syncthreads();
  if (ty == 0) {
    const float a = fmaxf(fmaxf(red[0][tx], red[1][tx]), fmaxf(red[2][tx], red[3][tx]));
    const bf16 s = __float2bfloat16_rn(__fdiv_rn(a, 127.0f));
    if (n0 + tx < N) scale[n0 + tx] = s;
    s_scale[tx] = __bfloat162float(s);
  }
  __syncthreads();
  const int groups = min(8, (N - n0) / 8);
  const int words_per_group = 2 * K;                       // K/16 units of 32 words
  const int64_t words = static_cast<int64_t>(groups) * words_per_group;
  uint32_t* q = Q + static_cast<int64_t>(n0 / 8) * words_per_group;
  for (int64_t w = threadIdx.x; w < words; w += blockDim.x) {
    const int g = static_cast<int>(w / words_per_group), r = static_cast<int>(w % words_per_group);
    const int lane = r & 31, c = g * 8 + (lane >> 2);
    const int k = (r >> 5) * 16 + 2 * (lane & 3);
    const float s = s_scale[c];
    const bf16* col = W + n0 + c;
    uint32_t word = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int kb = k + (b & 1) + 8 * (b >> 1);
      int v = 0;
      if (s != 0.f) {
        v = __float2int_rn(__fdiv_rn(__bfloat162float(col[static_cast<int64_t>(kb) * ldw]), s));
        v = max(-127, min(127, v));
      }
      word |= (static_cast<uint32_t>(v) & 0xFFu) << (8 * b);
    }
    q[w] = word;
  }
}

// Token tile: the narrowest wgmma N that holds M rows, at most 128 (a 64 x 256 fp32 accumulator next to the 16 A-fragment
// registers does not fit the 168 registers per thread this block size allows, and the B-operand bytes per MAC do not depend
// on N).
static int pick_nt(int64_t M) { return M <= 8 ? 8 : M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : 128; }
static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

template <int NT>
static int launch(const void* X, const void* Q, void* Y, Params p, int64_t ldx, int64_t ldy, cudaStream_t stream) {
  using C = Cfg<NT>;
  CUtensorMap tmW, tmX, tmY;
  memset(&tmY, 0, sizeof(tmY));
  int rc;
  {  // packed weights: {128 bytes, K/16 k-steps, N/8 channel groups}, box = one 128-channel x 64-k tile
    const uint64_t dims[3] = {128, static_cast<uint64_t>(p.K / 16), static_cast<uint64_t>(p.N / 8)};
    const uint64_t strides[2] = {128, static_cast<uint64_t>(p.K) * 8};
    const uint32_t box[3] = {128, BK / 16, BC / 8};
    if ((rc = encode_tmap_u8(&tmW, Q, 3, dims, strides, box)) != 0) return rc;
  }
  {  // activations [M, K], K-major: box {64 k, NT tokens}
    const uint64_t dims[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.M)}, strides[1] = {static_cast<uint64_t>(ldx) * 2};
    const uint32_t box[2] = {BK, NT};
    if ((rc = encode_tmap_bf16(&tmX, X, 2, dims, strides, box)) != 0) return rc;
  }
  {  // output [M, N]: bf16 box {64 channels, TC tokens}, fp32 box {32 channels, TC tokens}
    const uint64_t dims[2] = {static_cast<uint64_t>(p.N), static_cast<uint64_t>(p.M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldy) * (p.f32_out ? 4 : 2)};
    const uint32_t box[2] = {static_cast<uint32_t>(p.f32_out ? 32 : 64), static_cast<uint32_t>(C::TC)};
    rc = p.f32_out ? encode_tmap_f32(&tmY, Y, 2, dims, strides, box) : encode_tmap_bf16(&tmY, Y, 2, dims, strides, box);
    if (rc != 0) return rc;
  }
  auto kern = w8_gemm_kernel<NT>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(weight_only gemm smem=%d): %s", C::SMEM_BYTES, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  // Raster group: 16 token tiles share each channel column while their activations (16 NT K bf16) fit in ~18 MB of L2, 8 otherwise.
  p.gm = (16ll * NT * p.K * 2 <= (18ll << 20)) ? 16 : 8;
  const int num_items = p.num_c_tiles * p.num_t_tiles * p.split_k;
  const int ctas = min(sm_count(), num_items);
  cudaError_t e = launch_pdl(kern, dim3(ctas), dim3(NUM_THREADS), C::SMEM_BYTES, stream, tmW, tmX, tmY, p);
  if (e != cudaSuccess) {
    set_last_error("weight_only gemm launch: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  return 0;
}

// Per work item, the pipeline fill (first TMA round trip) costs about as much as streaming this many k-blocks.
constexpr int ITEM_FILL_KB = 3;

// Tiles and split of an [M, N, K] product.  split_k <= 0 chooses the split with the shortest critical path,
// waves x (k-blocks per item + ITEM_FILL_KB), preferring the smaller split on a tie.  Counting whole waves is what matters:
// "enough items for every SM" (ceil(SMs / tiles)) gives the Llama-3-8B o-projection 160 items on 132 SMs, two waves of 13
// k-blocks where 128 items make one wave of 16.
static Params plan(int64_t M, int64_t N, int64_t K, int split_k) {
  Params p = {};
  p.M = static_cast<int>(M);
  p.N = static_cast<int>(N);
  p.K = static_cast<int>(K);
  const int nt = pick_nt(M);
  p.num_c_tiles = static_cast<int>((N + BC - 1) / BC);
  p.num_t_tiles = static_cast<int>((M + nt - 1) / nt);
  const int num_kb = static_cast<int>((K + BK - 1) / BK);
  if (split_k <= 0) {
    const int64_t tiles = static_cast<int64_t>(p.num_c_tiles) * p.num_t_tiles, sms = sm_count();
    int64_t best = -1;
    split_k = 1;
    for (int s = 1; s <= num_kb && s <= 64; ++s) {
      const int kbp = (num_kb + s - 1) / s;
      const int s_eff = (num_kb + kbp - 1) / kbp;
      if (s_eff != s) continue;                            // the same split as a smaller s
      const int64_t cost = (tiles * s + sms - 1) / sms * (kbp + ITEM_FILL_KB);
      if (best < 0 || cost < best) {
        best = cost;
        split_k = s;
      }
    }
  }
  if (split_k > num_kb) split_k = num_kb;
  p.kb_per_split = (num_kb + split_k - 1) / split_k;
  p.split_k = (num_kb + p.kb_per_split - 1) / p.kb_per_split;   // no empty ranges
  return p;
}

static int run(const void* X, const void* Q, void* Y, const Params& p, int64_t ldx, int64_t ldy, cudaStream_t stream) {
  switch (pick_nt(p.M)) {
    case 8: return launch<8>(X, Q, Y, p, ldx, ldy, stream);
    case 16: return launch<16>(X, Q, Y, p, ldx, ldy, stream);
    case 32: return launch<32>(X, Q, Y, p, ldx, ldy, stream);
    case 64: return launch<64>(X, Q, Y, p, ldx, ldy, stream);
    default: return launch<128>(X, Q, Y, p, ldx, ldy, stream);
  }
}

static int check_common(const char* what, const void* X, const void* Q, const void* scale, int64_t M, int64_t N, int64_t K,
                        int64_t ldx) {
  B200_CHECK_ARG(X && Q && scale, "%s: null pointer", what);
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "%s: non-positive dimension M=%lld N=%lld K=%lld", what, (long long)M, (long long)N,
                 (long long)K);
  B200_CHECK_ARG(K % 16 == 0, "%s: K must be a multiple of 16 (got %lld)", what, (long long)K);
  B200_CHECK_ARG(N % 8 == 0, "%s: N must be a multiple of 8 (got %lld)", what, (long long)N);
  B200_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 28), "%s: dimension too large", what);
  B200_CHECK_ARG(ldx % 8 == 0 && ldx >= K, "%s: ldx must be a multiple of 8 and >= K (ldx=%lld K=%lld)", what, (long long)ldx,
                 (long long)K);
  B200_CHECK_ARG(aligned16(X) && aligned16(Q), "%s: x and the packed weight must be 16-byte aligned", what);
  return 0;
}

}  // namespace w8
}  // namespace b200

extern "C" int b200_weight_quantize_int8(const void* W, void* Q, void* scale, int64_t K, int64_t N, int64_t ldw,
                                         cudaStream_t stream) {
  using namespace b200;
  B200_CHECK_ARG(W && Q && scale, "weight_quantize: null pointer");
  B200_CHECK_ARG(K > 0 && N > 0, "weight_quantize: non-positive dimension K=%lld N=%lld", (long long)K, (long long)N);
  B200_CHECK_ARG(K % 16 == 0, "weight_quantize: K must be a multiple of 16 (got %lld)", (long long)K);
  B200_CHECK_ARG(N % 8 == 0, "weight_quantize: N must be a multiple of 8 (got %lld)", (long long)N);
  B200_CHECK_ARG(K < (1ll << 28) && N < (1ll << 31), "weight_quantize: dimension too large");
  B200_CHECK_ARG(ldw >= N, "weight_quantize: ldw must be >= N (ldw=%lld N=%lld)", (long long)ldw, (long long)N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(Q) & 3) == 0, "weight_quantize: the packed weight must be 4-byte aligned");
  w8::quantize_kernel<<<static_cast<unsigned>((N + 63) / 64), 256, 0, stream>>>(
      static_cast<const bf16*>(W), static_cast<uint32_t*>(Q), static_cast<bf16*>(scale), static_cast<int>(K), static_cast<int>(N), ldw);
  return check_launch("weight_quantize");
}

extern "C" int b200_weight_only_gemm_bf16(const void* X, const void* Q, const void* scale, const float* bias, void* C,
                                          void* workspace, int64_t M, int64_t N, int64_t K, int64_t ldx, int64_t ldc, int split_k,
                                          cudaStream_t stream) {
  using namespace b200;
  using namespace b200::w8;
  int rc;
  if ((rc = check_common("weight_only_gemm", X, Q, scale, M, N, K, ldx)) != 0) return rc;
  B200_CHECK_ARG(C != nullptr, "weight_only_gemm: null pointer");
  B200_CHECK_ARG(ldc % 8 == 0 && ldc >= N, "weight_only_gemm: ldc must be a multiple of 8 and >= N (ldc=%lld N=%lld)",
                 (long long)ldc, (long long)N);
  B200_CHECK_ARG(aligned16(C), "weight_only_gemm: C must be 16-byte aligned");
  B200_CHECK_ARG(workspace != nullptr || split_k <= 1, "weight_only_gemm: split_k=%d needs a workspace", split_k);
  B200_CHECK_ARG(!workspace || aligned16(workspace), "weight_only_gemm: the workspace must be 16-byte aligned");
  Params p = plan(M, N, K, workspace ? split_k : 1);
  p.scale = static_cast<const bf16*>(scale);
  if (p.split_k == 1) {
    p.bias = bias;
    return run(X, Q, C, p, ldx, ldc, stream);
  }
  // split-K: scaled fp32 partial sums reduce-added into the zero-on-entry workspace, then bias, one rounding, re-zeroing
  p.f32_out = 1;
  if ((rc = run(X, Q, workspace, p, ldx, N, stream)) != 0) return rc;
  return splitk_finish(static_cast<float*>(workspace), bias, C, M, N, ldc, stream);
}

extern "C" int b200_weight_only_gemm_f32(const void* X, const void* Q, const void* scale, float* workspace, int64_t M, int64_t N,
                                         int64_t K, int64_t ldx, int split_k, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::w8;
  int rc;
  if ((rc = check_common("weight_only_gemm_f32", X, Q, scale, M, N, K, ldx)) != 0) return rc;
  B200_CHECK_ARG(workspace != nullptr && aligned16(workspace), "weight_only_gemm_f32: the workspace must be non-null and 16-byte aligned");
  Params p = plan(M, N, K, split_k);
  p.scale = static_cast<const bf16*>(scale);
  p.f32_out = 1;
  return run(X, Q, workspace, p, ldx, N, stream);
}
