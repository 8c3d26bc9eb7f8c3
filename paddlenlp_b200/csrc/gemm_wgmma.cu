// bf16 GEMM on Hopper tensor cores (wgmma.mma_async, accumulators in registers, operands staged by TMA).
//
//   C[M,N] (+)= op(A)[M,K] * op(B)[K,N] (+ bias[N])      bf16 in, fp32 accumulate, one rounding to bf16
//   C_f32[M,N] (+)= op(A)[M,K] * op(B)[K,N]              the same, fp32 out, no rounding (fp32 weight gradients).
//
// Replaces the cuBLAS(Lt) calls under paddle `nn.Linear` on the Llama/Qwen2 hot path
// (reference: paddlenlp/transformers/llama/modeling.py:771-799 q/k/v/o, :627-630 gate/up/down, :1894-1921 lm_head;
//  weights are stored [in,out] = "B is [K,N] row-major" = MN-major B operand) and the dX / dW GEMMs of their backward.
//
// Design (one persistent kernel, warp-specialised, 3 warpgroups = 384 threads, 128x256 output tiles):
//   warpgroup 0     TMA producer   : one thread streams A (128 x 64) and B (64 x 256) k-blocks into a 4-stage ring of
//                                    128B-swizzled shared memory (48 KB per stage); its registers go to the consumers
//   warpgroups 1,2  MMA + epilogue : each owns 64 rows of the tile: wgmma m64n256k16 x 4 per k-block, fp32 accumulators in
//                                    128 registers per thread, the four wgmmas of a k-block issued back to back; a
//                                    k-block's stage is released once the next block's wgmmas are in flight; the epilogue
//                                    (+bias, +C_old | +residual, SwiGLU forms) stages bf16 64 x 64 boxes in shared memory and
//                                    stores them with TMA (C_old / residual / gate|up prefetched into L2 during the tile's
//                                    last k-blocks); fp32 outputs leave as 64 x 32 fp32 boxes through the same buffers,
//                                    stored or reduce-added by TMA; split-K adds its fp32 partial sums from the registers
//                                    into L2
//   Operand majors: both K-major (contraction dim contiguous) and MN-major operands are fed straight from their
//   row-major global layout through TMA (wgmma reads either major for 16-bit types); no transposes are materialised.
#include "../../include/b200nlp.h"
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace gemm {

constexpr int BN = 256;   // tile columns (wgmma N)
constexpr int BK = 64;    // K per pipeline stage (= one 128-byte swizzle row of bf16)
constexpr int B_BYTES = BN * BK * 2;              // 32 KB
constexpr int EPI_BOX = 64;                       // epilogue TMA box: 64 rows x 64 columns (one 128-byte swizzle row wide)
constexpr int EPI_BOX_BYTES = EPI_BOX * EPI_BOX * 2;   // 8 KB
constexpr int EPI_BOX_F32 = 32;                   // fp32 epilogue box: 64 rows x 32 columns, also 8 KB

// NWG consumer warpgroups of 64 rows each.  NWG = 2 (128-row tiles) for the training shapes; NWG = 1 (64-row tiles) for the
// decode step's M <= 64 token rows, where the kernel is a weight stream: 8 KB of activations and 32 KB of weights per stage,
// five stages in flight, no warpgroup computing padding rows.
template <int NWG>
struct Tile {
  static constexpr int BM = 64 * NWG;
  static constexpr int NUM_THREADS = 128 * (NWG + 1);
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = NWG == 2 ? 4 : 5;
  // two 64 x 64 bf16 output boxes per consumer warpgroup for the shared-memory epilogue
  static constexpr int EPI_BYTES = NWG * 2 * EPI_BOX_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 256 + 1024;   // + barriers + alignment slack (<= 227 KB)
};
static int tile_wgs(int64_t M) { return M <= 64 ? 1 : 2; }

struct Params {
  int M, N, K;
  int num_m_tiles, num_n_tiles;
  int epi_mode;            // 0: C = acc ; 1: C = bf16(C_old + acc) ; 2: C = bf16(bf16(acc) + R) ; 3: ws += acc (fp32 split-K)
                           // 4: gate|up GEMM + SwiGLU: a 256-column tile = 128 gate columns | the 128 up columns of the same
                           //    channels; aux (if set) gets gate and up (bf16, their [M, 2I] positions), out2 gets
                           //    m = bf16(silu(gate) * up) [M, I]
                           // 5: down-proj dX GEMM + SwiGLU backward: acc = d(m) tile; aux = saved gate|up [M, 2I];
                           //    C = [d(gate) | d(up)] [M, 2I]
                           // 6: C_f32 = acc ; 7: C_f32 += acc (fp32 output through tmC, no bias: weight gradients)
  int swiglu_inter;        // modes 4, 5: I (the up half starts at column I)
  int gm;                  // m-tiles per raster group (tile_coords)
  int split_k;             // work items per output tile (K is cut into split_k ranges of kb_per_split k-blocks)
  int kb_per_split;
  const float* bias;       // [N] fp32 or nullptr
  bf16* c;                 // output (modes 0, 1, 2, 5; mode 4: m)
  int64_t ldc;
  const bf16* r;           // mode 2: residual
  int64_t ldr;
  bf16* aux;               // mode 4: gate|up output (nullable); mode 5: saved gate|up input
  int64_t ld_aux;
  float* ws;               // mode 3: fp32 [M, N] accumulation buffer; modes 6, 7: the fp32 output (leading dimension ldc)
};

// Compiler-level fence on the accumulator registers (wgmma reads and writes them asynchronously): no access to them may be
// scheduled across it.
__device__ __forceinline__ void fence_acc(float (&acc)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

// ---- shared-memory epilogue (every mode but split-K) ----
// A consumer warpgroup's 64 x 256 accumulator tile leaves as 64 x 64 bf16 boxes.  The warpgroup writes a box into one of its
// two 8 KB buffers in the 128B-swizzled TMA layout, one thread stores it with cp.async.bulk.tensor, and the warpgroup goes on
// to the next box, or to the next tile's wgmmas, while the store drains.  TMA drops rows >= M and columns past the tensor
// map's width.  The global loads of a box's inputs (C_old, residual, saved gate|up) are all issued before its first use:
// no store to global memory sits between them any more.
//
// Address of this thread's bf16 pair in row r, columns 8 jj + 2 (lane % 4) + {0, 1}, of a box buffer: 16-byte chunk jj of row r
// sits at chunk jj ^ (r % 8).  A warp's 8 rows then hit 8 different chunks: the stores are free of bank conflicts.
__device__ __forceinline__ uint32_t epi_slot(uint32_t buf, int r, int jj, int lane) {
  return buf + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3);
}
// Before a warpgroup writes box buffers: at most KEEP earlier stores (the ones reading the other buffer) may still be reading
// shared memory.
template <int KEEP>
__device__ __forceinline__ void epi_begin(int cw, bool leader) {
  if (leader) tma_store_wait_read<KEEP>();
  named_bar_sync(1 + cw, 128);
}
// After: the writes are visible to the TMA unit, and the leader may store the boxes.
__device__ __forceinline__ void epi_end(int cw) {
  fence_proxy_async_smem();
  named_bar_sync(1 + cw, 128);
}
// The bf16 pair at (row, col), col even; 0 outside the matrix (those outputs are not stored).
__device__ __forceinline__ uint32_t ld_pair(const bf16* base, int64_t ld, int row, int col, int M, int N) {
  if (row >= M || col >= N) return 0u;
  const bf16* src = base + static_cast<int64_t>(row) * ld + col;
  if (col + 1 < N) return *reinterpret_cast<const uint32_t*>(src);
  return static_cast<uint32_t>(__bfloat16_as_ushort(*src));
}
// Pull the epilogue inputs of a warpgroup's 64 rows into L2 while the tile's last k-blocks run, so the loads above hit L2.
__device__ __forceinline__ void epi_prefetch(const CUtensorMap* tmC, const CUtensorMap* tmX, const Params& p, int n_blk, int row0) {
  for (int s = 0; s < BN / EPI_BOX; ++s) {
    const int col0 = n_blk * BN + EPI_BOX * s;
    if (col0 >= p.N) break;
    if (p.epi_mode == 1) {
      tma_prefetch_l2_2d(tmC, col0, row0);
    } else if (p.epi_mode == 2) {
      tma_prefetch_l2_2d(tmX, col0, row0);
    } else {
      tma_prefetch_l2_2d(tmX, col0, row0);
      tma_prefetch_l2_2d(tmX, p.swiglu_inter + col0, row0);
    }
  }
}

// tmC / tmX: the epilogue's tensor maps outside split-K (box {64, 64}).  tmC is the output (mode 4: m); tmX is the
// residual (mode 2, read through L2 prefetches only), gate|up (mode 4 output, mode 5 input).
template <int NWG, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(Tile<NWG>::NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmX, const Params p) {
  using T = Tile<NWG>;
  constexpr int BM = T::BM, A_BYTES = T::A_BYTES, STAGE_BYTES = T::STAGE_BYTES, STAGES = T::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + T::EPI_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                           // [STAGES]

  const int num_items = p.num_m_tiles * p.num_n_tiles * p.split_k;
  const int num_kb_total = (p.K + BK - 1) / BK;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NWG * 128);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();   // PDL: the predecessor's outputs (A, B, C_old, residual) are complete from here on

  const int wg = threadIdx.x >> 7;
  if (wg == 0) {
    // ===================================== TMA producer =====================================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < num_items; t += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(t / p.split_k, p.num_m_tiles, p.num_n_tiles, m_blk, n_blk, p.gm);
        const int kb0 = (t % p.split_k) * p.kb_per_split;
        const int kb1 = min(num_kb_total, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int st = static_cast<int>(it % STAGES);
          // No wait in this kernel may contain a function call (mbar_wait's printf), not even here in the producer: ptxas then
          // serialises every wgmma of the kernel (it reports C7510), one k-step at a time with the tensor cores idle between them.
          mbar_wait_nocall(&empty_bar[st], ((it / STAGES) & 1u) ^ 1u);
          uint8_t* sA = smem + st * STAGE_BYTES;
          uint8_t* sB = sA + A_BYTES;
          mbar_arrive_expect_tx(&full_bar[st], STAGE_BYTES);
          if constexpr (A_MN) {    // stored [K, M]: NWG {64 m, 64 k} boxes
#pragma unroll
            for (int h = 0; h < NWG; ++h) tma_load_2d(&tmA, &full_bar[st], sA + h * (64 * BK * 2), m_blk * BM + 64 * h, kb * BK);
          } else {                 // stored [M, K]: one {64 k, BM m} box
            tma_load_2d(&tmA, &full_bar[st], sA, kb * BK, m_blk * BM);
          }
          if constexpr (B_MN) {    // stored [K, N]: four {64 n, 64 k} boxes
#pragma unroll
            for (int h = 0; h < 4; ++h) {
              const int c0 = p.epi_mode == 4 ? (h >> 1) * p.swiglu_inter + n_blk * 128 + (h & 1) * 64 : n_blk * BN + h * 64;
              tma_load_2d(&tmB, &full_bar[st], sB + h * (B_BYTES / 4), c0, kb * BK);
            }
          } else {                 // stored [N, K]: two {64 k, 128 n} boxes
            tma_load_2d(&tmB, &full_bar[st], sB, kb * BK, n_blk * BN);
            tma_load_2d(&tmB, &full_bar[st], sB + B_BYTES / 2, kb * BK, n_blk * BN + 128);
          }
        }
      }
    }
    return;
  }

  // ===================================== MMA + epilogue =====================================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                                   // 64-row half of the tile
  const int wi = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const uint32_t ring = smem_u32(smem);
  // descriptor byte offsets of k-step kk (16 k) inside a stage
  constexpr uint32_t A_KSTEP = A_MN ? 2048u : 32u, B_KSTEP = B_MN ? 2048u : 32u;
  const uint32_t a_off = static_cast<uint32_t>(cw) * (64 * BK * 2);
  const bool leader = (threadIdx.x & 127) == 0;           // issues the warpgroup's epilogue stores and prefetches
  const bool prefetch = leader && (p.epi_mode == 1 || p.epi_mode == 2 || p.epi_mode == 5);
  const uint32_t ebuf = smem_u32(smem + STAGES * STAGE_BYTES) + cw * 2 * EPI_BOX_BYTES;   // this warpgroup's two boxes
  uint32_t nbox = 0;                                       // boxes stored so far (modes 0-2 alternate the two buffers)
  uint32_t it = 0;
  float acc[128];
  for (int t = blockIdx.x; t < num_items; t += gridDim.x) {
    int m_blk, n_blk;
    tile_coords(t / p.split_k, p.num_m_tiles, p.num_n_tiles, m_blk, n_blk, p.gm);
    const int kb0 = (t % p.split_k) * p.kb_per_split;
    const int nkb = min(num_kb_total, kb0 + p.kb_per_split) - kb0;
    const int prefetch_kb = nkb > 8 ? nkb - 8 : 0;
    fence_acc(acc);                                        // the previous tile's epilogue reads precede the zeroing
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    fence_acc(acc);
    for (int i = 0; i < nkb; ++i, ++it) {
      const int st = static_cast<int>(it % STAGES);
      mbar_wait_nocall(&full_bar[st], (it / STAGES) & 1u);
      const uint32_t sA = ring + st * STAGE_BYTES + a_off, sB = ring + st * STAGE_BYTES + A_BYTES;
      const uint64_t dA = wgmma_desc_sw128(sA, A_MN ? 64 * BK * 2 : 16, 1024);
      const uint64_t dB = wgmma_desc_sw128(sB, B_MN ? B_BYTES / 4 : 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)
        wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, dA + ((kk * A_KSTEP) >> 4), dB + ((kk * B_KSTEP) >> 4),
                                                     (i > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
      if (prefetch && i == prefetch_kb) epi_prefetch(&tmC, &tmX, p, n_blk, m_blk * BM + cw * 64);
      wgmma_wait<1>();                                     // k-block i-1 is finished: its stage can be refilled
      if (i > 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    fence_acc(acc);                                        // no accumulator access may move above the wait
    if (nkb > 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);

    // accumulator fragment: register 4j + 2i + e holds row 16 wi + lane/4 + 8i, column 8j + 2 (lane % 4) + e
    const int row0 = m_blk * BM + cw * 64;                 // first row of the warpgroup's rows and boxes
    const int r_lo = wi * 16 + (lane >> 2);                // this thread's rows: row0 + r_lo + 8 i
    const int cq = 2 * (lane & 3);
    if (p.epi_mode == 3) {
      // split-K: fp32 partial sums reduced in L2 (N % 8 == 0: a pair is 8-byte aligned); the bias is added where the sums are
      // rounded to bf16
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = row0 + r_lo + 8 * i;
        if (row >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int col = n_blk * BN + 8 * j + cq;
          if (col >= p.N) continue;
          float* w = p.ws + static_cast<int64_t>(row) * p.N + col;
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(w), "f"(acc[4 * j + 2 * i]), "f"(acc[4 * j + 2 * i + 1])
                       : "memory");
        }
      }
      continue;
    }
    if (p.epi_mode == 4) {
      // gate|up + SwiGLU (llama/modeling.py:38-45, 632-652): accumulator columns [0,128) = gate, [128,256) = up of channels
      // [128 n_blk, +128).  Rounding points of the unfused path: gate and up each rounded to bf16 (the Linear outputs, kept for
      // the backward), then silu(g) * u in fp32 and one rounding.
#pragma unroll
      for (int h = 0; h < 2; ++h) {                        // 64 channels per box
        const int ch0 = n_blk * 128 + EPI_BOX * h;
        if (ch0 >= p.swiglu_inter) continue;
        if (p.aux != nullptr) {                            // gate and up, as the unfused GEMM rounds them
          epi_begin<0>(cw, leader);
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * h + jj;
              st_shared_u32(epi_slot(ebuf, r_lo + 8 * i, jj, lane), pack_bf16x2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]));
              st_shared_u32(epi_slot(ebuf + EPI_BOX_BYTES, r_lo + 8 * i, jj, lane),
                            pack_bf16x2(acc[4 * (j + 16) + 2 * i], acc[4 * (j + 16) + 2 * i + 1]));
            }
          epi_end(cw);
          if (leader) {
            tma_store_2d(&tmX, ebuf, ch0, row0);
            tma_store_2d(&tmX, ebuf + EPI_BOX_BYTES, p.swiglu_inter + ch0, row0);
            tma_store_commit();
          }
        }
        epi_begin<0>(cw, leader);
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * h + jj;
            const uint32_t gp = pack_bf16x2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
            const uint32_t up = pack_bf16x2(acc[4 * (j + 16) + 2 * i], acc[4 * (j + 16) + 2 * i + 1]);
            st_shared_u32(epi_slot(ebuf, r_lo + 8 * i, jj, lane), swiglu_fwd_pair(gp, up));
          }
        epi_end(cw);
        if (leader) {
          tma_store_2d(&tmC, ebuf, ch0, row0);
          tma_store_commit();
        }
      }
      continue;
    }
    if (p.epi_mode == 5) {                                 // d(gate) box | d(up) box per 64 channels
#pragma unroll
      for (int s = 0; s < BN / EPI_BOX; ++s) {
        const int ch0 = n_blk * BN + EPI_BOX * s;
        if (ch0 >= p.N) continue;
        epi_begin<0>(cw, leader);
#pragma unroll
        for (int q = 0; q < 4; ++q) {                      // 8 input registers at a time next to the 128 accumulators
          const int i = q >> 1, jj0 = 4 * (q & 1);
          uint32_t g[4], u[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int row = row0 + r_lo + 8 * i, ch = ch0 + 8 * (jj0 + k) + cq;
            g[k] = ld_pair(p.aux, p.ld_aux, row, ch, p.M, p.N);
            u[k] = ld_pair(p.aux + p.swiglu_inter, p.ld_aux, row, ch, p.M, p.N);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int jj = jj0 + k, j = 8 * s + jj;
            uint32_t dg2, du2;                             // d(m) with the GEMM's own bf16 output rounding
            swiglu_bwd_pair(g[k], u[k], bf16_round(acc[4 * j + 2 * i]), bf16_round(acc[4 * j + 2 * i + 1]), dg2, du2);
            st_shared_u32(epi_slot(ebuf, r_lo + 8 * i, jj, lane), dg2);
            st_shared_u32(epi_slot(ebuf + EPI_BOX_BYTES, r_lo + 8 * i, jj, lane), du2);
          }
        }
        epi_end(cw);
        if (leader) {
          tma_store_2d(&tmC, ebuf, ch0, row0);
          tma_store_2d(&tmC, ebuf + EPI_BOX_BYTES, p.swiglu_inter + ch0, row0);
          tma_store_commit();
        }
      }
      continue;
    }
    // modes 0, 1, 2, 6, 7
#pragma unroll
    for (int s = 0; s < BN / EPI_BOX; ++s) {
      const int col0 = n_blk * BN + EPI_BOX * s;
      if (col0 >= p.N) continue;
      if (p.epi_mode >= 6) {
        // fp32 output: the 64 columns leave as two 64 x 32 fp32 boxes (128 bytes per row, like a bf16 box), one in each
        // buffer.  Mode 7 adds them onto C in L2 (TMA reduce-add): one fp32 add per element, C_old never enters the
        // registers.  Row r's byte b sits at b ^ (16 (r % 8)); this thread's pair of box column 8 jj + 2 (lane % 4) is row
        // byte 32 jj + 8 (lane % 4), and r % 8 = lane / 4 for both of its rows: a warp's 8 rows fill every chunk twice.
        const uint32_t sw = (lane >> 2) << 4;
        const uint32_t row_off = r_lo * 128 + ((8 * (lane & 3)) ^ (sw & 16));
        epi_begin<0>(cw, leader);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 8 * s + 4 * h + jj;
            const uint32_t slot = ebuf + h * EPI_BOX_BYTES + row_off + ((32 * jj) ^ (sw & 96));
            st_shared_f32x2(slot, acc[4 * j], acc[4 * j + 1]);
            st_shared_f32x2(slot + 8 * 128, acc[4 * j + 2], acc[4 * j + 3]);
          }
        epi_end(cw);
        if (leader) {
          if (p.epi_mode == 7) {
            tma_reduce_add_2d(&tmC, ebuf, col0, row0);
            tma_reduce_add_2d(&tmC, ebuf + EPI_BOX_BYTES, col0 + EPI_BOX_F32, row0);
          } else {
            tma_store_2d(&tmC, ebuf, col0, row0);
            tma_store_2d(&tmC, ebuf + EPI_BOX_BYTES, col0 + EPI_BOX_F32, row0);
          }
          tma_store_commit();
        }
        continue;
      }
      const uint32_t buf = ebuf + (nbox++ & 1u) * EPI_BOX_BYTES;
      epi_begin<1>(cw, leader);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        uint32_t o[8];                                     // C_old (mode 1) or residual (mode 2) pairs of row r_lo + 8 i
        if (p.epi_mode != 0) {
          const bf16* src = p.epi_mode == 1 ? p.c : p.r;
          const int64_t ld = p.epi_mode == 1 ? p.ldc : p.ldr;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) o[jj] = ld_pair(src, ld, row0 + r_lo + 8 * i, col0 + 8 * jj + cq, p.M, p.N);
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * s + jj, col = col0 + 8 * jj + cq;
          float f0 = acc[4 * j + 2 * i], f1 = acc[4 * j + 2 * i + 1];
          if (p.bias != nullptr) {
            if (col < p.N) f0 += __ldg(p.bias + col);
            if (col + 1 < p.N) f1 += __ldg(p.bias + col + 1);
          }
          if (p.epi_mode != 0) {
            if (p.epi_mode == 2) { f0 = bf16_round(f0); f1 = bf16_round(f1); }
            const float2 of = unpack_bf16x2(o[jj]);
            f0 += of.x;
            f1 += of.y;
          }
          st_shared_u32(epi_slot(buf, r_lo + 8 * i, jj, lane), pack_bf16x2(f0, f1));
        }
      }
      epi_end(cw);
      if (leader) {
        tma_store_2d(&tmC, buf, col0, row0);
        tma_store_commit();
      }
    }
  }
  if (leader) tma_store_wait<0>();                         // the box buffers stay allocated until the last store is done
}

template <int NWG, bool A_MN, bool B_MN>
static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmX, const Params& p,
                  int max_ctas, cudaStream_t stream) {
  using T = Tile<NWG>;
  constexpr int SMEM_BYTES = T::SMEM_BYTES;
  auto kern = gemm_bf16_kernel<NWG, A_MN, B_MN>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(gemm smem=%d): %s", SMEM_BYTES, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  const int num_items = p.num_m_tiles * p.num_n_tiles * p.split_k;
  int ctas = sm_count();
  if (max_ctas > 0 && max_ctas < ctas) ctas = max_ctas;
  if (ctas > num_items) ctas = num_items;
  Params pp = p;
  // Raster group: the tiles of GM consecutive m-tiles are walked n-column by n-column, so the group's A panels are re-used
  // out of L2 by every wave while the B panels stream through once per group.  16 m-tiles of 128 rows keep the group's A
  // panels within ~18 MB of the 50 MB L2 for K <= 4608; longer K takes 8.
  pp.gm = (16ll * 128 * p.K * 2 <= (18ll << 20)) ? 16 : 8;
  cudaError_t e = launch_pdl(kern, dim3(ctas), dim3(T::NUM_THREADS), SMEM_BYTES, stream, tmA, tmB, tmC, tmX, pp);
  if (e != cudaSuccess) {
    set_last_error("gemm launch: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  return 0;
}

// Epilogue box map: a [rows, cols] bf16 matrix with leading dimension ld, box {64 columns, 64 rows}.
static int make_epi_map(CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld) {
  const uint64_t dims[2] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(rows)}, strides[1] = {static_cast<uint64_t>(ld) * 2};
  const uint32_t box[2] = {EPI_BOX, EPI_BOX};
  return encode_tmap_bf16(tm, base, 2, dims, strides, box);
}
// fp32 output map (modes 6, 7): [rows, cols] fp32, box {32 columns, 64 rows}.
static int make_epi_map_f32(CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld) {
  const uint64_t dims[2] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(rows)}, strides[1] = {static_cast<uint64_t>(ld) * 4};
  const uint32_t box[2] = {EPI_BOX_F32, EPI_BOX};
  return encode_tmap_f32(tm, base, 2, dims, strides, box);
}
static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

// Tensor maps of the shared-memory epilogue (every mode but split-K).  TMA needs 16-byte aligned base addresses (the strides
// are multiples of 8 elements already): the entry points reject outputs and epilogue inputs that are not.
static int setup_smem_epilogue(const Params& p, CUtensorMap* tmC, CUtensorMap* tmX) {
  int rc;
  switch (p.epi_mode) {
    case 2:
      if ((rc = make_epi_map(tmX, p.r, p.M, p.N, p.ldr)) != 0) return rc;
      return make_epi_map(tmC, p.c, p.M, p.N, p.ldc);
    case 3:
      return 0;
    case 6:
    case 7:
      return make_epi_map_f32(tmC, p.ws, p.M, p.N, p.ldc);
    case 4:   // p.N = 2 I: tmC is m [M, I], tmX the gate|up output [M, 2I]
      if (p.aux != nullptr && (rc = make_epi_map(tmX, p.aux, p.M, p.N, p.ld_aux)) != 0) return rc;
      return make_epi_map(tmC, p.c, p.M, p.swiglu_inter, p.ldc);
    case 5:   // p.N = I: tmC is d(gate)|d(up) [M, 2I], tmX the saved gate|up [M, 2I]
      if ((rc = make_epi_map(tmX, p.aux, p.M, 2ll * p.N, p.ld_aux)) != 0) return rc;
      return make_epi_map(tmC, p.c, p.M, 2ll * p.N, p.ldc);
    default:  // 0, 1
      return make_epi_map(tmC, p.c, p.M, p.N, p.ldc);
  }
}

static int dispatch(bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB, Params p, int max_ctas,
                    cudaStream_t stream) {
  CUtensorMap tmC, tmX;
  memset(&tmC, 0, sizeof(tmC));
  memset(&tmX, 0, sizeof(tmX));
  int rc;
  if ((rc = setup_smem_epilogue(p, &tmC, &tmX)) != 0) return rc;
  if (tile_wgs(p.M) == 1) {
    if (a_mn && b_mn) return launch<1, true, true>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
    if (a_mn) return launch<1, true, false>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
    if (b_mn) return launch<1, false, true>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
    return launch<1, false, false>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
  }
  if (a_mn && b_mn) return launch<2, true, true>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
  if (a_mn) return launch<2, true, false>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
  if (b_mn) return launch<2, false, true>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
  return launch<2, false, false>(tmA, tmB, tmC, tmX, p, max_ctas, stream);
}

// A operand map.  K-major: stored [M, K], box {64 k, 128 m}.  MN-major: stored [K, M], box {64 m, 64 k}.
static int make_a_map(CUtensorMap* tm, const void* A, int64_t M, int64_t K, int64_t lda, bool mn) {
  uint64_t dims[2], strides[1] = {static_cast<uint64_t>(lda) * 2};
  uint32_t box[2];
  if (mn) { dims[0] = M; dims[1] = K; box[0] = 64; box[1] = BK; }
  else    { dims[0] = K; dims[1] = M; box[0] = BK; box[1] = 64 * tile_wgs(M); }
  return encode_tmap_bf16(tm, A, 2, dims, strides, box);
}
// B operand map.  K-major: stored [N, K], box {64 k, 128 n}.  MN-major: stored [K, N], box {64 n, 64 k}.
static int make_b_map(CUtensorMap* tm, const void* B, int64_t N, int64_t K, int64_t ldb, bool mn) {
  uint64_t dims[2], strides[1] = {static_cast<uint64_t>(ldb) * 2};
  uint32_t box[2];
  if (mn) { dims[0] = N; dims[1] = K; box[0] = 64; box[1] = BK; }
  else    { dims[0] = K; dims[1] = N; box[0] = BK; box[1] = 128; }
  return encode_tmap_bf16(tm, B, 2, dims, strides, box);
}

static Params base_params(int64_t M, int64_t N, int64_t K) {
  Params p = {};
  p.M = static_cast<int>(M);
  p.N = static_cast<int>(N);
  p.K = static_cast<int>(K);
  const int64_t bm = 64 * tile_wgs(M);
  p.num_m_tiles = static_cast<int>((M + bm - 1) / bm);
  p.num_n_tiles = static_cast<int>((N + BN - 1) / BN);
  p.split_k = 1;
  p.kb_per_split = static_cast<int>((K + BK - 1) / BK);
  return p;
}

}  // namespace gemm
}  // namespace b200

extern "C" int b200_gemm_bf16_ex(const void* A, const void* B, void* C, const float* bias, const void* residual,
                                 int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int64_t ldr,
                                 int a_mn_major, int b_mn_major, int accumulate, int max_ctas, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::gemm;
  B200_CHECK_ARG(A && B && C, "gemm: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: non-positive dimension M=%lld N=%lld K=%lld", (long long)M,
                 (long long)N, (long long)K);
  B200_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldc % 8 == 0, "gemm: leading dimensions must be multiples of 8");
  B200_CHECK_ARG(!(residual && accumulate), "gemm: residual and accumulate are mutually exclusive");
  B200_CHECK_ARG(!residual || ldr % 8 == 0, "gemm: ldr must be a multiple of 8");
  B200_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "gemm: dimension too large");
  B200_CHECK_ARG(aligned16(C), "gemm: C must be 16-byte aligned");
  B200_CHECK_ARG(!residual || aligned16(residual), "gemm: residual must be 16-byte aligned");
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_a_map(&tmA, A, M, K, lda, a_mn_major)) != 0) return rc;
  if ((rc = make_b_map(&tmB, B, N, K, ldb, b_mn_major)) != 0) return rc;
  Params p = base_params(M, N, K);
  p.epi_mode = residual ? 2 : (accumulate ? 1 : 0);
  p.bias = bias;
  p.c = static_cast<bf16*>(C);
  p.ldc = ldc;
  p.r = static_cast<const bf16*>(residual);
  p.ldr = ldr;
  return dispatch(a_mn_major, b_mn_major, tmA, tmB, p, max_ctas, stream);
}

// fp32-output form for weight gradients kept in fp32 (fused_linear_param_grad_add(..., multi_precision=True),
// llm/utils/fused_layers.py:44-50): C_f32 = acc, or C_f32 += acc with one fp32 add per element by TMA reduce-add.
extern "C" int b200_gemm_bf16_f32(const void* A, const void* B, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                                  int64_t ldb, int64_t ldc, int a_mn_major, int b_mn_major, int accumulate, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::gemm;
  B200_CHECK_ARG(A && B && C, "gemm_f32: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm_f32: non-positive dimension M=%lld N=%lld K=%lld", (long long)M,
                 (long long)N, (long long)K);
  B200_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "gemm_f32: lda and ldb must be multiples of 8");
  B200_CHECK_ARG(ldc % 4 == 0 && ldc >= N, "gemm_f32: ldc must be a multiple of 4 and >= N (ldc=%lld N=%lld)", (long long)ldc,
                 (long long)N);
  B200_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "gemm_f32: dimension too large");
  B200_CHECK_ARG(aligned16(C), "gemm_f32: C must be 16-byte aligned");
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_a_map(&tmA, A, M, K, lda, a_mn_major)) != 0) return rc;
  if ((rc = make_b_map(&tmB, B, N, K, ldb, b_mn_major)) != 0) return rc;
  Params p = base_params(M, N, K);
  p.epi_mode = accumulate ? 7 : 6;
  p.ws = C;
  p.ldc = ldc;
  return dispatch(a_mn_major, b_mn_major, tmA, tmB, p, 0, stream);
}

// gate|up projection + SwiGLU in one kernel (training forward of LlamaMLP, llama/modeling.py:632-652 with fuse_attention_ffn):
//   GU[M, 2I] = bf16(X[M, K] * W[K, 2I])   (gate columns [0, I), up columns [I, 2I): kept for the backward)
//   Mout[M, I] = bf16( silu(GU[:, c]) * GU[:, I + c] )
// The 256-column tile is formed from 128 gate columns and the 128 up columns of the same channels (TMA boxes at different
// column coordinates of the SAME row-major weight), so the epilogue holds both halves of every channel.
extern "C" int b200_gemm_swiglu_bf16(const void* X, const void* W, void* GU, void* Mout, int64_t M, int64_t inter, int64_t K,
                                     int64_t ldx, int64_t ldw, int64_t ldgu, int64_t ldm, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::gemm;
  B200_CHECK_ARG(X && W && Mout, "gemm_swiglu: null pointer");     // GU may be null: gate|up are then not written (inference)
  B200_CHECK_ARG(M > 0 && inter > 0 && K > 0 && inter % 64 == 0, "gemm_swiglu: intermediate size must be a multiple of 64 (got %lld)",
                 (long long)inter);
  B200_CHECK_ARG(ldx % 8 == 0 && ldw % 8 == 0 && ldgu % 8 == 0 && ldm % 8 == 0, "gemm_swiglu: leading dimensions must be multiples of 8");
  B200_CHECK_ARG(M < (1ll << 31) && inter < (1ll << 30) && K < (1ll << 31), "gemm_swiglu: dimension too large");
  B200_CHECK_ARG(aligned16(Mout), "gemm_swiglu: Mout must be 16-byte aligned");
  B200_CHECK_ARG(!GU || aligned16(GU), "gemm_swiglu: GU must be 16-byte aligned");
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_a_map(&tmA, X, M, K, ldx, false)) != 0) return rc;
  if ((rc = make_b_map(&tmB, W, 2 * inter, K, ldw, true)) != 0) return rc;
  Params p = base_params(M, 2 * inter, K);
  p.num_n_tiles = static_cast<int>((inter + 127) / 128);   // a last tile of 64 channels loads (and ignores) 64 columns past them
  p.epi_mode = 4;
  p.swiglu_inter = static_cast<int>(inter);
  p.c = static_cast<bf16*>(Mout);
  p.ldc = ldm;
  p.aux = static_cast<bf16*>(GU);
  p.ld_aux = ldgu;
  return dispatch(false, true, tmA, tmB, p, 0, stream);
}

// down-projection dX GEMM + SwiGLU backward in one kernel (backward of LlamaMLP, llama/modeling.py:632-652):
//   d(m)[M, I] = dY[M, h] * W_down[I, h]^T   (never written),   DGU[M, 2I] = [ d(m) * up * silu'(gate) | d(m) * silu(gate) ]
// GU is the saved gate|up projection [M, 2I].  Bit-identical to b200_gemm_bf16 (dX) followed by b200_swiglu_bwd.  I % 64 == 0.
extern "C" int b200_gemm_swiglu_bwd_bf16(const void* dY, const void* Wdown, const void* GU, void* DGU, int64_t M, int64_t inter,
                                         int64_t K, int64_t lddy, int64_t ldw, int64_t ldgu, int64_t lddgu, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::gemm;
  B200_CHECK_ARG(dY && Wdown && GU && DGU, "gemm_swiglu_bwd: null pointer");
  B200_CHECK_ARG(M > 0 && inter > 0 && K > 0 && inter % 64 == 0, "gemm_swiglu_bwd: intermediate size must be a multiple of 64 (got %lld)",
                 (long long)inter);
  B200_CHECK_ARG(lddy % 8 == 0 && ldw % 8 == 0 && ldgu % 8 == 0 && lddgu % 8 == 0, "gemm_swiglu_bwd: leading dimensions must be multiples of 8");
  B200_CHECK_ARG(M < (1ll << 31) && inter < (1ll << 30) && K < (1ll << 31), "gemm_swiglu_bwd: dimension too large");
  B200_CHECK_ARG(aligned16(GU), "gemm_swiglu_bwd: GU must be 16-byte aligned");
  B200_CHECK_ARG(aligned16(DGU), "gemm_swiglu_bwd: DGU must be 16-byte aligned");
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_a_map(&tmA, dY, M, K, lddy, false)) != 0) return rc;
  if ((rc = make_b_map(&tmB, Wdown, inter, K, ldw, false)) != 0) return rc;   // W_down stored [I, h] = [N, K]: K-major B
  Params p = base_params(M, inter, K);
  p.epi_mode = 5;
  p.swiglu_inter = static_cast<int>(inter);
  p.c = static_cast<bf16*>(DGU);
  p.ldc = lddgu;
  p.aux = const_cast<bf16*>(static_cast<const bf16*>(GU));
  p.ld_aux = ldgu;
  return dispatch(false, false, tmA, tmB, p, 0, stream);
}

namespace b200 {
namespace gemm {
// out[m, n] = bf16(ws[m, n] + bias[n]) ; ws is re-zeroed for the next split-K GEMM that uses it
__global__ void splitk_finish_kernel(float* __restrict__ ws, const float* __restrict__ bias, bf16* __restrict__ out,
                                     int64_t M, int64_t N, int64_t ldc) {
  const int64_t nch = N >> 3;
  const int64_t total = M * nch;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nch, c = i % nch;
    float4* src = reinterpret_cast<float4*>(ws + r * N) + 2 * c;
    float4 a = src[0], b = src[1];
    src[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    src[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias != nullptr) {
      const float4* bp = reinterpret_cast<const float4*>(bias) + 2 * c;
      const float4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
      a.x += b0.x; a.y += b0.y; a.z += b0.z; a.w += b0.w;
      b.x += b1.x; b.y += b1.y; b.z += b1.z; b.w += b1.w;
    }
    uint4 o;
    o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
    o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
    *(reinterpret_cast<uint4*>(out + r * ldc) + c) = o;
  }
}
}  // namespace gemm

int splitk_finish(float* ws, const float* bias, void* out, int64_t M, int64_t N, int64_t ldc, cudaStream_t stream) {
  const int64_t total = M * (N / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  gemm::splitk_finish_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(ws, bias, static_cast<bf16*>(out), M, N, ldc);
  return check_launch("gemm_splitk(finish)");
}

}  // namespace b200

extern "C" int64_t b200_gemm_splitk_workspace_bytes(int64_t M, int64_t N) { return M * N * 4; }

// Weight-streaming GEMM for the decode step: M <= 128 tokens, the weight matrix dominates the traffic, so K is split across
// CTAs until the persistent grid covers every SM; fp32 partial tiles are reduced in L2 with atomic adds.
extern "C" int b200_gemm_bf16_splitk(const void* A, const void* B, void* C, const float* bias, void* workspace, int64_t M,
                                     int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int a_mn_major,
                                     int b_mn_major, int split_k, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::gemm;
  B200_CHECK_ARG(A && B && workspace, "gemm_splitk: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0 && N % 8 == 0, "gemm_splitk: bad dimensions (N must be a multiple of 8)");
  B200_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldc % 8 == 0, "gemm_splitk: leading dimensions must be multiples of 8");
  B200_CHECK_ARG(!C || aligned16(C), "gemm_splitk: C must be 16-byte aligned");
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_a_map(&tmA, A, M, K, lda, a_mn_major)) != 0) return rc;
  if ((rc = make_b_map(&tmB, B, N, K, ldb, b_mn_major)) != 0) return rc;
  Params p = base_params(M, N, K);
  const int num_kb = p.kb_per_split;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  if (split_k <= 0) {
    // smallest split that gives every SM at least one work item, capped so each item keeps >= 4 k-blocks
    const int sms = sm_count();
    split_k = (sms + tiles - 1) / tiles;
    if (split_k > num_kb / 4) split_k = num_kb / 4;
    if (split_k < 1) split_k = 1;
  }
  p.kb_per_split = (num_kb + split_k - 1) / split_k;
  p.split_k = (num_kb + p.kb_per_split - 1) / p.kb_per_split;   // no empty ranges
  p.epi_mode = 3;
  p.ws = static_cast<float*>(workspace);
  // `workspace` must be all-zero on entry; the finish kernel leaves it zeroed again (no memset per GEMM).
  if ((rc = dispatch(a_mn_major, b_mn_major, tmA, tmB, p, 0, stream)) != 0) return rc;
  if (C == nullptr) return 0;   // C == NULL: the consumer kernel reads (and re-zeroes) the fp32 workspace itself
  return splitk_finish(static_cast<float*>(workspace), bias, C, M, N, ldc, stream);
}

extern "C" int b200_gemm_bf16(const void* A, const void* B, void* C, const float* bias, int64_t M, int64_t N, int64_t K,
                              int64_t lda, int64_t ldb, int64_t ldc, int a_mn_major, int b_mn_major, int accumulate,
                              cudaStream_t stream) {
  return b200_gemm_bf16_ex(A, B, C, bias, nullptr, M, N, K, lda, ldb, ldc, 0, a_mn_major, b_mn_major, accumulate,
                           /*max_ctas=*/0, stream);
}
