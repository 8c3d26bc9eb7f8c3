// Causal GQA flash-attention backward on Hopper tensor cores (head_dim 64 or 128).
//
//   inputs : q, k, v, o, do, lse            outputs: dq, dk, dv (bf16; fp32 accumulation buffers in the workspace)
//   P = exp(S*scale - lse) ; dP = dO V^T ; dS = P o (dP - D) * scale, D = rowsum(dO o O)
//   dV = P^T dO ; dK = dS^T Q ; dQ = dS K
//
// Replaces Paddle-core flash_attn_grad (reference: fusion_ops.py:240-246 backward of scaled_dot_product_attention;
// wrapper shape in csrc/gpu/flash_attn_bwd.cc:22-92).
//
// Two kernels (b200_set_fa_bwd_impl); both keep one q-head's dK / dV tile in registers while they walk the q tiles that can
// see it, and work per q-head (not per kv-head) so that a GQA group's heads spread over the SMs.  P and dS are rounded to
// bf16 before their matmuls, accumulation is fp32, and dq / dk / dv are rounded to bf16 once by the finishing kernels.
//
// impl 2 (default), fa_bwd_wgmma_kernel: one CTA = (batch, q-head, 128-row kv tile), two warpgroups of 64 kv rows each.
//   TMA (issued by thread 0): K and V once; then per 64-row q tile Q, dO (4-D tensor maps, 128-byte swizzle, rows past S
//                             zero-filled) and the tile's lse*log2(e) and delta rows into a 2-stage mbarrier ring
//   each warpgroup, wgmma throughout:
//                   S^T = K Q^T, dP^T = V dO^T            (m64n64k16, both operands in shared memory)
//                   P^T, dS^T in registers                (causal + FlashMask start rows)
//                   dV += P^T dO, dK += dS^T Q            (m64n128k16, A = the bf16-packed P^T / dS^T registers)
//                   dQ = dS K                             (dS^T through shared memory; each warpgroup 64 of the d columns)
//                   dQ tile -> fp32 staging -> cp.reduce.async.bulk.tensor add into the dQ buffer
//                   dK / dV -> TMA reduce-adds into the kv head's fp32 buffers once per CTA
//   head_dim 64: one [128 kv][64 d] swizzled block for K and V, one [64 q][64 d] block for Q and dO; S^T and dP^T take 4
//   k-steps, dV / dK are m64n64k16.  dQ = dS K is split over the kv rows instead of the d columns: each warpgroup multiplies
//   its own 64 rows of dS^T by its own 64 rows of K into a full [64 q][64 d] partial and reduce-adds it, so every wgmma keeps
//   the m64n64k16 shape with swizzle-atom-aligned operands and the warpgroups need no shared barrier for dS^T; the price is
//   twice the dQ reduce-add bytes (2 x 16 KB per q tile, as at head_dim 128).  (A d split would need m64n32 tiles that start
//   inside a swizzle row; a q-row split is below wgmma's 64-row M.)
// impl 1, fa_bwd_kernel: the mma.sync cross-check.  One CTA (8 warps) = (batch, q-head, 64-row kv tile), 64-row q tiles
// through cp.async; per q tile S and dP per warp in registers -> P, dS as bf16 in shared memory -> dV, dK (ldmatrix.trans
// operands) and dQ, which it adds to the fp32 dQ buffer with atomics, as it does dK / dV at the end.
#include <climits>

#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace fab {

constexpr int BKV = 64;
constexpr int NUM_THREADS = 256;

struct Params {
  const bf16 *q, *k, *v, *dout;
  int64_t ldq, ldk, ldv, lddo;
  int S, B, nh, kvh, Spad;
  float scale, scale_log2;
  const float* lse2;    // [B, nh, Spad]  lse * log2(e); +inf on the padding rows s >= S (P = 0 there)
  const float* delta;   // [B, nh, Spad]  rowsum(dO o O); 0 on the padding rows
  const int* mask_start;   // FlashMask causal-LT start rows [B, S] (see fa_fwd.cu) or nullptr
  float* dq_acc;        // [B, S, nh, D]
  float* dk_acc;        // [B, S, kvh, D]
  float* dv_acc;
};

// [rows][D] bf16 tiles: 16-byte chunks XOR-swizzled by row & 7 (as fa_fwd.cu); [rows][64] tiles (P, dS): 128-byte rows
template <int D>
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return static_cast<uint32_t>(row * (D * 2) + ((chunk ^ (row & 7)) << 4)); }
__device__ __forceinline__ uint32_t swz64(int row, int chunk) { return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4)); }

template <int D, int BQ, bool MASK>
__global__ void __launch_bounds__(NUM_THREADS, 1) fa_bwd_kernel(const Params p) {
  constexpr int DCH = D / 8, DCH_LOG2 = D == 128 ? 4 : 3;   // 16-byte chunks per row of a [rows][D] tile
  constexpr int RG = BQ / 16;            // phase 1: row groups of 16 q rows
  constexpr int CH = 8 / RG;             //          column slices of the 64 kv columns
  constexpr int NT = 8 / CH;             //          8-column n-tiles per warp
  constexpr int QG = BQ / 16;            // dQ: row groups
  constexpr int DH = 8 / QG;             //     d slices
  constexpr int DTQ = DCH / DH;           //     8-column d tiles per warp
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sK = smem_u32(smem), sV = sK + BKV * D * 2, sQ = sV + BKV * D * 2, sdO = sQ + BQ * D * 2;
  const uint32_t sP = sdO + BQ * D * 2, sdS = sP + BQ * 128;
  float* s_lse = reinterpret_cast<float*>(smem + 2 * BKV * D * 2 + 2 * BQ * D * 2 + 2 * BQ * 128);
  float* s_delta = s_lse + BQ;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int num_kv_tiles = (p.S + BKV - 1) / BKV;
  const int jt = static_cast<int>(blockIdx.x);   // early kv tiles see the most q rows (causal): launched first
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / (p.nh / p.kvh);
  const int kv0 = jt * BKV;
  const size_t tok0 = static_cast<size_t>(batch) * p.S;
  int q_lo = kv0 / BQ, q_hi = (p.S + BQ - 1) / BQ;
  if constexpr (MASK) {   // rows at or past the last column's document end see none of this tile
    const int last = __ldg(p.mask_start + tok0 + min(kv0 + BKV - 1, p.S - 1));
    q_hi = min(q_hi, (last + BQ - 1) / BQ);
  }
  for (int i = threadIdx.x; i < BKV * DCH; i += NUM_THREADS) {
    const int r = i >> DCH_LOG2, ch = i & (DCH - 1);
    const bool ok = kv0 + r < p.S;
    cp_async_16(sK + swz<D>(r, ch), ok ? p.k + (tok0 + kv0 + r) * p.ldk + kv_head * D + ch * 8 : p.k, ok ? 16u : 0u);
    cp_async_16(sV + swz<D>(r, ch), ok ? p.v + (tok0 + kv0 + r) * p.ldv + kv_head * D + ch * 8 : p.v, ok ? 16u : 0u);
  }
  // dK / dV accumulators: warp = 16 kv rows (kg) x D/2 d columns (dh)
  const int kg = warp >> 1, dh = warp & 1;
  float dk[D / 16][4], dv[D / 16][4];
#pragma unroll
  for (int i = 0; i < D / 16; ++i) dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;

  for (int qt = q_lo; qt < q_hi; ++qt) {
    const int q0 = qt * BQ;
    for (int i = threadIdx.x; i < BQ * DCH; i += NUM_THREADS) {
      const int r = i >> DCH_LOG2, ch = i & (DCH - 1);
      const bool ok = q0 + r < p.S;
      cp_async_16(sQ + swz<D>(r, ch), ok ? p.q + (tok0 + q0 + r) * p.ldq + head * D + ch * 8 : p.q, ok ? 16u : 0u);
      cp_async_16(sdO + swz<D>(r, ch), ok ? p.dout + (tok0 + q0 + r) * p.lddo + head * D + ch * 8 : p.dout, ok ? 16u : 0u);
    }
    cp_async_commit();
    for (int i = threadIdx.x; i < BQ; i += NUM_THREADS) {   // BQ divides Spad
      const size_t idx = (static_cast<size_t>(batch) * p.nh + head) * p.Spad + q0 + i;
      s_lse[i] = __ldg(p.lse2 + idx);
      s_delta[i] = __ldg(p.delta + idx);
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---------------- phase 1: S = Q K^T, dP = dO V^T  (16 q rows x 8 NT kv columns per warp) ----------------
    {
      const int rg = warp % RG, cs = warp / RG;
      float s[NT][4], dp[NT][4];
#pragma unroll
      for (int i = 0; i < NT; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < D / 16; ++kc) {
        uint32_t a[4], ad[4];
        ldsm_x4(sQ + swz<D>(rg * 16 + (lane & 15), kc * 2 + (lane >> 4)), a);
        ldsm_x4(sdO + swz<D>(rg * 16 + (lane & 15), kc * 2 + (lane >> 4)), ad);
#pragma unroll
        for (int np = 0; np < NT / 2; ++np) {
          const int kr = cs * NT * 8 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
          uint32_t b[4], bv[4];
          ldsm_x4(sK + swz<D>(kr, kc * 2 + ((lane >> 3) & 1)), b);
          ldsm_x4(sV + swz<D>(kr, kc * 2 + ((lane >> 3) & 1)), bv);
          mma_bf16_16816(s[2 * np], a, b[0], b[1]);
          mma_bf16_16816(s[2 * np + 1], a, b[2], b[3]);
          mma_bf16_16816(dp[2 * np], ad, bv[0], bv[1]);
          mma_bf16_16816(dp[2 * np + 1], ad, bv[2], bv[3]);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rl = rg * 16 + g + 8 * h, r = q0 + rl;
        const float lse2 = s_lse[rl], dl = s_delta[rl];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          float pv[2], dsv[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = kv0 + cs * NT * 8 + nt * 8 + 2 * tq + e;
            bool dead = c > r;
            if constexpr (MASK) {
              if (!dead && c < p.S) dead = r >= __ldg(p.mask_start + tok0 + c);
            }
            pv[e] = dead ? 0.f : fast_exp2(fmaf(s[nt][2 * h + e], p.scale_log2, -lse2));
            dsv[e] = pv[e] * (dp[nt][2 * h + e] - dl) * p.scale;
          }
          const int cc = cs * NT + nt;     // 8-column chunk index within the 64 kv columns
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(sP + swz64(rl, cc) + tq * 4), "r"(pack_bf16x2(pv[0], pv[1])) : "memory");
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(sdS + swz64(rl, cc) + tq * 4), "r"(pack_bf16x2(dsv[0], dsv[1])) : "memory");
        }
      }
    }
    __syncthreads();

    // ---------------- phase 2: dV += P^T dO, dK += dS^T Q, dQ += dS K ----------------
#pragma unroll
    for (int qc = 0; qc < BQ / 16; ++qc) {
      uint32_t ap[4], as[4];
      const int pr = qc * 16 + (lane & 7) + ((lane >> 4) << 3), pc = kg * 2 + ((lane >> 3) & 1);
      ldsm_x4_t(sP + swz64(pr, pc), ap);
      ldsm_x4_t(sdS + swz64(pr, pc), as);
#pragma unroll
      for (int dp2 = 0; dp2 < D / 32; ++dp2) {
        const int br = qc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, bc = dh * (DCH / 2) + dp2 * 2 + (lane >> 4);
        uint32_t bo[4], bq[4];
        ldsm_x4_t(sdO + swz<D>(br, bc), bo);
        ldsm_x4_t(sQ + swz<D>(br, bc), bq);
        mma_bf16_16816(dv[2 * dp2], ap, bo[0], bo[1]);
        mma_bf16_16816(dv[2 * dp2 + 1], ap, bo[2], bo[3]);
        mma_bf16_16816(dk[2 * dp2], as, bq[0], bq[1]);
        mma_bf16_16816(dk[2 * dp2 + 1], as, bq[2], bq[3]);
      }
    }
    {
      const int qg = warp % QG, dsl = warp / QG;
      float dq[DTQ][4];
#pragma unroll
      for (int i = 0; i < DTQ; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < BKV / 16; ++kc) {
        uint32_t a[4];
        ldsm_x4(sdS + swz64(qg * 16 + (lane & 15), kc * 2 + (lane >> 4)), a);
#pragma unroll
        for (int dp2 = 0; dp2 < DTQ / 2; ++dp2) {
          uint32_t b[4];
          ldsm_x4_t(sK + swz<D>(kc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dsl * (DTQ) + dp2 * 2 + (lane >> 4)), b);
          mma_bf16_16816(dq[2 * dp2], a, b[0], b[1]);
          mma_bf16_16816(dq[2 * dp2 + 1], a, b[2], b[3]);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = q0 + qg * 16 + g + 8 * h;
        if (r >= p.S) continue;
        float* dst = p.dq_acc + ((tok0 + r) * p.nh + head) * D + dsl * DTQ * 8 + 2 * tq;
#pragma unroll
        for (int dt = 0; dt < DTQ; ++dt) {
          atomicAdd(dst + dt * 8, dq[dt][2 * h]);
          atomicAdd(dst + dt * 8 + 1, dq[dt][2 * h + 1]);
        }
      }
    }
    __syncthreads();   // Q, dO, P, dS are overwritten by the next q tile
  }
  // this head's dK / dV partials -> the kv head's fp32 buffers (the GQA group's heads add up there)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = kv0 + kg * 16 + g + 8 * h;
    if (r >= p.S) continue;
    const size_t off = ((tok0 + r) * p.kvh + kv_head) * D + dh * (D / 2) + 2 * tq;
#pragma unroll
    for (int dt = 0; dt < D / 16; ++dt) {
      atomicAdd(p.dk_acc + off + dt * 8, dk[dt][2 * h]);
      atomicAdd(p.dk_acc + off + dt * 8 + 1, dk[dt][2 * h + 1]);
      atomicAdd(p.dv_acc + off + dt * 8, dv[dt][2 * h]);
      atomicAdd(p.dv_acc + off + dt * 8 + 1, dv[dt][2 * h + 1]);
    }
  }
}

// Per-row statistics of both kernels, [B, nh, Spad] (Spad = S rounded up to 64, so that every 64-row q tile's rows are one
// 16-byte-aligned block for any S):
//   delta[b, h, s] = sum_d dO[b,s,h,d] * O[b,s,h,d]      (D / 8 lanes per row)
//   lse2[b, h, s]  = lse[b, h, s] * log2(e)
// padding rows s >= S get delta = 0 and lse2 = +inf, so P = 0 there.
template <int D>
__global__ void fa_bwd_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout, const float* __restrict__ lse,
                                    float* __restrict__ lse2, float* __restrict__ delta, int B, int S, int Spad, int nh,
                                    int64_t ldo, int64_t lddo) {
  constexpr int LPR = D / 8, LPR_LOG2 = D == 128 ? 4 : 3;   // lanes per row
  const int64_t row = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> LPR_LOG2;   // (b, s < Spad, h) flattened
  const int sub = threadIdx.x & (LPR - 1);
  const int64_t total = static_cast<int64_t>(B) * Spad * nh;
  float acc = 0.f;
  int b = 0, s = 0, h = 0;
  if (row < total) {
    h = static_cast<int>(row % nh);
    s = static_cast<int>((row / nh) % Spad);
    b = static_cast<int>(row / nh / Spad);
  }
  if (row < total && s < S) {
    const int64_t tok = static_cast<int64_t>(b) * S + s;
    const uint4 ov = ld_nc_v4(reinterpret_cast<const uint4*>(o + tok * ldo + h * D) + sub);
    const uint4 dv = ld_nc_v4(reinterpret_cast<const uint4*>(dout + tok * lddo + h * D) + sub);
    const uint32_t* oi = reinterpret_cast<const uint32_t*>(&ov);
    const uint32_t* di = reinterpret_cast<const uint32_t*>(&dv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16x2(oi[j]), d = unpack_bf16x2(di[j]);
      acc += a.x * d.x + a.y * d.y;
    }
  }
#pragma unroll
  for (int off = LPR / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (row < total && sub == 0) {
    const size_t bh = static_cast<size_t>(b) * nh + h;
    delta[bh * Spad + s] = acc;
    lse2[bh * Spad + s] = s < S ? lse[bh * S + s] * 1.4426950408889634f : INFINITY;
  }
}

// out (bf16, token stride ld) = bf16(acc fp32 [tokens, width])
__global__ void fa_bwd_dq_finish_kernel(const float* __restrict__ acc, bf16* __restrict__ dq, int64_t tokens, int width,
                                        int64_t lddq) {
  const int64_t nchunk_row = width >> 3;
  const int64_t total = tokens * nchunk_row;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t t = i / nchunk_row, c = i % nchunk_row;
    const float4* src = reinterpret_cast<const float4*>(acc + t * width) + 2 * c;
    const float4 a = src[0], b = src[1];
    uint4 o;
    o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
    o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
    *(reinterpret_cast<uint4*>(dq + t * lddq) + c) = o;
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// impl 2: warp-specialised wgmma kernel
// ------------------------------------------------------------------------------------------------------------------------
namespace wg {
constexpr int BKV = 128;                                  // kv rows per CTA, 64 per consumer warpgroup
constexpr int BQ = 64;                                    // q rows per ring stage
constexpr int STAGES = 2;
constexpr int NUM_THREADS = 256;                          // two warpgroups, 64 kv rows each
constexpr int HK = BKV * 64 * 2;                          // one swizzled [128 kv rows][64 d] block of K or V
constexpr int HQ = BQ * 64 * 2;                           // one swizzled [64 q rows][64 d] block of Q or dO

// shared-memory layout at head_dim D
template <int D>
struct Layout {
  static constexpr int KV_BYTES = BKV * D * 2;                       // K or V: D / 64 blocks of HK bytes
  static constexpr int QT_BYTES = BQ * D * 2;                        // Q or dO tile: D / 64 blocks of HQ bytes
  static constexpr int STAGE_BYTES = 2 * QT_BYTES + 2 * BQ * 4;      // Q, dO, lse2, delta
  static constexpr int STAGE_STRIDE = (STAGE_BYTES + 1023) / 1024 * 1024;   // every stage 1024-byte aligned (swizzle atoms)
  static constexpr int DS_BYTES = BKV * BQ * 2;                      // dS^T [128 kv][64 q] bf16
  static constexpr int DQ_BYTES = BQ * 64 * 4;                       // one warpgroup's fp32 dQ tile: two [64 q][32 d] boxes
  static constexpr int OFF_K = 0, OFF_V = KV_BYTES, OFF_RING = 2 * KV_BYTES;
  static constexpr int OFF_DS = OFF_RING + STAGES * STAGE_STRIDE;    // two dS^T buffers (alternate q tiles)
  static constexpr int OFF_DQ = OFF_DS + 2 * DS_BYTES;
  static constexpr int OFF_BAR = OFF_DQ + 2 * DQ_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;             // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 227 * 1024, "fa_bwd_wgmma: shared memory");
  // the final dK / dV staging (64 rows x D fp32 per warpgroup) reuses a ring stage, the dS buffers and the dQ buffers
  static_assert(64 * D * 4 <= STAGE_STRIDE && 64 * D * 4 <= 2 * DS_BYTES && 64 * D * 4 <= 2 * DQ_BYTES,
                "fa_bwd_wgmma: shared-memory layout");
};
static_assert(Layout<128>::STAGE_STRIDE == 33 * 1024, "fa_bwd_wgmma: head_dim 128 layout");

struct Params {
  int S, nh, kvh, Spad;
  float scale, scale_log2;
  const float* lse2;       // [B, nh, Spad] (fa_bwd_delta_kernel)
  const float* delta;
  const int* mask_start;   // [B, S] or nullptr
};

// Compiler-level fence on registers that wgmma reads or writes asynchronously: no access may be scheduled across it.
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// fp32 accumulator fragment of one warpgroup (64 rows x 8 NJ columns; register 4j + 2i + e = row 16 wi + lane/4 + 8i,
// column 8j + 2 (lane % 4) + e) -> NJ/4 boxes of [64 rows][32 columns], 128-byte swizzled as the fp32 tensor maps expect.
template <int NJ>
__device__ __forceinline__ void stage_f32(uint32_t base, const float (&acc)[4 * NJ], int wi, int lane) {
  const int g = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wi * 16 + g + 8 * i;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int chunk = (j & 3) * 2 + (tq >> 1);
      const uint32_t a = base + (j >> 2) * (64 * 128) + row * 128 + ((chunk ^ (row & 7)) << 4) + (tq & 1) * 8;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(acc[4 * j + 2 * i]), "f"(acc[4 * j + 2 * i + 1]) : "memory");
    }
  }
}

template <int D, bool MASK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
fa_bwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                    const __grid_constant__ CUtensorMap tmdQ, const __grid_constant__ CUtensorMap tmdK,
                    const __grid_constant__ CUtensorMap tmdV, const Params p) {
  using L = Layout<D>;
  constexpr int KV_BYTES = L::KV_BYTES, QT_BYTES = L::QT_BYTES, STAGE_BYTES = L::STAGE_BYTES, STAGE_STRIDE = L::STAGE_STRIDE;
  constexpr int DS_BYTES = L::DS_BYTES, DQ_BYTES = L::DQ_BYTES;
  constexpr int OFF_K = L::OFF_K, OFF_V = L::OFF_V, OFF_RING = L::OFF_RING, OFF_DS = L::OFF_DS, OFF_DQ = L::OFF_DQ, OFF_BAR = L::OFF_BAR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                              // [STAGES]
  uint64_t* kv_bar = empty_bar + STAGES;

  const int head = static_cast<int>(blockIdx.x) % p.nh, batch = static_cast<int>(blockIdx.x) / p.nh;
  const int kv_head = head / (p.nh / p.kvh);
  const int kv0 = static_cast<int>(blockIdx.y) * BKV;   // grid.y: early kv tiles see the most q rows (causal) and go first
  int q_lo = kv0 / BQ, q_hi = (p.S + BQ - 1) / BQ;
  if constexpr (MASK) {   // rows at or past the last column's document end see none of this tile
    const int last = __ldg(p.mask_start + static_cast<size_t>(batch) * p.S + min(kv0 + BKV - 1, p.S - 1));
    q_hi = min(q_hi, (last + BQ - 1) / BQ);
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
    tma_prefetch_desc(&tmdQ); tma_prefetch_desc(&tmdK); tma_prefetch_desc(&tmdV);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);
    }
    mbar_init(kv_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  // Thread 0 also issues the TMA loads: K and V once, then each q tile into the ring (see the refill in the loop).  A separate
  // producer warpgroup would make the CTA 384 threads, which caps ptxas at 168 registers per thread for the whole kernel
  // (setmaxnreg does not raise the allocation limit); the warpgroups' dK / dV accumulators alone take 128 of them.
  const size_t stat0 = (static_cast<size_t>(batch) * p.nh + head) * p.Spad;
  auto load_q_tile = [&](int qt, int st) {
    uint8_t* sq = smem + OFF_RING + st * STAGE_STRIDE;
    mbar_arrive_expect_tx(&full_bar[st], STAGE_BYTES);
#pragma unroll
    for (int h = 0; h < D / 64; ++h) {
      tma_load_4d(&tmQ, &full_bar[st], sq + h * HQ, h * 64, head, qt * BQ, batch);
      tma_load_4d(&tmdO, &full_bar[st], sq + QT_BYTES + h * HQ, h * 64, head, qt * BQ, batch);
    }
    bulk_load(sq + 2 * QT_BYTES, p.lse2 + stat0 + qt * BQ, BQ * 4, &full_bar[st]);
    bulk_load(sq + 2 * QT_BYTES + BQ * 4, p.delta + stat0 + qt * BQ, BQ * 4, &full_bar[st]);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(kv_bar, 2 * KV_BYTES);
#pragma unroll
    for (int h = 0; h < D / 64; ++h) {
      tma_load_4d(&tmK, kv_bar, smem + OFF_K + h * HK, h * 64, kv_head, kv0, batch);
      tma_load_4d(&tmV, kv_bar, smem + OFF_V + h * HK, h * 64, kv_head, kv0, batch);
    }
    for (int i = 0; i < STAGES && q_lo + i < q_hi; ++i) load_q_tile(q_lo + i, i);
  }

  const int cw = threadIdx.x >> 7;                          // warpgroup = 64-row half of the kv tile
  const int wi = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;             // issues (and waits for) this warpgroup's TMA reduce-adds
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sK = sbase + OFF_K, sV = sbase + OFF_V;
  const int kv_r = kv0 + cw * 64 + wi * 16 + g;             // kv row of accumulator rows i = 0 (and + 8 for i = 1)
  int ms[2] = {INT_MAX, INT_MAX};
  if constexpr (MASK) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (kv_r + 8 * i < p.S) ms[i] = __ldg(p.mask_start + static_cast<size_t>(batch) * p.S + kv_r + 8 * i);
  }
  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait_nocall(kv_bar, 0);

  for (int qt = q_lo, it = 0; qt < q_hi; ++qt, ++it) {
    const int st = it % STAGES, q0 = qt * BQ;
    const uint32_t sQ = sbase + OFF_RING + st * STAGE_STRIDE, sdO = sQ + QT_BYTES;
    const float* s_lse = reinterpret_cast<const float*>(smem + OFF_RING + st * STAGE_STRIDE + 2 * QT_BYTES);
    const float* s_delta = s_lse + BQ;
    if (threadIdx.x == 0 && it > 0 && qt - 1 + STAGES < q_hi) {
      // refill: the stage of q tile it - 1 takes tile it - 1 + STAGES once both warpgroups have released it
      const int ps = (it - 1) % STAGES;
      mbar_wait_nocall(&empty_bar[ps], ((it - 1) / STAGES) & 1);
      load_q_tile(qt - 1 + STAGES, ps);
    }
    mbar_wait_nocall(&full_bar[st], (it / STAGES) & 1);

    // S^T = K Q^T: [64 kv] x [64 q], both operands K-major (d contiguous)
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ko = (kk >> 2) * HK + cw * 64 * 128 + (kk & 3) * 32, qo = (kk >> 2) * HQ + (kk & 3) * 32;
      wgmma_m64n64k16<0, 0>(s, wgmma_desc_sw128(sK + ko, 16, 1024), wgmma_desc_sw128(sQ + qo, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    // P^T = exp2(S^T scale log2(e) - lse2), dead where kv > q (causal) or q >= the kv column's FlashMask start row
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + 2 * tq + e, r = q0 + c;
        const float l2 = s_lse[c];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          bool dead = kv_r + 8 * i > r;
          if constexpr (MASK) dead = dead || r >= ms[i];
          float& x = s[4 * j + 2 * i + e];
          x = dead ? 0.f : fast_exp2(fmaf(x, p.scale_log2, -l2));
        }
      }
    }
    // dP^T = V dO^T (as S^T)
    float dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ko = (kk >> 2) * HK + cw * 64 * 128 + (kk & 3) * 32, qo = (kk >> 2) * HQ + (kk & 3) * 32;
      wgmma_m64n64k16<0, 0>(dp, wgmma_desc_sw128(sV + ko, 16, 1024), wgmma_desc_sw128(sdO + qo, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dp);
    // dS^T = P^T o (dP^T - delta) * scale
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float dl = s_delta[8 * j + 2 * tq + e];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float& x = dp[4 * j + 2 * i + e];
          x = s[4 * j + 2 * i + e] * (x - dl) * p.scale;
        }
      }
    }
    // bf16 A fragments: register pair t = (2j + i) holds row 16 wi + g + 8i, columns 8j + 2 tq + {0, 1}; k-step k = t / 4
    uint32_t pa[16], da[16];
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      pa[t] = pack_bf16x2(s[2 * t], s[2 * t + 1]);
      da[t] = pack_bf16x2(dp[2 * t], dp[2 * t + 1]);
    }
    // dV += P^T dO, dK += dS^T Q: B = dO / Q, MN-major (d contiguous), k = 16 q rows = 2048 bytes
    wgmma_fence();
    if constexpr (D == 128) {
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n128k16_rs<1>(dv, pa + 4 * k, wgmma_desc_sw128(sdO + k * 2048, HQ, 1024), 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n128k16_rs<1>(dk, da + 4 * k, wgmma_desc_sw128(sQ + k * 2048, HQ, 1024), 1u);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64k16_rs<1>(dv, pa + 4 * k, wgmma_desc_sw128(sdO + k * 2048, HQ, 1024), 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64k16_rs<1>(dk, da + 4 * k, wgmma_desc_sw128(sQ + k * 2048, HQ, 1024), 1u);
    }
    wgmma_commit();
    // dS^T -> shared memory, [128 kv][64 q] bf16, 128-byte swizzle: the MN-major A operand of dQ = dS K
    const uint32_t sdS = sbase + OFF_DS + (it & 1) * DS_BYTES;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = cw * 64 + wi * 16 + g + 8 * i;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sdS + row * 128 + ((j ^ (row & 7)) << 4) + tq * 4), "r"(da[2 * j + i]) : "memory");
    }
    fence_proxy_async_smem();
    float dq[32];   // no initial value: the first wgmma (accumulate = 0) overwrites it
    if constexpr (D == 128) {
      named_bar_sync(1, 256);   // both warpgroups' dS^T rows are in shared memory
      // dQ[64 q][64 d of this warpgroup] = dS K: A = dS^T buffer (MN-major), B = K half cw (MN-major), k = 16 kv rows
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_m64n64k16<1, 1>(dq, wgmma_desc_sw128(sdS + kk * 2048, DS_BYTES, 1024),
                              wgmma_desc_sw128(sK + cw * HK + kk * 2048, HK, 1024), kk > 0 ? 1u : 0u);
    } else {
      named_bar_sync(2 + cw, 128);   // this warpgroup's dS^T rows are in shared memory
      // dQ partial [64 q][64 d] = dS[:, this warpgroup's 64 kv rows] K[those rows, :]
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16<1, 1>(dq, wgmma_desc_sw128(sdS + cw * 64 * 128 + kk * 2048, DS_BYTES, 1024),
                              wgmma_desc_sw128(sK + cw * 64 * 128 + kk * 2048, HK, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dq);
    reg_fence(dk);
    reg_fence(dv);
    mbar_arrive(&empty_bar[st]);   // Q, dO and the statistics of this stage are consumed
    // dQ tile -> fp32 staging -> one TMA reduce-add per 32 d columns into the dQ buffer (rows past S are clipped)
    uint8_t* sdq = smem + OFF_DQ + cw * DQ_BYTES;
    if (leader) tma_store_wait_read<0>();   // the previous tile's reduce has read the staging buffer
    named_bar_sync(2 + cw, 128);
    stage_f32<8>(smem_u32(sdq), dq, wi, lane);
    fence_proxy_async_smem();
    named_bar_sync(2 + cw, 128);
    if (leader) {
      const int d0 = D == 128 ? cw * 64 : 0;
      tma_reduce_add_4d(&tmdQ, sdq, d0, head, q0, batch);
      tma_reduce_add_4d(&tmdQ, sdq + DQ_BYTES / 2, d0 + 32, head, q0, batch);
      tma_store_commit();
    }
  }

  // this head's dK / dV partials -> the kv head's fp32 buffers (the GQA group's heads add up there), staged in the ring
  // (dK) and in the dS / dQ buffers (dV), which no warpgroup reads any more after this barrier
  if (leader) tma_store_wait_read<0>();
  named_bar_sync(1, 256);
  uint8_t* sdk = smem + OFF_RING + cw * STAGE_STRIDE;
  uint8_t* sdv = smem + (cw == 0 ? OFF_DS : OFF_DQ);
  stage_f32<D / 8>(smem_u32(sdk), dk, wi, lane);
  stage_f32<D / 8>(smem_u32(sdv), dv, wi, lane);
  fence_proxy_async_smem();
  named_bar_sync(2 + cw, 128);
  if (leader) {
#pragma unroll
    for (int b = 0; b < D / 32; ++b) {
      tma_reduce_add_4d(&tmdK, sdk + b * (64 * 128), b * 32, kv_head, kv0 + cw * 64, batch);
      tma_reduce_add_4d(&tmdV, sdv + b * (64 * 128), b * 32, kv_head, kv0 + cw * 64, batch);
    }
    tma_store_commit();
    tma_store_wait<0>();
  }
}

// [B, S, heads, D] fp32 accumulation buffer, box {32 d, 1 head, 64 rows, 1}
static int make_f32_map(CUtensorMap* tm, float* base, int64_t B, int64_t S, int64_t heads, int64_t D) {
  const uint64_t dims[4] = {static_cast<uint64_t>(D), static_cast<uint64_t>(heads), static_cast<uint64_t>(S), static_cast<uint64_t>(B)};
  const uint64_t row = static_cast<uint64_t>(D) * 4;
  const uint64_t strides[3] = {row, static_cast<uint64_t>(heads) * row, static_cast<uint64_t>(S * heads) * row};
  const uint32_t box[4] = {32, 1, 64, 1};
  return encode_tmap_f32(tm, base, 4, dims, strides, box);
}

template <int D, bool MASK>
static int launch(const CUtensorMap (&tm)[7], const Params& p, int B, cudaStream_t stream) {
  constexpr int SMEM_BYTES = Layout<D>::SMEM_BYTES;
  auto kern = fa_bwd_wgmma_kernel<D, MASK>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      set_last_error("fa_bwd_wgmma smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  const dim3 grid(static_cast<unsigned>(p.nh * B), static_cast<unsigned>((p.S + BKV - 1) / BKV));
  kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], tm[6], p);
  return check_launch("fa_bwd_wgmma");
}
}  // namespace wg

template <int D, int BQ, bool MASK>
static int launch(const Params& p, cudaStream_t stream) {
  constexpr int SMEM = 2 * BKV * D * 2 + 2 * BQ * D * 2 + 2 * BQ * 128 + 2 * BQ * 4;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(fa_bwd_kernel<D, BQ, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("fa_bwd smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  dim3 grid(static_cast<unsigned>((p.S + BKV - 1) / BKV), static_cast<unsigned>(p.nh), static_cast<unsigned>(p.B));
  fa_bwd_kernel<D, BQ, MASK><<<grid, NUM_THREADS, SMEM, stream>>>(p);
  return check_launch("fa_bwd");
}

}  // namespace fab
}  // namespace b200

extern "C" int64_t b200_fa_bwd_workspace_bytes(int64_t B, int64_t S, int64_t num_heads, int64_t head_dim) {
  // fp32 dQ accumulation buffer + fp32 dK/dV accumulation buffers (at most num_heads wide) + per-row statistics (the sequence padded
  // to a multiple of 64, two floats per row)
  const int64_t Spad = (S + 63) / 64 * 64;
  return 3 * B * Spad * num_heads * head_dim * 4 + B * num_heads * Spad * 8;
}

extern "C" int b200_fa_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                           void* dq, void* dk, void* dv, void* workspace, int64_t B, int64_t S, int64_t num_heads,
                           int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                           int64_t lddo, int64_t lddq, int64_t lddk, int64_t lddv, float softmax_scale,
                           cudaStream_t stream) {
  return b200_fa_bwd_flashmask(q, k, v, o, dout, lse, nullptr, dq, dk, dv, workspace, B, S, num_heads, num_kv_heads, head_dim,
                               ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv, softmax_scale, stream);
}

extern "C" int b200_fa_bwd_flashmask(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                     const float* lse, const int32_t* mask_start_rows, void* dq, void* dk, void* dv,
                                     void* workspace, int64_t B, int64_t S, int64_t num_heads, int64_t num_kv_heads,
                                     int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, int64_t lddo,
                                     int64_t lddq, int64_t lddk, int64_t lddv, float softmax_scale, cudaStream_t stream) {
  using namespace b200;
  using namespace b200::fab;
  B200_CHECK_ARG(q && k && v && o && dout && lse && dq && dk && dv && workspace, "fa_bwd: null pointer");
  B200_CHECK_ARG(head_dim == 64 || head_dim == 128, "fa_bwd: head_dim must be 64 or 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && S > 0 && num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0, "fa_bwd: bad shape");
  B200_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                     lddk % 8 == 0 && lddv % 8 == 0,
                 "fa_bwd: token strides must be multiples of 8");
  {
    // TMA (impl 2) and cp.async / 16-byte vector loads (impl 1) address rows in 16-byte units
    const void* ptrs[8] = {q, k, v, o, dout, dq, dk, dv};
    const char* names[8] = {"q", "k", "v", "o", "dout", "dq", "dk", "dv"};
    for (int i = 0; i < 8; ++i)
      B200_CHECK_ARG((reinterpret_cast<uintptr_t>(ptrs[i]) & 15) == 0, "fa_bwd: %s must be 16-byte aligned (got %p)", names[i], ptrs[i]);
  }
  const int64_t Spad = (S + 63) / 64 * 64;
  float* dq_acc = static_cast<float*>(workspace);
  float* dk_acc = dq_acc + B * S * num_heads * head_dim;
  float* dv_acc = dk_acc + B * S * num_kv_heads * head_dim;
  float* lse2 = dq_acc + 3 * B * S * num_heads * head_dim;
  float* delta = lse2 + B * num_heads * Spad;
  cudaError_t e = cudaMemsetAsync(dq_acc, 0, static_cast<size_t>(B) * S * (num_heads + 2 * num_kv_heads) * head_dim * 4, stream);
  if (e != cudaSuccess) {
    set_last_error("fa_bwd memset: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  {
    const int64_t rows = B * Spad * num_heads;
    const int64_t threads = rows * (head_dim / 8);
    const unsigned blocks = static_cast<unsigned>((threads + 255) / 256);
    const bf16 *op = static_cast<const bf16*>(o), *dop = static_cast<const bf16*>(dout);
    if (head_dim == 64)
      fa_bwd_delta_kernel<64><<<blocks, 256, 0, stream>>>(op, dop, lse, lse2, delta, (int)B, (int)S, (int)Spad, (int)num_heads, ldo, lddo);
    else
      fa_bwd_delta_kernel<128><<<blocks, 256, 0, stream>>>(op, dop, lse, lse2, delta, (int)B, (int)S, (int)Spad, (int)num_heads, ldo, lddo);
    int rc = check_launch("fa_bwd(delta)");
    if (rc) return rc;
  }
  int rc;
  if (fa_bwd_impl() == 1) {
    Params p;
    p.q = static_cast<const bf16*>(q); p.k = static_cast<const bf16*>(k); p.v = static_cast<const bf16*>(v);
    p.dout = static_cast<const bf16*>(dout);
    p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.lddo = lddo;
    p.S = (int)S; p.B = (int)B; p.nh = (int)num_heads; p.kvh = (int)num_kv_heads; p.Spad = (int)Spad;
    p.scale = softmax_scale;
    p.scale_log2 = softmax_scale * 1.4426950408889634f;
    p.lse2 = lse2; p.delta = delta;
    p.mask_start = mask_start_rows;
    p.dq_acc = dq_acc; p.dk_acc = dk_acc; p.dv_acc = dv_acc;
    if (head_dim == 64)
      rc = mask_start_rows ? launch<64, 64, true>(p, stream) : launch<64, 64, false>(p, stream);
    else
      rc = mask_start_rows ? launch<128, 64, true>(p, stream) : launch<128, 64, false>(p, stream);
  } else {
    CUtensorMap tm[7];
    if ((rc = make_bf16_map(&tm[0], q, B, S, num_heads, head_dim, ldq, wg::BQ)) != 0) return rc;
    if ((rc = make_bf16_map(&tm[1], k, B, S, num_kv_heads, head_dim, ldk, wg::BKV)) != 0) return rc;
    if ((rc = make_bf16_map(&tm[2], v, B, S, num_kv_heads, head_dim, ldv, wg::BKV)) != 0) return rc;
    if ((rc = make_bf16_map(&tm[3], dout, B, S, num_heads, head_dim, lddo, wg::BQ)) != 0) return rc;
    if ((rc = wg::make_f32_map(&tm[4], dq_acc, B, S, num_heads, head_dim)) != 0) return rc;
    if ((rc = wg::make_f32_map(&tm[5], dk_acc, B, S, num_kv_heads, head_dim)) != 0) return rc;
    if ((rc = wg::make_f32_map(&tm[6], dv_acc, B, S, num_kv_heads, head_dim)) != 0) return rc;
    wg::Params p;
    p.S = (int)S; p.nh = (int)num_heads; p.kvh = (int)num_kv_heads; p.Spad = (int)Spad;
    p.scale = softmax_scale;
    p.scale_log2 = softmax_scale * 1.4426950408889634f;
    p.lse2 = lse2; p.delta = delta;
    p.mask_start = mask_start_rows;
    if (head_dim == 64)
      rc = mask_start_rows ? wg::launch<64, true>(tm, p, (int)B, stream) : wg::launch<64, false>(tm, p, (int)B, stream);
    else
      rc = mask_start_rows ? wg::launch<128, true>(tm, p, (int)B, stream) : wg::launch<128, false>(tm, p, (int)B, stream);
  }
  if (rc) return rc;
  {
    const int64_t tokens = B * S;
    const int width = static_cast<int>(num_heads * head_dim);
    const int64_t total = tokens * (width / 8);
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
    if (blocks > cap) blocks = cap;
    fa_bwd_dq_finish_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(dq_acc, static_cast<bf16*>(dq), tokens,
                                                                              width, lddq);
    if ((rc = check_launch("fa_bwd(dq finish)")) != 0) return rc;
    const int kvw = static_cast<int>(num_kv_heads * head_dim);
    int64_t kblocks = (tokens * (kvw / 8) + 255) / 256;
    if (kblocks > cap) kblocks = cap;
    fa_bwd_dq_finish_kernel<<<static_cast<unsigned>(kblocks), 256, 0, stream>>>(dk_acc, static_cast<bf16*>(dk), tokens, kvw,
                                                                               lddk);
    if ((rc = check_launch("fa_bwd(dk finish)")) != 0) return rc;
    fa_bwd_dq_finish_kernel<<<static_cast<unsigned>(kblocks), 256, 0, stream>>>(dv_acc, static_cast<bf16*>(dv), tokens, kvw,
                                                                               lddv);
    rc = check_launch("fa_bwd(dv finish)");
  }
  return rc;
}
