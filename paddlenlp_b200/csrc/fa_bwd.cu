// Causal GQA flash-attention backward on Hopper tensor cores (mma.sync m16n8k16, head_dim 128).
//
//   inputs : q, k, v, o, do, lse            outputs: dq, dk, dv (bf16; fp32 accumulation buffers in the workspace)
//   P = exp(S*scale - lse) ; dP = dO V^T ; dS = P o (dP - D) * scale, D = rowsum(dO o O)
//   dV = P^T dO ; dK = dS^T Q ; dQ = dS K
//
// Replaces Paddle-core flash_attn_grad (reference: fusion_ops.py:240-246 backward of scaled_dot_product_attention;
// wrapper shape in csrc/gpu/flash_attn_bwd.cc:22-92).
//
// One CTA (8 warps) = one (batch, q-head, 64-row kv tile); it loops over the q tiles of BQ rows that can see the kv tile
// (b200_set_fa_bwd_impl: 2 = 128-row q tiles, 1 = 64-row q tiles), keeping this head's dK / dV tile in registers.  Per q tile:
//   phase 1   S and dP (BQ x 64) per warp in registers -> P, dS rounded to bf16 into shared memory
//   phase 2   dV += P^T dO, dK += dS^T Q (operands transposed by ldmatrix.trans), dQ = dS K added to the fp32 dQ buffer
// Work units are per q-head (not per kv-head) so that the GQA group's heads spread over the SMs; their dK/dV partials and the
// dQ tiles are reduced into fp32 buffers with atomic adds, then converted to bf16 by a finishing kernel.
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace fab {

constexpr int D = 128;
constexpr int BKV = 64;
constexpr int NUM_THREADS = 256;

struct Params {
  const bf16 *q, *k, *v, *dout;
  int64_t ldq, ldk, ldv, lddo;
  int S, B, nh, kvh;
  float scale, scale_log2;
  const float* lse;     // [B, nh, S]  natural log
  const float* delta;   // [B, nh, S]  rowsum(dO o O)
  const int* mask_start;   // FlashMask causal-LT start rows [B, S] (see fa_fwd.cu) or nullptr
  float* dq_acc;        // [B, S, nh, 128]
  float* dk_acc;        // [B, S, kvh, 128]
  float* dv_acc;
};

// [rows][128] bf16 tiles: 16-byte chunks XOR-swizzled by row & 7 (as fa_fwd.cu); [rows][64] tiles (P, dS): 128-byte rows
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return static_cast<uint32_t>(row * 256 + ((chunk ^ (row & 7)) << 4)); }
__device__ __forceinline__ uint32_t swz64(int row, int chunk) { return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4)); }

template <int BQ, bool MASK>
__global__ void __launch_bounds__(NUM_THREADS, 1) fa_bwd_kernel(const Params p) {
  constexpr int RG = BQ / 16;            // phase 1: row groups of 16 q rows
  constexpr int CH = 8 / RG;             //          column slices of the 64 kv columns
  constexpr int NT = 8 / CH;             //          8-column n-tiles per warp
  constexpr int QG = BQ / 16;            // dQ: row groups
  constexpr int DH = 8 / QG;             //     d slices
  constexpr int DTQ = 16 / DH;           //     8-column d tiles per warp
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sK = smem_u32(smem), sV = sK + BKV * 256, sQ = sV + BKV * 256, sdO = sQ + BQ * 256;
  const uint32_t sP = sdO + BQ * 256, sdS = sP + BQ * 128;
  float* s_lse = reinterpret_cast<float*>(smem + 2 * BKV * 256 + 2 * BQ * 256 + 2 * BQ * 128);
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
  for (int i = threadIdx.x; i < BKV * 16; i += NUM_THREADS) {
    const int r = i >> 4, ch = i & 15;
    const bool ok = kv0 + r < p.S;
    cp_async_16(sK + swz(r, ch), ok ? p.k + (tok0 + kv0 + r) * p.ldk + kv_head * D + ch * 8 : p.k, ok ? 16u : 0u);
    cp_async_16(sV + swz(r, ch), ok ? p.v + (tok0 + kv0 + r) * p.ldv + kv_head * D + ch * 8 : p.v, ok ? 16u : 0u);
  }
  // dK / dV accumulators: warp = 16 kv rows (kg) x 64 d columns (dh)
  const int kg = warp >> 1, dh = warp & 1;
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;

  for (int qt = q_lo; qt < q_hi; ++qt) {
    const int q0 = qt * BQ;
    for (int i = threadIdx.x; i < BQ * 16; i += NUM_THREADS) {
      const int r = i >> 4, ch = i & 15;
      const bool ok = q0 + r < p.S;
      cp_async_16(sQ + swz(r, ch), ok ? p.q + (tok0 + q0 + r) * p.ldq + head * D + ch * 8 : p.q, ok ? 16u : 0u);
      cp_async_16(sdO + swz(r, ch), ok ? p.dout + (tok0 + q0 + r) * p.lddo + head * D + ch * 8 : p.dout, ok ? 16u : 0u);
    }
    cp_async_commit();
    for (int i = threadIdx.x; i < BQ; i += NUM_THREADS) {
      const bool ok = q0 + i < p.S;
      const size_t idx = (static_cast<size_t>(batch) * p.nh + head) * p.S + q0 + i;
      s_lse[i] = ok ? __ldg(p.lse + idx) * 1.4426950408889634f : INFINITY;   // rows past S: P = 0
      s_delta[i] = ok ? __ldg(p.delta + idx) : 0.f;
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
      for (int kc = 0; kc < 8; ++kc) {
        uint32_t a[4], ad[4];
        ldsm_x4(sQ + swz(rg * 16 + (lane & 15), kc * 2 + (lane >> 4)), a);
        ldsm_x4(sdO + swz(rg * 16 + (lane & 15), kc * 2 + (lane >> 4)), ad);
#pragma unroll
        for (int np = 0; np < NT / 2; ++np) {
          const int kr = cs * NT * 8 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
          uint32_t b[4], bv[4];
          ldsm_x4(sK + swz(kr, kc * 2 + ((lane >> 3) & 1)), b);
          ldsm_x4(sV + swz(kr, kc * 2 + ((lane >> 3) & 1)), bv);
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
      for (int dp2 = 0; dp2 < 4; ++dp2) {
        const int br = qc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, bc = dh * 8 + dp2 * 2 + (lane >> 4);
        uint32_t bo[4], bq[4];
        ldsm_x4_t(sdO + swz(br, bc), bo);
        ldsm_x4_t(sQ + swz(br, bc), bq);
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
          ldsm_x4_t(sK + swz(kc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dsl * (DTQ) + dp2 * 2 + (lane >> 4)), b);
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
    const size_t off = ((tok0 + r) * p.kvh + kv_head) * D + dh * 64 + 2 * tq;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      atomicAdd(p.dk_acc + off + dt * 8, dk[dt][2 * h]);
      atomicAdd(p.dk_acc + off + dt * 8 + 1, dk[dt][2 * h + 1]);
      atomicAdd(p.dv_acc + off + dt * 8, dv[dt][2 * h]);
      atomicAdd(p.dv_acc + off + dt * 8 + 1, dv[dt][2 * h + 1]);
    }
  }
}

// delta[b, h, s] = sum_d dO[b,s,h,d] * O[b,s,h,d]      (16 lanes per row of 128)
__global__ void fa_bwd_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout, float* __restrict__ delta,
                                    int B, int S, int nh, int64_t ldo, int64_t lddo) {
  const int64_t row = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 4;   // (b, s, h) flattened
  const int sub = threadIdx.x & 15;
  const int64_t total = static_cast<int64_t>(B) * S * nh;
  float acc = 0.f;
  int b = 0, s = 0, h = 0;
  if (row < total) {
    h = static_cast<int>(row % nh);
    const int64_t tok = row / nh;
    s = static_cast<int>(tok % S);
    b = static_cast<int>(tok / S);
    const uint4 ov = ld_nc_v4(reinterpret_cast<const uint4*>(o + tok * ldo + h * 128) + sub);
    const uint4 dv = ld_nc_v4(reinterpret_cast<const uint4*>(dout + tok * lddo + h * 128) + sub);
    const uint32_t* oi = reinterpret_cast<const uint32_t*>(&ov);
    const uint32_t* di = reinterpret_cast<const uint32_t*>(&dv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16x2(oi[j]), d = unpack_bf16x2(di[j]);
      acc += a.x * d.x + a.y * d.y;
    }
  }
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (row < total && sub == 0) delta[(static_cast<size_t>(b) * nh + h) * S + s] = acc;
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

template <int BQ, bool MASK>
static int launch(const Params& p, cudaStream_t stream) {
  constexpr int SMEM = 2 * BKV * 256 + 2 * BQ * 256 + 2 * BQ * 128 + 2 * BQ * 4;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(fa_bwd_kernel<BQ, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("fa_bwd smem attr: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    attr_set = true;
  }
  dim3 grid(static_cast<unsigned>((p.S + BKV - 1) / BKV), static_cast<unsigned>(p.nh), static_cast<unsigned>(p.B));
  fa_bwd_kernel<BQ, MASK><<<grid, NUM_THREADS, SMEM, stream>>>(p);
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
  B200_CHECK_ARG(head_dim == 128, "fa_bwd: head_dim must be 128 (got %lld)", (long long)head_dim);
  B200_CHECK_ARG(B > 0 && S > 0 && num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0, "fa_bwd: bad shape");
  B200_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                     lddk % 8 == 0 && lddv % 8 == 0,
                 "fa_bwd: token strides must be multiples of 8");
  float* dq_acc = static_cast<float*>(workspace);
  float* dk_acc = dq_acc + B * S * num_heads * 128;
  float* dv_acc = dk_acc + B * S * num_kv_heads * 128;
  float* delta = dq_acc + 3 * B * S * num_heads * 128;
  cudaError_t e = cudaMemsetAsync(dq_acc, 0, static_cast<size_t>(B) * S * (num_heads + 2 * num_kv_heads) * 128 * 4, stream);
  if (e != cudaSuccess) {
    set_last_error("fa_bwd memset: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  {
    const int64_t rows = B * S * num_heads;
    const int64_t threads = rows * 16;
    fa_bwd_delta_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(
        static_cast<const bf16*>(o), static_cast<const bf16*>(dout), delta, (int)B, (int)S, (int)num_heads, ldo, lddo);
    int rc = check_launch("fa_bwd(delta)");
    if (rc) return rc;
  }
  Params p;
  p.q = static_cast<const bf16*>(q); p.k = static_cast<const bf16*>(k); p.v = static_cast<const bf16*>(v);
  p.dout = static_cast<const bf16*>(dout);
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.lddo = lddo;
  p.S = (int)S; p.B = (int)B; p.nh = (int)num_heads; p.kvh = (int)num_kv_heads;
  p.scale = softmax_scale;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.lse = lse; p.delta = delta;
  p.mask_start = mask_start_rows;
  p.dq_acc = dq_acc; p.dk_acc = dk_acc; p.dv_acc = dv_acc;
  int rc;
  if (fa_bwd_impl() == 1) rc = mask_start_rows ? launch<64, true>(p, stream) : launch<64, false>(p, stream);
  else rc = mask_start_rows ? launch<128, true>(p, stream) : launch<128, false>(p, stream);
  if (rc) return rc;
  {
    const int64_t tokens = B * S;
    const int width = static_cast<int>(num_heads * 128);
    const int64_t total = tokens * (width / 8);
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
    if (blocks > cap) blocks = cap;
    fa_bwd_dq_finish_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(dq_acc, static_cast<bf16*>(dq), tokens,
                                                                              width, lddq);
    if ((rc = check_launch("fa_bwd(dq finish)")) != 0) return rc;
    const int kvw = static_cast<int>(num_kv_heads * 128);
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
