// HBM-bound fusions of the decoder hot path: RMSNorm fwd/bwd, RoPE, SwiGLU fwd/bwd, embedding gather /
// scatter-add, bias-gradient column sums.  All are 128-bit vectorised, fp32 math, ONE rounding to bf16 per output
// (rounding points listed in SURVEY.md §8a).  Roofline for each: algorithmic bytes / measured HBM bandwidth.
#include "../../include/b200nlp.h"
#include <type_traits>
#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace ew {

// ------------------------------------------------------------------------------------------------
// RMSNorm forward.  y = bf16( bf16(x * rstd) * w ),  rstd = rsqrt(mean(x^2) + eps)  (fp32 stats).
// Reference: llama/modeling.py:367-386 (unfused), fusion_ops.py:119-125 -> fused_ln/layer_norm_cuda.h:447-531.
// One warp per row; the row stays in registers between the statistics pass and the scaling pass, so HBM traffic
// is exactly 2 * T * h * 2 bytes.
// ------------------------------------------------------------------------------------------------
template <int MAXV>
__global__ void __launch_bounds__(128) rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                          bf16* __restrict__ y, float* __restrict__ rstd_out,
                                                          int rows, int h, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + warp;
  if (row >= rows) return;
  const int nchunk = h >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * h);
  // branch-free load phase: every 16-byte load of the row is in flight before the first use
  uint4 v[MAXV];
  const int last = nchunk - 1;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) v[i] = ld_nc_v4(xr + min(lane + 32 * i, last));
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const float2 a = unpack_bf16x2(v[i].x), b = unpack_bf16x2(v[i].y), cc = unpack_bf16x2(v[i].z), d = unpack_bf16x2(v[i].w);
    const float part = a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + cc.x * cc.x + cc.y * cc.y + d.x * d.x + d.y * d.y;
    ss += ((lane + 32 * i) < nchunk) ? part : 0.f;
  }
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / static_cast<float>(h) + eps);
  if (lane == 0 && rstd_out != nullptr) rstd_out[row] = rstd;
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * h);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunk) {
      const uint4 wv = __ldg(wr + c);
      uint4 o;
      const uint32_t* xi = reinterpret_cast<const uint32_t*>(&v[i]);
      const uint32_t* wi = reinterpret_cast<const uint32_t*>(&wv);
      uint32_t* oi = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(xi[j]);
        const float2 wf = unpack_bf16x2(wi[j]);
        const float n0 = bf16_round(xf.x * rstd), n1 = bf16_round(xf.y * rstd);
        oi[j] = pack_bf16x2(n0 * wf.x, n1 * wf.y);
      }
      st_na_v4(yr + c, o);
    }
  }
}

// Same op, one CTA (128 threads) per row, persistent over rows: thread t owns the 16-byte chunks t, t + 128, ... (4 per thread at
// h = 4096 instead of 16 per lane in the warp-per-row kernel above: 64 instead of 146 registers, 8 CTAs = this row + the next row of
// each = 16 rows of loads in flight per SM instead of 12), and the NEXT row's loads are issued before this row's reduction.  The warp-per-row kernel ran at
// 4.65 TB/s on [8192, 4096] (ncu); this one is used for h >= 1024.  Summation order: per-thread chunks, warp tree, the four warp
// partials in order (the order of the decode step's add_rmsnorm kernel).
template <int MAXV>
__global__ void __launch_bounds__(128, MAXV <= 4 ? 8 : 4) rmsnorm_fwd_cta_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                              bf16* __restrict__ y, float* __restrict__ rstd_out, int rows, int h,
                                                              float eps) {
  __shared__ float s_part[2][4];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int nchunk = h >> 3;
  const int last = nchunk - 1;
  const uint4* wr = reinterpret_cast<const uint4*>(w);       // re-read per row: 8 KB, L1-resident
  uint4 nxt[MAXV];
  int row = blockIdx.x;
  if (row < rows) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * h);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) nxt[i] = ld_nc_v4(xr + min(t + 128 * i, last));
  }
  for (int it = 0; row < rows; row += gridDim.x, ++it) {
    uint4 v[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) v[i] = nxt[i];
    const int nrow = row + gridDim.x;
    if (nrow < rows) {
      const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(nrow) * h);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) nxt[i] = ld_nc_v4(xr + min(t + 128 * i, last));
    }
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const float2 a = unpack_bf16x2(v[i].x), b = unpack_bf16x2(v[i].y), cc = unpack_bf16x2(v[i].z), d = unpack_bf16x2(v[i].w);
      const float part = a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + cc.x * cc.x + cc.y * cc.y + d.x * d.x + d.y * d.y;
      ss += ((t + 128 * i) < nchunk) ? part : 0.f;
    }
    ss = warp_sum(ss);
    float* sp = s_part[it & 1];                 // double-buffered: one barrier per row
    if (lane == 0) sp[warp] = ss;
    __syncthreads();
    ss = sp[0] + sp[1] + sp[2] + sp[3];
    const float rstd = rsqrtf(ss / static_cast<float>(h) + eps);
    if (t == 0 && rstd_out != nullptr) rstd_out[row] = rstd;
    uint4* yr = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * h);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = t + 128 * i;
      if (c < nchunk) {
        uint4 o;
        const uint4 wv = __ldg(wr + c);
        const uint32_t* xi = reinterpret_cast<const uint32_t*>(&v[i]);
        const uint32_t* wi = reinterpret_cast<const uint32_t*>(&wv);
        uint32_t* oi = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 xf = unpack_bf16x2(xi[j]);
          const float2 wf = unpack_bf16x2(wi[j]);
          const float n0 = bf16_round(xf.x * rstd), n1 = bf16_round(xf.y * rstd);
          oi[j] = pack_bf16x2(n0 * wf.x, n1 * wf.y);
        }
        st_na_v4(yr + c, o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RMSNorm backward (+ fused residual-gradient add).
//   xhat = x * rstd ; g = dy * w ; dx = rstd * (g - xhat * mean(g * xhat)) (+ dres) ; dw_partial += dy * bf16(xhat)
// Reference: fused_ln/layer_norm_cuda.h:1190-1260 (HostRMSNormGradient).
// One CTA per row-slice, thread t owns columns [8t, 8t+8): the per-thread dw partial lives in 8 registers across
// the CTA's rows; partials go to a [gridDim.x, h] fp32 workspace reduced by rmsnorm_dw_reduce_kernel.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                   const bf16* __restrict__ w, const float* __restrict__ rstd,
                                   const bf16* __restrict__ dres, bf16* __restrict__ dx,
                                   float* __restrict__ dw_partial, int rows, int h) {
  __shared__ float red[32];
  const int t = threadIdx.x;
  const int nchunk = h >> 3;
  const bool active = t < nchunk;
  const int warp = t >> 5, lane = t & 31, nwarps = blockDim.x >> 5;
  float wf[8], dwacc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { wf[j] = 0.f; dwacc[j] = 0.f; }
  if (active) {
    const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w) + t);
    const uint32_t* wi = reinterpret_cast<const uint32_t*>(&wv);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = unpack_bf16x2(wi[j]); wf[2 * j] = f.x; wf[2 * j + 1] = f.y; }
  }
  // software pipeline: the next row's x / dy / dres loads are in flight while this row's CTA-wide reduction (two barriers) runs
  uint4 xv_n = make_uint4(0u, 0u, 0u, 0u), dv_n = xv_n, rv_n = xv_n;
  float rs_n = 0.f;
  auto issue = [&](int row) {
    if (row < rows) {
      rs_n = rstd[row];
      if (active) {
        xv_n = ld_nc_v4(reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * h) + t);
        dv_n = ld_nc_v4(reinterpret_cast<const uint4*>(dy + static_cast<size_t>(row) * h) + t);
        if (dres != nullptr) rv_n = ld_nc_v4(reinterpret_cast<const uint4*>(dres + static_cast<size_t>(row) * h) + t);
      }
    }
  };
  issue(blockIdx.x);
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    float xh[8], g[8];
    float dot = 0.f;
    const float rs = rs_n;
    const uint4 xv = xv_n, dv = dv_n, rv = rv_n;
    issue(row + gridDim.x);
    if (active) {
      const uint32_t* xi = reinterpret_cast<const uint32_t*>(&xv);
      const uint32_t* di = reinterpret_cast<const uint32_t*>(&dv);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(xi[j]);
        const float2 df = unpack_bf16x2(di[j]);
        xh[2 * j] = xf.x * rs; xh[2 * j + 1] = xf.y * rs;
        g[2 * j] = df.x * wf[2 * j]; g[2 * j + 1] = df.y * wf[2 * j + 1];
        dwacc[2 * j] += df.x * bf16_round(xh[2 * j]);
        dwacc[2 * j + 1] += df.y * bf16_round(xh[2 * j + 1]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) dot += g[j] * xh[j];
    }
    dot = warp_sum(dot);
    if (lane == 0) red[warp] = dot;
    __syncthreads();
    float tot = (lane < nwarps) ? red[lane] : 0.f;
    tot = warp_sum(tot);
    __syncthreads();
    const float mean = tot / static_cast<float>(h);
    if (active) {
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = rs * (g[j] - xh[j] * mean);
      if (dres != nullptr) {
        const uint32_t* ri = reinterpret_cast<const uint32_t*>(&rv);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = unpack_bf16x2(ri[j]); r[2 * j] += f.x; r[2 * j + 1] += f.y; }
      }
      uint4 o;
      o.x = pack_bf16x2(r[0], r[1]); o.y = pack_bf16x2(r[2], r[3]);
      o.z = pack_bf16x2(r[4], r[5]); o.w = pack_bf16x2(r[6], r[7]);
      st_na_v4(reinterpret_cast<uint4*>(dx + static_cast<size_t>(row) * h) + t, o);
    }
  }
  if (active) {
    float* dst = dw_partial + static_cast<size_t>(blockIdx.x) * h + t * 8;
    reinterpret_cast<float4*>(dst)[0] = make_float4(dwacc[0], dwacc[1], dwacc[2], dwacc[3]);
    reinterpret_cast<float4*>(dst)[1] = make_float4(dwacc[4], dwacc[5], dwacc[6], dwacc[7]);
  }
}

// dw[c] (+)= sum_p partial[p, c]   (fp32 sum; the gradient OutT is bf16, or fp32 for fp32 master gradients).
// Block = 32 column-quads (128 columns, float4 loads) x 8 partial-row lanes; the 8 lanes are folded through smem.
template <typename OutT>
__global__ void __launch_bounds__(256) colsum_reduce_kernel(const float* __restrict__ partial, OutT* __restrict__ dw,
                                                            int nparts, int h, int accumulate) {
  __shared__ float4 red[8][32];
  const int cq = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + cq) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < h) {
    for (int p = pl; p < nparts; p += 8) {
      const float4 v = *reinterpret_cast<const float4*>(partial + static_cast<size_t>(p) * h + col);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  red[pl][cq] = acc;
  __syncthreads();
  if (pl == 0 && col < h) {
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      const float4 v = red[k][cq];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if constexpr (std::is_same<OutT, float>::value) {
      float4* d4 = reinterpret_cast<float4*>(dw + col);
      if (accumulate) {
        const float4 o = *d4;
        acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
      }
      *d4 = acc;
    } else {
      __nv_bfloat162* d2 = reinterpret_cast<__nv_bfloat162*>(dw + col);
      if (accumulate) {
        const float2 o0 = __bfloat1622float2(d2[0]), o1 = __bfloat1622float2(d2[1]);
        acc.x += o0.x; acc.y += o0.y; acc.z += o1.x; acc.w += o1.y;
      }
      d2[0] = __floats2bfloat162_rn(acc.x, acc.y);
      d2[1] = __floats2bfloat162_rn(acc.z, acc.w);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Column sums of a bf16 matrix [rows, n] with leading dimension ld -> fp32 partials (bias gradient of Qwen2 q/k/v).
// ------------------------------------------------------------------------------------------------
__global__ void colsum_partial_kernel(const bf16* __restrict__ a, float* __restrict__ partial, int rows, int n,
                                      int64_t ld) {
  const int c8 = blockIdx.x * blockDim.x + threadIdx.x;  // chunk of 8 columns
  if (c8 * 8 >= n) return;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const uint4 v = ld_nc_v4(reinterpret_cast<const uint4*>(a + static_cast<size_t>(r) * ld) + c8);
    const uint32_t* vi = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = unpack_bf16x2(vi[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
  }
  float* dst = partial + static_cast<size_t>(blockIdx.y) * n + c8 * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) dst[j] = acc[j];
}

// ------------------------------------------------------------------------------------------------
// RoPE (rotate-half convention), in place on the q and k head slices of a packed [T, ld] activation.
//   x' = x * cos + rotate_half(x) * sin   ; backward = same with sin -> -sin.   fp32 math, one rounding.
// Reference: llama/modeling.py:557-577; fusion_ops.py:107-115 (use_neox_rotary_style=False == rotate-half).
// cos/sin tables are fp32 [max_pos, d/2] (first-half frequencies; the second half repeats them).
// Thread = 8 consecutive dims of the first half plus the matching 8 of the second half.
// ------------------------------------------------------------------------------------------------
__global__ void rope_kernel(bf16* __restrict__ x, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                            const int* __restrict__ pos_ids, int tokens, int seq_len, int64_t ld, int nheads,
                            int head_dim, float sign) {
  const int tok = blockIdx.x;
  const int half = head_dim >> 1;
  const int per_head = half >> 3;               // threads per head
  const int idx = threadIdx.x;
  if (idx >= nheads * per_head) return;
  const int head = idx / per_head;
  const int j8 = (idx % per_head) * 8;
  const int pos = pos_ids ? pos_ids[tok] : (tok % seq_len);
  bf16* base = x + static_cast<size_t>(tok) * ld + head * head_dim;
  uint4 a = *reinterpret_cast<const uint4*>(base + j8);
  uint4 b = *reinterpret_cast<const uint4*>(base + half + j8);
  rope_rotate_chunk<true>(a, b, cos_t, sin_t, pos, half, j8, sign);
  *reinterpret_cast<uint4*>(base + j8) = a;
  *reinterpret_cast<uint4*>(base + half + j8) = b;
}

// ------------------------------------------------------------------------------------------------
// SwiGLU.  gu = [gate | up] packed [T, 2I];  m = bf16( silu(g) * u )   (llama/modeling.py:38-45, 648-650)
// backward: dg = dm * u * silu'(g), du = dm * silu(g), written packed as [dg | du].
// ------------------------------------------------------------------------------------------------
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ m, int64_t rows, int inter) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t nchunk_row = inter >> 3;
  const int64_t total = rows * nchunk_row;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nchunk_row, c = i % nchunk_row;
    const uint4* row = reinterpret_cast<const uint4*>(gu + r * 2 * inter);
    const uint4 g = ld_nc_v4(row + c);
    const uint4 u = ld_nc_v4(row + nchunk_row + c);
    const uint32_t* gi = reinterpret_cast<const uint32_t*>(&g);
    const uint32_t* ui = reinterpret_cast<const uint32_t*>(&u);
    uint4 o;
    uint32_t* oi = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oi[j] = swiglu_fwd_pair(gi[j], ui[j]);
    st_na_v4(reinterpret_cast<uint4*>(m + r * inter) + c, o);
  }
}

// Same op fed by the fp32 split-K workspace of the producing GEMM [rows, 2*inter]: gate and up are rounded to bf16 first
// (the Linear output rounding), the workspace is handed back zeroed.
__global__ void swiglu_fwd_f32_kernel(float* __restrict__ acc, bf16* __restrict__ m, int64_t rows, int inter) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t nchunk_row = inter >> 3;
  const int64_t total = rows * nchunk_row;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nchunk_row, c = i % nchunk_row;
    float4* gp = reinterpret_cast<float4*>(acc + r * 2 * inter) + 2 * c;
    float4* up = gp + 2 * nchunk_row;
    const float4 g0 = gp[0], g1 = gp[1], u0 = up[0], u1 = up[1];
    gp[0] = zero; gp[1] = zero; up[0] = zero; up[1] = zero;
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float uv[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
    uint4 o;
    uint32_t* oi = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      oi[j] = swiglu_fwd_pair(pack_bf16x2(gv[2 * j], gv[2 * j + 1]), pack_bf16x2(uv[2 * j], uv[2 * j + 1]));
    st_na_v4(reinterpret_cast<uint4*>(m + r * inter) + c, o);
  }
}

__global__ void swiglu_bwd_kernel(const bf16* __restrict__ gu, const bf16* __restrict__ dm, bf16* __restrict__ dgu,
                                  int64_t rows, int inter) {
  const int64_t nchunk_row = inter >> 3;
  const int64_t total = rows * nchunk_row;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nchunk_row, c = i % nchunk_row;
    const uint4* row = reinterpret_cast<const uint4*>(gu + r * 2 * inter);
    const uint4 g = ld_nc_v4(row + c);
    const uint4 u = ld_nc_v4(row + nchunk_row + c);
    const uint4 d = ld_nc_v4(reinterpret_cast<const uint4*>(dm + r * inter) + c);
    const uint32_t* gi = reinterpret_cast<const uint32_t*>(&g);
    const uint32_t* ui = reinterpret_cast<const uint32_t*>(&u);
    const uint32_t* di = reinterpret_cast<const uint32_t*>(&d);
    uint4 og, ou;
    uint32_t* ogi = reinterpret_cast<uint32_t*>(&og);
    uint32_t* oui = reinterpret_cast<uint32_t*>(&ou);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 df = unpack_bf16x2(di[j]);
      swiglu_bwd_pair(gi[j], ui[j], df.x, df.y, ogi[j], oui[j]);
    }
    uint4* orow = reinterpret_cast<uint4*>(dgu + r * 2 * inter);
    st_na_v4(orow + c, og);
    st_na_v4(orow + nchunk_row + c, ou);
  }
}

// ------------------------------------------------------------------------------------------------
// Embedding gather (llama/modeling.py:1634) and its scatter-add gradient.
// ------------------------------------------------------------------------------------------------
__global__ void embedding_fwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ table,
                                     bf16* __restrict__ out, int tokens, int h, int vocab) {
  const int tok = blockIdx.x;
  int64_t id = ids[tok];
  if (id < 0 || id >= vocab) id = 0;
  const uint4* src = reinterpret_cast<const uint4*>(table + id * h);
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(tok) * h);
  for (int c = threadIdx.x; c < (h >> 3); c += blockDim.x) dst[c] = __ldg(src + c);
}

// dtable[ids[t]] += dout[t]: bf16 pair atomics into a bf16 table, or fp32 vector atomics (4 columns per red) into an fp32 one.
template <typename T>
__global__ void embedding_bwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ dout,
                                     T* __restrict__ dtable, int tokens, int h, int vocab) {
  const int tok = blockIdx.x;
  const int64_t id = ids[tok];
  if (id < 0 || id >= vocab) return;
  if constexpr (std::is_same<T, float>::value) {
    const uint2* src = reinterpret_cast<const uint2*>(dout + static_cast<size_t>(tok) * h);
    float* dst = dtable + id * h;
    for (int c = threadIdx.x; c < (h >> 2); c += blockDim.x) {
      const uint2 v = src[c];
      const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y);
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4 * c), "f"(a.x), "f"(a.y), "f"(b.x), "f"(b.y)
                   : "memory");
    }
  } else {
    const __nv_bfloat162* src = reinterpret_cast<const __nv_bfloat162*>(dout + static_cast<size_t>(tok) * h);
    __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(dtable + id * h);
    for (int c = threadIdx.x; c < (h >> 1); c += blockDim.x) atomicAdd(dst + c, src[c]);
  }
}

}  // namespace ew
}  // namespace b200

using namespace b200;
using namespace b200::ew;

extern "C" int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t rows, int64_t h, float eps,
                                cudaStream_t stream) {
  B200_CHECK_ARG(x && w && y, "rmsnorm_fwd: null pointer");
  B200_CHECK_ARG(rows > 0 && h > 0 && h % 8 == 0 && h <= 8192, "rmsnorm_fwd: need 0 < h <= 8192, h %% 8 == 0 (h=%lld)",
                 (long long)h);
  const int nchunk = static_cast<int>(h / 8);
  const dim3 grid(static_cast<unsigned>((rows + 3) / 4)), block(128);
  const bf16* xp = static_cast<const bf16*>(x);
  const bf16* wp = static_cast<const bf16*>(w);
  bf16* yp = static_cast<bf16*>(y);
  if (nchunk >= 128) {           // h >= 1024: one CTA per row, persistent
    int64_t ctas = static_cast<int64_t>(sm_count()) * 8;
    if (ctas > rows) ctas = rows;
    const dim3 g(static_cast<unsigned>(ctas));
    if (nchunk <= 128 * 4) rmsnorm_fwd_cta_kernel<4><<<g, block, 0, stream>>>(xp, wp, yp, rstd, (int)rows, (int)h, eps);
    else rmsnorm_fwd_cta_kernel<8><<<g, block, 0, stream>>>(xp, wp, yp, rstd, (int)rows, (int)h, eps);
    return check_launch("rmsnorm_fwd");
  }
  if (nchunk <= 32 * 4) rmsnorm_fwd_kernel<4><<<grid, block, 0, stream>>>(xp, wp, yp, rstd, (int)rows, (int)h, eps);
  else if (nchunk <= 32 * 16) rmsnorm_fwd_kernel<16><<<grid, block, 0, stream>>>(xp, wp, yp, rstd, (int)rows, (int)h, eps);
  else rmsnorm_fwd_kernel<32><<<grid, block, 0, stream>>>(xp, wp, yp, rstd, (int)rows, (int)h, eps);
  return check_launch("rmsnorm_fwd");
}

extern "C" int64_t b200_rmsnorm_bwd_workspace_bytes(int64_t rows, int64_t h) {
  int64_t parts = sm_count() * 2;
  if (parts > rows) parts = rows;
  if (parts < 1) parts = 1;
  return parts * h * 4;
}

template <typename OutT>
static int rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx, OutT* dw,
                       int accumulate_dw, void* workspace, int64_t rows, int64_t h, cudaStream_t stream) {
  B200_CHECK_ARG(dy && x && w && rstd && dx && dw && workspace, "rmsnorm_bwd: null pointer");
  B200_CHECK_ARG(rows > 0 && h > 0 && h % 8 == 0 && h <= 8192, "rmsnorm_bwd: need 0 < h <= 8192, h %% 8 == 0 (h=%lld)",
                 (long long)h);
  int parts = sm_count() * 2;
  if (parts > rows) parts = static_cast<int>(rows);
  int threads = static_cast<int>((h / 8 + 31) / 32 * 32);
  rmsnorm_bwd_kernel<<<parts, threads, 0, stream>>>(static_cast<const bf16*>(dy), static_cast<const bf16*>(x),
                                                    static_cast<const bf16*>(w), rstd, static_cast<const bf16*>(dres),
                                                    static_cast<bf16*>(dx), static_cast<float*>(workspace), (int)rows,
                                                    (int)h);
  int rc = check_launch("rmsnorm_bwd");
  if (rc) return rc;
  colsum_reduce_kernel<<<static_cast<unsigned>((h + 127) / 128), 256, 0, stream>>>(
      static_cast<const float*>(workspace), dw, parts, (int)h, accumulate_dw);
  return check_launch("rmsnorm_bwd(dw reduce)");
}

extern "C" int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres,
                                void* dx, void* dw, int accumulate_dw, void* workspace, int64_t rows, int64_t h,
                                cudaStream_t stream) {
  return rmsnorm_bwd(dy, x, w, rstd, dres, dx, static_cast<bf16*>(dw), accumulate_dw, workspace, rows, h, stream);
}

extern "C" int b200_rmsnorm_bwd_f32(const void* dy, const void* x, const void* w, const float* rstd, const void* dres,
                                    void* dx, float* dw, int accumulate_dw, void* workspace, int64_t rows, int64_t h,
                                    cudaStream_t stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dw) & 15) == 0, "rmsnorm_bwd_f32: dw must be 16-byte aligned");
  return rmsnorm_bwd(dy, x, w, rstd, dres, dx, dw, accumulate_dw, workspace, rows, h, stream);
}

extern "C" int64_t b200_colsum_workspace_bytes(int64_t rows, int64_t n) {
  int64_t parts = rows < 64 ? rows : 64;
  return parts * n * 4;
}

template <typename OutT>
static int colsum(const void* a, OutT* out, int accumulate, void* workspace, int64_t rows, int64_t n, int64_t ld,
                  cudaStream_t stream) {
  B200_CHECK_ARG(a && out && workspace, "colsum: null pointer");
  B200_CHECK_ARG(rows > 0 && n > 0 && n % 8 == 0 && ld % 8 == 0, "colsum: n and ld must be multiples of 8");
  const int parts = static_cast<int>(rows < 64 ? rows : 64);
  dim3 grid(static_cast<unsigned>((n / 8 + 127) / 128), parts);
  colsum_partial_kernel<<<grid, 128, 0, stream>>>(static_cast<const bf16*>(a), static_cast<float*>(workspace), (int)rows,
                                                  (int)n, ld);
  int rc = check_launch("colsum(partial)");
  if (rc) return rc;
  colsum_reduce_kernel<<<static_cast<unsigned>((n + 127) / 128), 256, 0, stream>>>(
      static_cast<const float*>(workspace), out, parts, (int)n, accumulate);
  return check_launch("colsum(reduce)");
}

extern "C" int b200_colsum_bf16(const void* a, void* out, int accumulate, void* workspace, int64_t rows, int64_t n,
                                int64_t ld, cudaStream_t stream) {
  return colsum(a, static_cast<bf16*>(out), accumulate, workspace, rows, n, ld, stream);
}

extern "C" int b200_colsum_f32(const void* a, float* out, int accumulate, void* workspace, int64_t rows, int64_t n, int64_t ld,
                               cudaStream_t stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0, "colsum_f32: out must be 16-byte aligned");
  return colsum(a, out, accumulate, workspace, rows, n, ld, stream);
}

extern "C" int b200_rope_inplace(void* x, const float* cos_table, const float* sin_table, const int32_t* position_ids,
                                 int64_t tokens, int64_t seq_len, int64_t ld, int64_t num_heads, int64_t head_dim,
                                 int backward, cudaStream_t stream) {
  B200_CHECK_ARG(x && cos_table && sin_table, "rope: null pointer");
  B200_CHECK_ARG(head_dim % 16 == 0 && head_dim > 0, "rope: head_dim must be a multiple of 16 (got %lld)",
                 (long long)head_dim);
  B200_CHECK_ARG(ld % 8 == 0 && tokens > 0 && num_heads > 0 && seq_len > 0, "rope: bad sizes");
  const int threads_needed = static_cast<int>(num_heads * (head_dim / 16));
  B200_CHECK_ARG(threads_needed <= 1024, "rope: num_heads * head_dim / 16 must be <= 1024");
  const int threads = (threads_needed + 31) / 32 * 32;
  rope_kernel<<<static_cast<unsigned>(tokens), threads, 0, stream>>>(
      static_cast<bf16*>(x), cos_table, sin_table, position_ids, (int)tokens, (int)seq_len, ld, (int)num_heads,
      (int)head_dim, backward ? -1.f : 1.f);
  return check_launch("rope");
}

extern "C" int b200_swiglu_fwd(const void* gate_up, void* out, int64_t rows, int64_t inter, cudaStream_t stream) {
  B200_CHECK_ARG(gate_up && out, "swiglu_fwd: null pointer");
  B200_CHECK_ARG(rows > 0 && inter > 0 && inter % 8 == 0, "swiglu_fwd: intermediate size must be a multiple of 8");
  const int64_t total = rows * (inter / 8);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  launch_pdl(swiglu_fwd_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, static_cast<const bf16*>(gate_up),
             static_cast<bf16*>(out), rows, (int)inter);
  return check_launch("swiglu_fwd");
}

extern "C" int b200_swiglu_fwd_f32(float* gate_up_f32_ws, void* out, int64_t rows, int64_t inter, cudaStream_t stream) {
  B200_CHECK_ARG(gate_up_f32_ws && out, "swiglu_fwd_f32: null pointer");
  B200_CHECK_ARG(rows > 0 && inter > 0 && inter % 8 == 0, "swiglu_fwd_f32: intermediate size must be a multiple of 8");
  const int64_t total = rows * (inter / 8);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  launch_pdl(swiglu_fwd_f32_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, gate_up_f32_ws,
             static_cast<bf16*>(out), rows, (int)inter);
  return check_launch("swiglu_fwd_f32");
}

extern "C" int b200_swiglu_bwd(const void* gate_up, const void* dout, void* dgate_up, int64_t rows, int64_t inter,
                               cudaStream_t stream) {
  B200_CHECK_ARG(gate_up && dout && dgate_up, "swiglu_bwd: null pointer");
  B200_CHECK_ARG(rows > 0 && inter > 0 && inter % 8 == 0, "swiglu_bwd: intermediate size must be a multiple of 8");
  const int64_t total = rows * (inter / 8);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  swiglu_bwd_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      static_cast<const bf16*>(gate_up), static_cast<const bf16*>(dout), static_cast<bf16*>(dgate_up), rows, (int)inter);
  return check_launch("swiglu_bwd");
}

extern "C" int b200_embedding_fwd(const int64_t* ids, const void* table, void* out, int64_t tokens, int64_t h,
                                  int64_t vocab, cudaStream_t stream) {
  B200_CHECK_ARG(ids && table && out, "embedding_fwd: null pointer");
  B200_CHECK_ARG(tokens > 0 && h % 8 == 0, "embedding_fwd: hidden size must be a multiple of 8");
  embedding_fwd_kernel<<<static_cast<unsigned>(tokens), 128, 0, stream>>>(ids, static_cast<const bf16*>(table),
                                                                         static_cast<bf16*>(out), (int)tokens, (int)h,
                                                                         (int)vocab);
  return check_launch("embedding_fwd");
}

template <typename T>
static int embedding_bwd(const int64_t* ids, const void* dout, T* dtable, int64_t tokens, int64_t h, int64_t vocab,
                         cudaStream_t stream) {
  B200_CHECK_ARG(ids && dout && dtable, "embedding_bwd: null pointer");
  B200_CHECK_ARG(tokens > 0 && h % 8 == 0, "embedding_bwd: hidden size must be a multiple of 8");
  embedding_bwd_kernel<<<static_cast<unsigned>(tokens), 128, 0, stream>>>(ids, static_cast<const bf16*>(dout), dtable,
                                                                         (int)tokens, (int)h, (int)vocab);
  return check_launch("embedding_bwd");
}

extern "C" int b200_embedding_bwd(const int64_t* ids, const void* dout, void* dtable, int64_t tokens, int64_t h,
                                  int64_t vocab, cudaStream_t stream) {
  return embedding_bwd(ids, dout, static_cast<bf16*>(dtable), tokens, h, vocab, stream);
}

extern "C" int b200_embedding_bwd_f32(const int64_t* ids, const void* dout, float* dtable, int64_t tokens, int64_t h,
                                      int64_t vocab, cudaStream_t stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dtable) & 15) == 0 && (reinterpret_cast<uintptr_t>(dout) & 7) == 0,
                 "embedding_bwd_f32: dtable must be 16-byte and dout 8-byte aligned");
  return embedding_bwd(ids, dout, dtable, tokens, h, vocab, stream);
}
