// Cross-entropy criterion and the flat-buffer optimizer step (all HBM-bound).
//
//  * CE forward/backward: LlamaPretrainingCriterion (llama/modeling.py:1799-1825): fp32 CE on bf16 logits,
//    reduction none, ignore_index; loss = sum(l_i * [l_i > 0]) / count([l_i > 0]).
//  * Global-norm clip + AdamW with fp32 master weights on ONE flat buffer (trainer.py:1717-1750;
//    ClipGradByGlobalNorm(1.0); multi_precision=True under AMP O2).
#include "../../include/b200nlp.h"
#include "common.cuh"
#include "host_util.h"

namespace b200 {
namespace lo {

__device__ __forceinline__ void online_merge(float& m, float& s, float m2, float s2) {
  const float nm = fmaxf(m, m2);
  if (nm == -INFINITY) { m = nm; s = 0.f; return; }
  s = s * __expf(m - nm) + s2 * __expf(m2 - nm);
  m = nm;
}

// arg-max step with argmax_kernel's order: larger value wins, the lower index wins a tie, NaN never wins.
__device__ __forceinline__ void argmax_take(float& best, int& bi, float v, int i) {
  if (v > best || (v == best && i < bi)) { best = v; bi = i; }
}

// One CTA per token row.  Single pass online logsumexp over the bf16 row.  ARGMAX: the same pass also keeps the row's
// first maximal index (pred[row], equal to argmax_kernel's).  LSE: write lse_out (only the backward needs it).
template <bool ARGMAX, bool LSE>
__global__ void __launch_bounds__(256) ce_fwd_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ labels,
                                                     float* __restrict__ loss_tok, float* __restrict__ lse_out,
                                                     int64_t* __restrict__ pred, int vocab, int64_t ld, int ignore_index) {
  __shared__ float sm[8], ss[8];
  __shared__ float sbest[8];
  __shared__ int sbi[8];
  const int row = blockIdx.x;
  const bf16* lr = logits + static_cast<size_t>(row) * ld;
  const int nchunk = vocab >> 3;
  float m = -INFINITY, s = 0.f;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < nchunk; c += blockDim.x) {
    const uint4 v = ld_nc_v4(reinterpret_cast<const uint4*>(lr) + c);
    const uint32_t* vi = reinterpret_cast<const uint32_t*>(&v);
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 t = unpack_bf16x2(vi[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
    if (ARGMAX) {
#pragma unroll
      for (int j = 0; j < 8; ++j) argmax_take(best, bi, f[j], c * 8 + j);
    }
    float cm = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) cm = fmaxf(cm, f[j]);
    const float nm = fmaxf(m, cm);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(f[j] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  for (int i = (nchunk << 3) + threadIdx.x; i < vocab; i += blockDim.x) {  // tail (vocab % 8)
    const float f = __bfloat162float(lr[i]);
    if (ARGMAX) argmax_take(best, bi, f, i);
    const float nm = fmaxf(m, f);
    s = s * __expf(m - nm) + __expf(f - nm);
    m = nm;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    online_merge(m, s, m2, s2);
    if (ARGMAX) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      argmax_take(best, bi, ob, oi);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sm[warp] = m; ss[warp] = s;
    if (ARGMAX) { sbest[warp] = best; sbi[warp] = bi; }
  }
  __syncthreads();
  if (warp == 0) {
    m = lane < (blockDim.x >> 5) ? sm[lane] : -INFINITY;
    s = lane < (blockDim.x >> 5) ? ss[lane] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      online_merge(m, s, m2, s2);
    }
    if (ARGMAX && lane == 0) {
      for (int w = 1; w < (blockDim.x >> 5); ++w) argmax_take(best, bi, sbest[w], sbi[w]);
      pred[row] = bi;
    }
    if (lane == 0) {
      const float lse = m + logf(s);
      if (LSE) lse_out[row] = lse;
      const int64_t lab = labels[row];
      float l = 0.f;
      if (lab != ignore_index && lab >= 0 && lab < vocab) l = lse - __bfloat162float(lr[lab]);
      loss_tok[row] = l;
    }
  }
}

// out[0] = sum(l_i [l_i>0]) / max(count,1) (or the plain sum if count == 0) ; out[1] = count.  Deterministic.
__global__ void ce_reduce_kernel(const float* __restrict__ loss_tok, float* __restrict__ out, int64_t n) {
  __shared__ float ssum[32], scnt[32];
  float s = 0.f, c = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float l = loss_tok[i];
    if (l > 0.f) { s += l; c += 1.f; }
  }
  s = warp_sum(s);
  c = warp_sum(c);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { ssum[warp] = s; scnt[warp] = c; }
  __syncthreads();
  if (warp == 0) {
    s = lane < (blockDim.x >> 5) ? ssum[lane] : 0.f;
    c = lane < (blockDim.x >> 5) ? scnt[lane] : 0.f;
    s = warp_sum(s);
    c = warp_sum(c);
    if (lane == 0) { out[0] = c > 0.f ? s / c : s; out[1] = c; }
  }
}

// dlogits_i = (softmax_i - onehot_i) * [l_i > 0] * grad_scale / count, written over the logits (bf16).
__global__ void __launch_bounds__(256) ce_bwd_kernel(bf16* __restrict__ logits, const int64_t* __restrict__ labels,
                                                     const float* __restrict__ loss_tok,
                                                     const float* __restrict__ lse, const float* __restrict__ loss_out,
                                                     float grad_scale, const float* __restrict__ grad_scale_ptr,
                                                     int vocab, int64_t ld) {
  const int row = blockIdx.x;
  bf16* lr = logits + static_cast<size_t>(row) * ld;
  const float cnt = loss_out[1];
  if (grad_scale_ptr != nullptr) grad_scale *= grad_scale_ptr[0];
  const float l = loss_tok[row];
  const float scale = (l > 0.f) ? grad_scale / fmaxf(cnt, 1.f) : 0.f;
  const float row_lse = lse[row];
  const int lab = static_cast<int>(labels[row]);
  const int nchunk = vocab >> 3;
  for (int c = threadIdx.x; c < nchunk; c += blockDim.x) {
    uint4 v = *(reinterpret_cast<const uint4*>(lr) + c);
    uint32_t* vi = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = unpack_bf16x2(vi[j]);
      const int col = c * 8 + 2 * j;
      float p0 = __expf(t.x - row_lse), p1 = __expf(t.y - row_lse);
      if (col == lab) p0 -= 1.f;
      if (col + 1 == lab) p1 -= 1.f;
      vi[j] = pack_bf16x2(p0 * scale, p1 * scale);
    }
    *(reinterpret_cast<uint4*>(lr) + c) = v;
  }
  for (int i = (nchunk << 3) + threadIdx.x; i < vocab; i += blockDim.x) {
    float p = __expf(__bfloat162float(lr[i]) - row_lse);
    if (i == lab) p -= 1.f;
    lr[i] = __float2bfloat16_rn(p * scale);
  }
}

// argmax over a bf16 row (first maximal index, like paddle.argmax / torch.argmax on ties -> lowest index).
__global__ void __launch_bounds__(1024) argmax_kernel(const bf16* __restrict__ logits, int64_t* __restrict__ out,
                                                      int vocab, int64_t ld) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const int row = blockIdx.x;
  const bf16* lr = logits + static_cast<size_t>(row) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  const int nchunk = ((reinterpret_cast<uintptr_t>(lr) & 15) == 0) ? (vocab >> 3) : 0;   // 128-bit loads when aligned
  for (int c = threadIdx.x; c < nchunk; c += blockDim.x) {
    const uint4 v = ld_nc_v4(reinterpret_cast<const uint4*>(lr) + c);
    const uint32_t* vi = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(vi[j]);
      const int i0 = c * 8 + 2 * j;
      if (f.x > best || (f.x == best && i0 < bi)) { best = f.x; bi = i0; }
      if (f.y > best || (f.y == best && i0 + 1 < bi)) { best = f.y; bi = i0 + 1; }
    }
  }
  for (int i = (nchunk << 3) + threadIdx.x; i < vocab; i += blockDim.x) {
    const float f = __bfloat162float(lr[i]);
    if (f > best || (f == best && i < bi)) { best = f; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (blockDim.x >> 5); ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
    out[row] = bi;
  }
}

// ------------------------------------------------------------------------------------------------
// Optimizer
// ------------------------------------------------------------------------------------------------
// Gradients are bf16, or fp32 (fp32 master gradients): chunk c of 8 elements as fp32, read once (not cached in L1).
__device__ __forceinline__ void load8_f32(const bf16* g, int64_t c, float (&f)[8]) {
  const uint4 v = ld_nc_v4(reinterpret_cast<const uint4*>(g) + c);
  const uint32_t* vi = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float2 t = unpack_bf16x2(vi[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
}
__device__ __forceinline__ void load8_f32(const float* g, int64_t c, float (&f)[8]) {
  const uint4 a = ld_nc_v4(reinterpret_cast<const uint4*>(g) + 2 * c), b = ld_nc_v4(reinterpret_cast<const uint4*>(g) + 2 * c + 1);
  const uint32_t u[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = __uint_as_float(u[j]);
}
__device__ __forceinline__ float to_f32(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float to_f32(float x) { return x; }

template <typename G>
__global__ void __launch_bounds__(256) sqnorm_partial_kernel(const G* __restrict__ g, float* __restrict__ partial, int64_t n) {
  __shared__ float red[8];
  float acc = 0.f;
  const int64_t nchunk = n >> 3;
  for (int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; c < nchunk;
       c += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float f[8];
    load8_f32(g, c, f);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc += f[2 * j] * f[2 * j] + f[2 * j + 1] * f[2 * j + 1];
  }
  if (blockIdx.x == 0)
    for (int64_t i = (nchunk << 3) + threadIdx.x; i < n; i += blockDim.x) {
      const float t = to_f32(g[i]);
      acc += t * t;
    }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) partial[blockIdx.x] = t;
  }
}
// out[0] = sum(partials) * scale^2  (squared norm of scale * g)
__global__ void sqnorm_final_kernel(const float* __restrict__ partial, float* __restrict__ out, int n, float scale) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partial[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) out[0] = t * scale * scale;
  }
}

struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay;
  float bias_corr1, bias_corr2;   // 1 - beta^t
  float grad_scale;               // 1 / (world_size) etc., applied before clipping
  float max_grad_norm;            // <= 0: no clipping
  int64_t n, decay_end;           // elements [0, decay_end) get weight decay
};

// Paddle adamw kernel semantics: p *= (1 - lr*wd); m,v update; p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps).
template <typename G>
__global__ void __launch_bounds__(256) adamw_kernel(bf16* __restrict__ p16, const G* __restrict__ grads,
                                                    float* __restrict__ master, float* __restrict__ m,
                                                    float* __restrict__ v, const float* __restrict__ sqnorm,
                                                    AdamArgs a) {
  float gs = a.grad_scale;
  if (a.max_grad_norm > 0.f && sqnorm != nullptr) {
    const float norm = sqrtf(sqnorm[0]);
    gs *= a.max_grad_norm / fmaxf(norm, a.max_grad_norm);   // ClipGradByGlobalNorm
  }
  const float step = a.lr / a.bias_corr1;
  const float inv_sqrt_bc2 = rsqrtf(a.bias_corr2);
  const int64_t nchunk = a.n >> 3;
  for (int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; c < nchunk;
       c += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float g[8];
    load8_f32(grads, c, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= gs;
    float4* mp = reinterpret_cast<float4*>(m) + 2 * c;
    float4* vp = reinterpret_cast<float4*>(v) + 2 * c;
    float4* pp = reinterpret_cast<float4*>(master) + 2 * c;
    float4 m0 = mp[0], m1 = mp[1], v0 = vp[0], v1 = vp[1], p0 = pp[0], p1 = pp[1];
    float mm[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
    float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    float pm[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
    const float decay = (c * 8 < a.decay_end) ? (1.f - a.lr * a.weight_decay) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mm[j] = a.beta1 * mm[j] + (1.f - a.beta1) * g[j];
      vv[j] = a.beta2 * vv[j] + (1.f - a.beta2) * g[j] * g[j];
      const float denom = sqrtf(vv[j]) * inv_sqrt_bc2 + a.eps;
      pm[j] = pm[j] * decay - step * (mm[j] / denom);
    }
    mp[0] = make_float4(mm[0], mm[1], mm[2], mm[3]); mp[1] = make_float4(mm[4], mm[5], mm[6], mm[7]);
    vp[0] = make_float4(vv[0], vv[1], vv[2], vv[3]); vp[1] = make_float4(vv[4], vv[5], vv[6], vv[7]);
    pp[0] = make_float4(pm[0], pm[1], pm[2], pm[3]); pp[1] = make_float4(pm[4], pm[5], pm[6], pm[7]);
    uint4 o;
    o.x = pack_bf16x2(pm[0], pm[1]); o.y = pack_bf16x2(pm[2], pm[3]);
    o.z = pack_bf16x2(pm[4], pm[5]); o.w = pack_bf16x2(pm[6], pm[7]);
    *(reinterpret_cast<uint4*>(p16) + c) = o;
  }
}

// master[i] = float(p16[i])  (initialise fp32 master weights from the bf16 parameters)
__global__ void bf16_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = __bfloat162float(src[i]);
}

}  // namespace lo
}  // namespace b200

using namespace b200;
using namespace b200::lo;

extern "C" int b200_ce_fwd(const void* logits, const int64_t* labels, float* loss_tok, float* lse, float* loss_out,
                           int64_t tokens, int64_t vocab, int64_t ld, int64_t ignore_index, cudaStream_t stream) {
  B200_CHECK_ARG(logits && labels && loss_tok && lse && loss_out, "ce_fwd: null pointer");
  B200_CHECK_ARG(tokens > 0 && vocab > 0 && ld % 8 == 0, "ce_fwd: ld must be a multiple of 8");
  ce_fwd_kernel<false, true><<<static_cast<unsigned>(tokens), 256, 0, stream>>>(
      static_cast<const bf16*>(logits), labels, loss_tok, lse, nullptr, (int)vocab, ld, (int)ignore_index);
  int rc = check_launch("ce_fwd");
  if (rc) return rc;
  ce_reduce_kernel<<<1, 1024, 0, stream>>>(loss_tok, loss_out, tokens);
  return check_launch("ce_fwd(reduce)");
}

extern "C" int b200_ce_rows_fwd(const void* logits, const int64_t* labels, float* loss_tok, int64_t* pred, int64_t row0,
                                int64_t rows, int64_t vocab, int64_t ld, int64_t ignore_index, cudaStream_t stream) {
  B200_CHECK_ARG(logits && labels && loss_tok, "ce_rows_fwd: null pointer");
  B200_CHECK_ARG(row0 >= 0 && rows > 0 && vocab > 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0,
                 "ce_rows_fwd: ld must be a multiple of 8 and logits 16-byte aligned");
  const bf16* lg = static_cast<const bf16*>(logits);
  if (pred != nullptr)
    ce_fwd_kernel<true, false><<<static_cast<unsigned>(rows), 256, 0, stream>>>(
        lg, labels + row0, loss_tok + row0, nullptr, pred + row0, (int)vocab, ld, (int)ignore_index);
  else
    ce_fwd_kernel<false, false><<<static_cast<unsigned>(rows), 256, 0, stream>>>(
        lg, labels + row0, loss_tok + row0, nullptr, nullptr, (int)vocab, ld, (int)ignore_index);
  return check_launch("ce_rows_fwd");
}

extern "C" int b200_ce_reduce(const float* loss_tok, float* loss_out, int64_t tokens, cudaStream_t stream) {
  B200_CHECK_ARG(loss_tok && loss_out && tokens > 0, "ce_reduce: bad arguments");
  ce_reduce_kernel<<<1, 1024, 0, stream>>>(loss_tok, loss_out, tokens);
  return check_launch("ce_reduce");
}

extern "C" int b200_ce_bwd(void* logits_inout, const int64_t* labels, const float* loss_tok, const float* lse,
                           const float* loss_out, float grad_scale, const float* grad_scale_dev, int64_t tokens,
                           int64_t vocab, int64_t ld, cudaStream_t stream) {
  B200_CHECK_ARG(logits_inout && labels && loss_tok && lse && loss_out, "ce_bwd: null pointer");
  B200_CHECK_ARG(tokens > 0 && vocab > 0 && ld % 8 == 0, "ce_bwd: ld must be a multiple of 8");
  ce_bwd_kernel<<<static_cast<unsigned>(tokens), 256, 0, stream>>>(static_cast<bf16*>(logits_inout), labels, loss_tok, lse,
                                                                  loss_out, grad_scale, grad_scale_dev, (int)vocab, ld);
  return check_launch("ce_bwd");
}

extern "C" int b200_argmax_bf16(const void* logits, int64_t* out, int64_t rows, int64_t vocab, int64_t ld,
                                cudaStream_t stream) {
  B200_CHECK_ARG(logits && out && rows > 0 && vocab > 0, "argmax: bad arguments");
  argmax_kernel<<<static_cast<unsigned>(rows), 1024, 0, stream>>>(static_cast<const bf16*>(logits), out, (int)vocab, ld);
  return check_launch("argmax");
}

extern "C" int64_t b200_grad_sqnorm_workspace_bytes(void) { return static_cast<int64_t>(sm_count()) * 8 * 4; }

template <typename G>
static int grad_sqnorm(const G* grads, float* out, void* workspace, int64_t n, float scale, cudaStream_t stream) {
  B200_CHECK_ARG(grads && out && workspace && n > 0, "grad_sqnorm: bad arguments");
  const int blocks = sm_count() * 8;
  sqnorm_partial_kernel<<<blocks, 256, 0, stream>>>(grads, static_cast<float*>(workspace), n);
  int rc = check_launch("grad_sqnorm(partial)");
  if (rc) return rc;
  sqnorm_final_kernel<<<1, 1024, 0, stream>>>(static_cast<const float*>(workspace), out, blocks, scale);
  return check_launch("grad_sqnorm(final)");
}

extern "C" int b200_grad_sqnorm(const void* grads, float* out, void* workspace, int64_t n, float scale,
                                cudaStream_t stream) {
  return grad_sqnorm(static_cast<const bf16*>(grads), out, workspace, n, scale, stream);
}

extern "C" int b200_grad_sqnorm_f32(const float* grads, float* out, void* workspace, int64_t n, float scale,
                                    cudaStream_t stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "grad_sqnorm_f32: grads must be 16-byte aligned");
  return grad_sqnorm(grads, out, workspace, n, scale, stream);
}

template <typename G>
static int adamw_step(void* params_bf16, const G* grads, float* master, float* exp_avg, float* exp_avg_sq,
                      const float* grad_sqnorm, int64_t n, int64_t decay_end, float lr, float beta1, float beta2, float eps,
                      float weight_decay, int64_t step, float grad_scale, float max_grad_norm, cudaStream_t stream) {
  B200_CHECK_ARG(params_bf16 && grads && master && exp_avg && exp_avg_sq, "adamw: null pointer");
  B200_CHECK_ARG(n > 0 && n % 8 == 0 && decay_end % 8 == 0 && decay_end <= n && step >= 1,
                 "adamw: n and decay_end must be multiples of 8, step >= 1");
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  a.bias_corr1 = 1.f - powf(beta1, static_cast<float>(step));
  a.bias_corr2 = 1.f - powf(beta2, static_cast<float>(step));
  a.grad_scale = grad_scale; a.max_grad_norm = max_grad_norm; a.n = n; a.decay_end = decay_end;
  const int blocks = sm_count() * 8;
  adamw_kernel<<<blocks, 256, 0, stream>>>(static_cast<bf16*>(params_bf16), grads, master, exp_avg, exp_avg_sq, grad_sqnorm, a);
  return check_launch("adamw");
}

extern "C" int b200_adamw_step(void* params_bf16, const void* grads_bf16, float* master, float* exp_avg, float* exp_avg_sq,
                               const float* grad_sqnorm, int64_t n, int64_t decay_end, float lr, float beta1, float beta2,
                               float eps, float weight_decay, int64_t step, float grad_scale, float max_grad_norm,
                               cudaStream_t stream) {
  return adamw_step(params_bf16, static_cast<const bf16*>(grads_bf16), master, exp_avg, exp_avg_sq, grad_sqnorm, n, decay_end,
                    lr, beta1, beta2, eps, weight_decay, step, grad_scale, max_grad_norm, stream);
}

extern "C" int b200_adamw_step_f32(void* params_bf16, const float* grads, float* master, float* exp_avg, float* exp_avg_sq,
                                   const float* grad_sqnorm, int64_t n, int64_t decay_end, float lr, float beta1, float beta2,
                                   float eps, float weight_decay, int64_t step, float grad_scale, float max_grad_norm,
                                   cudaStream_t stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "adamw_f32: grads must be 16-byte aligned");
  return adamw_step(params_bf16, grads, master, exp_avg, exp_avg_sq, grad_sqnorm, n, decay_end, lr, beta1, beta2, eps,
                    weight_decay, step, grad_scale, max_grad_norm, stream);
}

extern "C" int b200_bf16_to_f32(const void* src, float* dst, int64_t n, cudaStream_t stream) {
  B200_CHECK_ARG(src && dst && n > 0, "bf16_to_f32: bad arguments");
  bf16_to_f32_kernel<<<sm_count() * 8, 256, 0, stream>>>(static_cast<const bf16*>(src), dst, n);
  return check_launch("bf16_to_f32");
}
