// Memory-bound helpers of the matcher layer:
//   * rope_split  : de-interleave the Wqkv output (feature = h*3*hd + d*3 + {q,k,v}, head dim hd = 64 or 32) and
//                   apply the cached rotary encoding to q and k   (lightglue.py:42-49, 156-160)
//   * ln_gelu     : LayerNorm(2D) + exact-erf GELU of the FFN (lightglue.py:143-148)
//   * adam_flat   : Adam on the flat parameter buffer (train.py:358-361, 513)
// All use 128-bit loads/stores; row reductions are warp shuffles.
#include <math.h>

#include <initializer_list>
#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

template <typename T> struct Vec8;  // 8 consecutive elements
template <> struct Vec8<float> {
  float v[8];
  __device__ static Vec8 load(const float* p) {
    Vec8 r;
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
  }
  __device__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
};
template <> struct Vec8<__nv_bfloat16> {
  float v[8];
  __device__ static Vec8 load(const __nv_bfloat16* p) {
    Vec8 r;
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      r.v[2 * i] = __uint_as_float(w[i] << 16);
      r.v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
    return r;
  }
  __device__ void store(__nv_bfloat16* p) const {
    uint4 u;
    u.x = pack_bf16(v[0], v[1]); u.y = pack_bf16(v[2], v[3]); u.z = pack_bf16(v[4], v[5]); u.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};

// ---------------------------------------------------------------------------------------------
// rope_split: thread <-> (token, group of 4 rotary pairs = 8 channels), loops over heads.  HD = head dim (64 or 32).
// qkv row layout per head: [q0 k0 v0 q1 k1 v1 ... q(HD-1) k(HD-1) v(HD-1)]; the 8 channels of a group are 24
// consecutive elements.  Outputs are token-major [T, H*HD]; theta is [T, HD/2].
// ---------------------------------------------------------------------------------------------
template <typename T, int HD>
__global__ void __launch_bounds__(256) rope_split_fwd_kernel(const T* __restrict__ qkv, const float* __restrict__ theta,
                                                            T* __restrict__ q, T* __restrict__ k, T* __restrict__ v,
                                                            int64_t ntok, int H) {
  static_assert(HD == 32 || HD == 64, "head_dim 32 or 64");
  constexpr int kGroups = HD / 8, kShift = HD == 64 ? 3 : 2;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t tok = gid >> kShift;
  const int grp = (int)(gid & (kGroups - 1));
  if (tok >= ntok) return;
  float c[4], s[4];
  {
    const float4 th = *reinterpret_cast<const float4*>(theta + tok * (HD / 2) + grp * 4);
    sincosf(th.x, &s[0], &c[0]); sincosf(th.y, &s[1], &c[1]); sincosf(th.z, &s[2], &c[2]); sincosf(th.w, &s[3], &c[3]);
  }
  for (int h = 0; h < H; ++h) {
    const T* src = qkv + tok * (int64_t)(H * 3 * HD) + h * 3 * HD + grp * 24;
    Vec8<T> a = Vec8<T>::load(src), b = Vec8<T>::load(src + 8), d = Vec8<T>::load(src + 16);
    float f[24];
#pragma unroll
    for (int i = 0; i < 8; ++i) { f[i] = a.v[i]; f[8 + i] = b.v[i]; f[16 + i] = d.v[i]; }
    Vec8<T> oq, ok, ov;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float q0 = f[6 * p + 0], k0 = f[6 * p + 1], v0 = f[6 * p + 2];
      const float q1 = f[6 * p + 3], k1 = f[6 * p + 4], v1 = f[6 * p + 5];
      oq.v[2 * p] = q0 * c[p] - q1 * s[p];
      oq.v[2 * p + 1] = q1 * c[p] + q0 * s[p];
      ok.v[2 * p] = k0 * c[p] - k1 * s[p];
      ok.v[2 * p + 1] = k1 * c[p] + k0 * s[p];
      ov.v[2 * p] = v0;
      ov.v[2 * p + 1] = v1;
    }
    const int64_t o = tok * (int64_t)(H * HD) + h * HD + grp * 8;
    oq.store(q + o);
    ok.store(k + o);
    ov.store(v + o);
  }
}

// backward: dq,dk are gradients w.r.t. the ROTATED q,k; q,k are the rotated values saved by forward.
//   d(unrotated) = R(-theta) d(rotated);  dtheta_p += sum_heads ( dq'[2p+1] q'[2p] - dq'[2p] q'[2p+1] ) + same for k
template <typename T, int HD>
__global__ void __launch_bounds__(256) rope_split_bwd_kernel(const T* __restrict__ dq, const T* __restrict__ dk,
                                                            const T* __restrict__ dv, const T* __restrict__ q,
                                                            const T* __restrict__ k, const float* __restrict__ theta,
                                                            T* __restrict__ dqkv, float* __restrict__ dtheta,
                                                            int64_t ntok, int H) {
  static_assert(HD == 32 || HD == 64, "head_dim 32 or 64");
  constexpr int kGroups = HD / 8, kShift = HD == 64 ? 3 : 2;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t tok = gid >> kShift;
  const int grp = (int)(gid & (kGroups - 1));
  if (tok >= ntok) return;
  float c[4], s[4], dth[4] = {0.f, 0.f, 0.f, 0.f};
  {
    const float4 th = *reinterpret_cast<const float4*>(theta + tok * (HD / 2) + grp * 4);
    sincosf(th.x, &s[0], &c[0]); sincosf(th.y, &s[1], &c[1]); sincosf(th.z, &s[2], &c[2]); sincosf(th.w, &s[3], &c[3]);
  }
  for (int h = 0; h < H; ++h) {
    const int64_t o = tok * (int64_t)(H * HD) + h * HD + grp * 8;
    Vec8<T> gq = Vec8<T>::load(dq + o), gk = Vec8<T>::load(dk + o), gv = Vec8<T>::load(dv + o);
    Vec8<T> rq = Vec8<T>::load(q + o), rk = Vec8<T>::load(k + o);
    float f[24];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float a0 = gq.v[2 * p], a1 = gq.v[2 * p + 1], b0 = gk.v[2 * p], b1 = gk.v[2 * p + 1];
      dth[p] += (a1 * rq.v[2 * p] - a0 * rq.v[2 * p + 1]) + (b1 * rk.v[2 * p] - b0 * rk.v[2 * p + 1]);
      f[6 * p + 0] = a0 * c[p] + a1 * s[p];
      f[6 * p + 3] = a1 * c[p] - a0 * s[p];
      f[6 * p + 1] = b0 * c[p] + b1 * s[p];
      f[6 * p + 4] = b1 * c[p] - b0 * s[p];
      f[6 * p + 2] = gv.v[2 * p];
      f[6 * p + 5] = gv.v[2 * p + 1];
    }
    Vec8<T> a, b, d;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a.v[i] = f[i]; b.v[i] = f[8 + i]; d.v[i] = f[16 + i]; }
    T* dst = dqkv + tok * (int64_t)(H * 3 * HD) + h * 3 * HD + grp * 24;
    a.store(dst);
    b.store(dst + 8);
    d.store(dst + 16);
  }
  if (!dtheta) return;  // the angles need no gradient (frozen position encoder)
  float4* pt = reinterpret_cast<float4*>(dtheta + tok * (HD / 2) + grp * 4);
  float4 acc = *pt;  // accumulated across layers; this thread is the only writer of these 4 floats
  acc.x += dth[0]; acc.y += dth[1]; acc.z += dth[2]; acc.w += dth[3];
  *pt = acc;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm + GELU: one warp per token, W = 128 * VPL channels (VPL float4/bf16x4 groups per lane)
// ---------------------------------------------------------------------------------------------
// Phi(z) = 0.5 (1 + erf(z / sqrt 2)) and e = exp(-z^2 / 2) from ONE exponential and ONE reciprocal:
// erfc(|x|) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-x^2), t = 1 / (1 + p |x|)   (Abramowitz-Stegun 7.1.26,
// |error| <= 1.5e-7 absolute, i.e. fp32 round-off level; libdevice erff + expf cost ~3x the instructions).
__device__ __forceinline__ void gauss_cdf_pdf(float z, float& cdf, float& ez) {
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752f, fabsf(z), 1.f)));
  ez = fast_exp2(-0.72134752044448170f * z * z);
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float half_erfc = 0.5f * p * t * ez;  // Phi(-|z|)
  cdf = z >= 0.f ? 1.f - half_erfc : half_erfc;
}
__device__ __forceinline__ float gelu_f(float x) {
  float cdf, ez;
  gauss_cdf_pdf(x, cdf, ez);
  return x * cdf;
}
__device__ __forceinline__ float gelu_grad(float x) {
  float cdf, ez;
  gauss_cdf_pdf(x, cdf, ez);
  return fmaf(x * 0.3989422804014327f, ez, cdf);
}

// 8 consecutive elements as loaded (conversion deferred so a prefetched token costs 4 registers per chunk in bf16)
template <typename T> struct Raw8;
template <> struct Raw8<float> {
  float4 a, b;
  __device__ static Raw8 load(const float* p) {
    Raw8 r;
    r.a = *reinterpret_cast<const float4*>(p);
    r.b = *reinterpret_cast<const float4*>(p + 4);
    return r;
  }
  __device__ void unpack(float* o) const {
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  }
};
template <> struct Raw8<__nv_bfloat16> {
  uint4 u;
  __device__ static Raw8 load(const __nv_bfloat16* p) {
    Raw8 r;
    r.u = *reinterpret_cast<const uint4*>(p);
    return r;
  }
  __device__ void unpack(float* o) const {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      o[2 * i] = __uint_as_float(w[i] << 16);
      o[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
};
template <typename T> __device__ __forceinline__ void store8(T* p, const float* o);
template <> __device__ __forceinline__ void store8<float>(float* p, const float* o) {
  *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(o[4], o[5], o[6], o[7]);
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float* o) {
  uint4 u;
  u.x = pack_bf16(o[0], o[1]); u.y = pack_bf16(o[2], o[3]); u.z = pack_bf16(o[4], o[5]); u.w = pack_bf16(o[6], o[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// forward: one warp per token, 16-byte accesses (lane owns 8 consecutive features of every 256-wide chunk), the
// loads of TPW tokens in flight together; two-pass mean / variance on the registers.
template <typename T, int NCH, int TPW>
__global__ void __launch_bounds__(256) ln_gelu_fwd_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, T* __restrict__ y,
                                                         float* __restrict__ mean, float* __restrict__ rstd,
                                                         int64_t ntok, float eps) {
  constexpr int W = 256 * NCH;
  const int lane = threadIdx.x & 31;
  const int64_t tok0 = ((int64_t)blockIdx.x * 8 + (threadIdx.x >> 5)) * TPW;
  if (tok0 >= ntok) return;
  Raw8<T> raw[TPW][NCH];
#pragma unroll
  for (int t = 0; t < TPW; ++t)
    if (tok0 + t < ntok) {
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) raw[t][ch] = Raw8<T>::load(x + (tok0 + t) * W + ch * 256 + lane * 8);
    }
#pragma unroll
  for (int t = 0; t < TPW; ++t) {
    const int64_t tok = tok0 + t;
    if (tok >= ntok) break;
    float v[NCH][8];
    float sum = 0.f;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      raw[t][ch].unpack(v[ch]);
#pragma unroll
      for (int e = 0; e < 8; e += 2) sum += v[ch][e] + v[ch][e + 1];
    }
    const float mu = warp_sum(sum) * (1.f / W);
    float sq = 0.f;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[ch][e] - mu;
        sq = fmaf(d, d, sq);
      }
    const float rs = rsqrtf(warp_sum(sq) * (1.f / W) + eps);
    const float nmr = -mu * rs;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      float g[8], bb[8], o[8];
      Raw8<float>::load(gamma + ch * 256 + lane * 8).unpack(g);
      Raw8<float>::load(beta + ch * 256 + lane * 8).unpack(bb);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = gelu_f(fmaf(fmaf(v[ch][e], rs, nmr), g[e], bb[e]));
      store8<T>(y + tok * W + ch * 256 + lane * 8, o);
    }
    if (lane == 0) {
      mean[tok] = mu;
      rstd[tok] = rs;
    }
  }
}

// backward: a token is handled by NCH cooperating warps (one 256-column chunk each, so a lane carries only
// 3 x 8 column accumulators and nothing spills); the 8/NCH token slots of a CTA walk tokens
// blockIdx.x*(8/NCH) + slot, + gridDim.x*(8/NCH), ... with the next token's x / dy already in flight.  The two
// row sums of the LayerNorm backward are exchanged between the NCH warps through smem and a named barrier.
// Per-lane partial dgamma / dbeta / sum(dx) are reduced over the token slots and written as one partial row per CTA.
template <typename T, int NCH>
__global__ void __launch_bounds__(256, 2)
    ln_gelu_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ gamma,
                       const float* __restrict__ beta, const float* __restrict__ mean,
                       const float* __restrict__ rstd, T* __restrict__ dx, float* __restrict__ dgamma_part,
                       float* __restrict__ dbeta_part, float* __restrict__ dxsum_part, int64_t ntok) {
  constexpr int W = 256 * NCH;
  constexpr int SLOTS = 8 / NCH;
  __shared__ __align__(16) float s_red[SLOTS][W];
  __shared__ float2 s_rows[2][SLOTS][NCH];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = warp % NCH, slot = warp / NCH;
  const int col = sub * 256 + lane * 8;
  float g[8], bb[8], dg[8], db[8], dxs[8];
  Raw8<float>::load(gamma + col).unpack(g);
  Raw8<float>::load(beta + col).unpack(bb);
#pragma unroll
  for (int e = 0; e < 8; ++e) dg[e] = db[e] = dxs[e] = 0.f;
  const int64_t stride = (int64_t)gridDim.x * SLOTS;
  int64_t tok = (int64_t)blockIdx.x * SLOTS + slot;
  Raw8<T> rx, rg;
  float mu = 0.f, rs = 0.f;
  if (tok < ntok) {
    rx = Raw8<T>::load(x + tok * W + col);
    rg = Raw8<T>::load(dy + tok * W + col);
    mu = mean[tok];
    rs = rstd[tok];
  }
  int par = 0;
  while (tok < ntok) {
    float xh[8], dz[8];
    rx.unpack(xh);
    rg.unpack(dz);
    const float crs = rs, nmr = -mu * rs;
    const int64_t nxt = tok + stride;
    if (nxt < ntok) {
      rx = Raw8<T>::load(x + nxt * W + col);
      rg = Raw8<T>::load(dy + nxt * W + col);
      mu = mean[nxt];
      rs = rstd[nxt];
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float h = fmaf(xh[e], crs, nmr);                       // normalised input
      const float dzz = dz[e] * gelu_grad(fmaf(h, g[e], bb[e]));   // dL/d(LN output)
      dg[e] = fmaf(dzz, h, dg[e]);
      db[e] += dzz;
      const float d = dzz * g[e];                                  // dL/dxhat
      s1 += d;
      s2 = fmaf(d, h, s2);
      xh[e] = h;
      dz[e] = d;
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (NCH > 1) {
      if (lane == 0) s_rows[par][slot][sub] = make_float2(s1, s2);
      asm volatile("bar.sync %0, %1;" ::"r"(1 + slot), "r"(32 * NCH) : "memory");
      s1 = s2 = 0.f;
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const float2 v = s_rows[par][slot][k];
        s1 += v.x;
        s2 += v.y;
      }
      par ^= 1;  // the other buffer is free again once every warp of the slot passed this token's barrier
    }
    const float c0 = -crs * s1 * (1.f / W), c2 = -crs * s2 * (1.f / W);
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      o[e] = fmaf(xh[e], c2, fmaf(dz[e], crs, c0));  // rs (d - mean(d) - xhat mean(d xhat))
      dxs[e] += o[e];
    }
    store8<T>(dx + tok * W + col, o);
    tok = nxt;
  }
  // reduce dgamma, dbeta and the column sums of dx over the token slots
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
#pragma unroll
    for (int e = 0; e < 8; ++e) s_red[slot][col + e] = pass == 0 ? dg[e] : (pass == 1 ? db[e] : dxs[e]);
    __syncthreads();
    float* dst = pass == 0 ? dgamma_part : (pass == 1 ? dbeta_part : dxsum_part);
    for (int c = threadIdx.x; c < W; c += 256) {
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < SLOTS; ++w) acc += s_red[w][c];
      dst[(int64_t)blockIdx.x * W + c] = acc;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// Optimiser updates on the flat buffers: one kernel body (flat_update_kernel) handles the controls every rule shares
// -- the skip flag, the device lr / step / loss-scale divisor, grad_scale (1/world for the summed all-reduce) and the
// per-element lr_scaling factor -- and hands each element to an update rule (AdamRule, AdamWRule, SgdRule,
// RmspropRule), which restates torch.optim.<X>'s single-tensor arithmetic in its order of operations (no amsgrad, no
// maximize).  Each thread owns 4 consecutive elements (128-bit loads); the grid depends on n only.
// fp32 words read + written per element (one more read with lr_scale): Adam / AdamW 7 (p, g, exp_avg, exp_avg_sq in;
// p, exp_avg, exp_avg_sq out); SGD 3, with momentum 5; RMSprop 5, + 2 with momentum, + 2 centered (9 for both).
// ---------------------------------------------------------------------------------------------
struct AdamDev {  // optional device-resident controls (all may be null); see lgb200_adam_flat in lgb200.h
  const int* step;          // 1-based step count (CUDA-graph replay)
  const float* lr;          // learning rate (so a scheduler can change it between graph replays)
  const float* loss_scale;  // GradScaler scale: gradients are multiplied by 1 / *loss_scale (GradScaler.unscale_)
  const float* found_inf;   // != 0: skip the update entirely (GradScaler.step / the NaN guard of train.py:477-480)
};

// torch.optim.Adam, L2 weight decay added to the gradient.  bc1 / bc2_sqrt: host bias corrections, recomputed here
// when the step count lives on the device.
struct AdamRule {
  float beta1, beta2, eps, wd, bc1, bc2_sqrt;
  __device__ void prepare(const int* step) {
    if (step) {
      const float t = (float)(*step);
      bc1 = 1.f - powf(beta1, t);
      bc2_sqrt = sqrtf(1.f - powf(beta2, t));
    }
  }
  __device__ void operator()(float& p, float g, float grad_scale, float l, float& m, float& v, float&) const {
    float gr = g * grad_scale + wd * p;
    m = beta1 * m + (1.f - beta1) * gr;
    v = beta2 * v + (1.f - beta2) * gr * gr;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p -= (l / bc1) * (m / denom);
  }
};

// torch.optim.AdamW: decoupled decay p *= 1 - lr_group * wd before the Adam step (lr_group includes lr_scaling).
struct AdamWRule : AdamRule {
  __device__ void operator()(float& p, float g, float grad_scale, float l, float& m, float& v, float&) const {
    p *= 1.f - l * wd;
    const float gr = g * grad_scale;
    m = beta1 * m + (1.f - beta1) * gr;
    v = beta2 * v + (1.f - beta2) * gr * gr;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p -= (l / bc1) * (m / denom);
  }
};

// torch.optim.SGD.  On the first step (step count 1) the momentum buffer becomes the gradient itself, undampened.
struct SgdRule {
  float momentum, dampening, wd;
  int nesterov, step;
  __device__ void prepare(const int* step_dev) {
    if (step_dev) step = *step_dev;
  }
  __device__ void operator()(float& p, float g, float grad_scale, float l, float& buf, float&, float&) const {
    float gr = g * grad_scale;
    if (wd != 0.f) gr = gr + wd * p;
    if (momentum != 0.f) {
      buf = step <= 1 ? gr : momentum * buf + (1.f - dampening) * gr;
      gr = nesterov ? gr + momentum * buf : buf;
    }
    p = p + -l * gr;
  }
};

// torch.optim.RMSprop (step count unused by the arithmetic).
struct RmspropRule {
  float alpha, eps, wd, momentum;
  int centered;
  __device__ void prepare(const int*) {}
  __device__ void operator()(float& p, float g, float grad_scale, float l, float& sq, float& buf, float& gavg) const {
    float gr = g * grad_scale;
    if (wd != 0.f) gr = gr + wd * p;
    sq = sq * alpha + (1.f - alpha) * gr * gr;
    float avg;
    if (centered) {
      gavg = gavg + (1.f - alpha) * (gr - gavg);  // lerp with weight 1 - alpha < 0.5
      avg = sqrtf(sq - gavg * gavg);
    } else {
      avg = sqrtf(sq);
    }
    avg = avg + eps;
    if (momentum > 0.f) {
      buf = buf * momentum + gr / avg;
      p = p + -l * buf;
    } else {
      p = p + -l * (gr / avg);
    }
  }
};

// s0..s2: the rule's state buffers in its argument order; a null one is neither read nor written.
template <class Rule>
__global__ void __launch_bounds__(256) flat_update_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                         float* __restrict__ s0, float* __restrict__ s1,
                                                         float* __restrict__ s2, int64_t n,
                                                         const float* __restrict__ lr_scale_or_null, float lr,
                                                         float grad_scale, Rule rule, AdamDev dev) {
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i0 >= n) return;
  if (dev.found_inf && *dev.found_inf != 0.f) return;  // whole grid takes the same branch
  rule.prepare(dev.step);
  if (dev.lr) lr = *dev.lr;
  if (dev.loss_scale) grad_scale *= 1.f / *dev.loss_scale;
  float* s[3] = {s0, s1, s2};
  if (i0 + 4 <= n) {
    float4 pp = *reinterpret_cast<float4*>(p + i0), gg = *reinterpret_cast<const float4*>(g + i0);
    float P[4] = {pp.x, pp.y, pp.z, pp.w}, G[4] = {gg.x, gg.y, gg.z, gg.w}, S[3][4] = {};
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (s[k]) {
        const float4 x = *reinterpret_cast<float4*>(s[k] + i0);
        S[k][0] = x.x, S[k][1] = x.y, S[k][2] = x.z, S[k][3] = x.w;
      }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float l = lr_scale_or_null ? lr * lr_scale_or_null[i0 + e] : lr;
      rule(P[e], G[e], grad_scale, l, S[0][e], S[1][e], S[2][e]);
    }
    *reinterpret_cast<float4*>(p + i0) = make_float4(P[0], P[1], P[2], P[3]);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (s[k]) *reinterpret_cast<float4*>(s[k] + i0) = make_float4(S[k][0], S[k][1], S[k][2], S[k][3]);
  } else {
    for (int64_t i = i0; i < n; ++i) {
      const float l = lr_scale_or_null ? lr * lr_scale_or_null[i] : lr;
      float x[3] = {s0 ? s0[i] : 0.f, s1 ? s1[i] : 0.f, s2 ? s2[i] : 0.f};
      rule(p[i], g[i], grad_scale, l, x[0], x[1], x[2]);
      for (int k = 0; k < 3; ++k)
        if (s[k]) s[k][i] = x[k];
    }
  }
}

static unsigned flat_update_grid(int64_t n) { return (unsigned)(((n + 3) / 4 + 255) / 256); }

// found_inf = 1 when any of g[0..n) is non-finite (the flat gradient after the all-reduce; the trainer appends the
// loss as one more element), else 0 -- GradScaler.unscale_'s inf check (train.py:490-512) without the host sync.
// Grid-stride, 128-bit loads; a CTA that sees a non-finite value writes the flag (benign race: all write 1).
__global__ void __launch_bounds__(256) grad_check_kernel(const float* __restrict__ g, int64_t n,
                                                        float* __restrict__ found_inf) {
  bool bad = false;
  const int64_t nv = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 x = reinterpret_cast<const float4*>(g)[i];
    // finite <=> x - x == 0
    bad |= !((x.x - x.x) == 0.f) | !((x.y - x.y) == 0.f) | !((x.z - x.z) == 0.f) | !((x.w - x.w) == 0.f);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float x = g[nv * 4 + threadIdx.x];
    bad |= !((x - x) == 0.f);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.f;
}

// Global gradient norm for clip_grad_norm_ (train.py:501-512), fused with the check above.  Pass 1: each CTA writes the
// fp64 sum of squares of its share of g[0..n_norm) to part[blockIdx.x]; an element of g[n_norm..n_check) adds x - x
// (0, or NaN when x is not finite), so a non-finite checked value makes the sum NaN, as an inf or NaN normed value does
// through its square.  fp64 squares of finite floats cannot overflow.  Pass 2 (one CTA) sums the partials.  Every
// thread's share and every tree step is fixed by n_norm and the grid, which depends on n_norm only: deterministic.
constexpr int kNormThreads = 256;
constexpr int kNormMaxCtas = 1024;

__device__ __forceinline__ double block_sum_f64(double v) {  // fixed tree; result valid in thread 0
  __shared__ double red[kNormThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = 0.0;
  if (threadIdx.x == 0)
#pragma unroll
    for (int w = 0; w < kNormThreads / 32; ++w) v += red[w];
  return v;
}

__device__ __forceinline__ double sq4(double acc, float4 x) {
  acc = fma((double)x.x, (double)x.x, acc);
  acc = fma((double)x.y, (double)x.y, acc);
  acc = fma((double)x.z, (double)x.z, acc);
  return fma((double)x.w, (double)x.w, acc);
}

__global__ void __launch_bounds__(kNormThreads) grad_sumsq_kernel(const float* __restrict__ g, int64_t n_norm,
                                                                 int64_t n_check, double* __restrict__ part) {
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const int64_t nv = n_norm / 4, stride = (int64_t)gridDim.x * kNormThreads;
  int64_t i = (int64_t)blockIdx.x * kNormThreads + threadIdx.x;
  double acc = 0.0;
  for (; i + stride < nv; i += 2 * stride) {  // two independent 128-bit loads in flight per thread
    const float4 a = g4[i], b = g4[i + stride];
    acc = sq4(sq4(acc, a), b);
  }
  if (i < nv) acc = sq4(acc, g4[i]);
  if (blockIdx.x == 0 && threadIdx.x < (n_norm & 3)) {
    const double x = g[nv * 4 + threadIdx.x];
    acc = fma(x, x, acc);
  }
  for (int64_t j = n_norm + (int64_t)blockIdx.x * kNormThreads + threadIdx.x; j < n_check; j += stride)
    acc += (double)(g[j] - g[j]);
  acc = block_sum_f64(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kNormThreads) grad_norm_finish_kernel(const double* __restrict__ part, int nparts,
                                                                       float grad_scale,
                                                                       const float* __restrict__ loss_scale,
                                                                       float max_norm, float* __restrict__ found_inf,
                                                                       float* __restrict__ norm_out,
                                                                       float* __restrict__ adam_div_out) {
  double acc = 0.0;
  for (int j = threadIdx.x; j < nparts; j += kNormThreads) acc += part[j];
  acc = block_sum_f64(acc);
  if (threadIdx.x == 0) {
    const float s = loss_scale ? *loss_scale : 1.f;
    const float norm = (float)(sqrt(acc) * fabs((double)grad_scale / (double)s));
    const bool bad = !isfinite(norm);
    // torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to at most 1, in fp32
    const float coef = fminf(max_norm / (norm + 1e-6f), 1.f);
    *found_inf = bad ? 1.f : 0.f;
    *norm_out = norm;
    *adam_div_out = bad ? s : s / coef;
  }
}

// One thread: advance the step count unless the step is skipped, and update the loss scale like
// torch.amp.GradScaler.update (backoff on overflow, growth after `growth_interval` clean steps).
__global__ void amp_update_kernel(const float* __restrict__ found_inf, int* __restrict__ step,
                                  float* __restrict__ loss_scale, int* __restrict__ growth_tracker,
                                  float growth_factor, float backoff_factor, int growth_interval) {
  const bool inf = *found_inf != 0.f;
  if (step && !inf) *step += 1;
  if (loss_scale) {
    if (inf) {
      *loss_scale *= backoff_factor;
      if (growth_tracker) *growth_tracker = 0;
    } else if (growth_tracker) {
      const int t = *growth_tracker + 1;
      if (t == growth_interval) {
        *loss_scale *= growth_factor;
        *growth_tracker = 0;
      } else {
        *growth_tracker = t;
      }
    }
  }
}

// fp32 -> bf16 cast of a flat buffer (bf16 shadow of the weights / activations)
__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                       int64_t n) {
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= n) return;
  if (i0 + 8 <= n) {
    Vec8<float> a = Vec8<float>::load(src + i0);
    Vec8<__nv_bfloat16> b;
#pragma unroll
    for (int e = 0; e < 8; ++e) b.v[e] = a.v[e];
    b.store(dst + i0);
  } else {
    for (int64_t i = i0; i < n; ++i) dst[i] = __float2bfloat16(src[i]);
  }
}

// dW[c][d] = sum_t g[t][c] * kp[t][d]: the weight gradient of the Fourier position encoder's projection
// (lightglue.py:37-44; theta = kp Wr^T with kp [T, 2 or 4]), a tall-skinny contraction cuBLAS runs as split-K sgemm +
// memset (0.2 ms per step).  C = head_dim / 2 = 32 or 16 angles: a warp reads 32 / C consecutive 4C-byte rows of g
// (128 bytes), 256 / C rows in flight per CTA; per-CTA partials, summed over the CTA's rows in a fixed order.
template <int C>
__global__ void __launch_bounds__(256) posenc_wgrad_kernel(const float* __restrict__ g, const float* __restrict__ kp,
                                                          float* __restrict__ part, int64_t T, int KD) {
  constexpr int kRows = 256 / C;
  __shared__ float red[kRows][C][4];
  const int c = threadIdx.x % C, slot = threadIdx.x / C;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int64_t t = (int64_t)blockIdx.x * kRows + slot; t < T; t += (int64_t)gridDim.x * kRows) {
    const float gv = __ldg(g + t * C + c);
#pragma unroll
    for (int d = 0; d < 4; ++d)
      if (d < KD) acc[d] = fmaf(gv, __ldg(kp + t * KD + d), acc[d]);
  }
#pragma unroll
  for (int d = 0; d < 4; ++d) red[slot][c][d] = acc[d];
  __syncthreads();
  if (slot == 0) {
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      float v = 0.f;
#pragma unroll
      for (int s8 = 0; s8 < kRows; ++s8) v += red[s8][c][d];
      if (d < KD) part[((int64_t)blockIdx.x * C + c) * KD + d] = v;
    }
  }
}

// Row and column counts of a 0/1 byte mask [B,M,N] in one pass (the ground-truth assignment's `gt.sum(2)` / `gt.sum(1)`,
// lightglue.py:595-600; torch first widens the 4.2 MB/pair mask to fp32 for each of the two sums).  A warp owns whole
// rows: per row a dp4a byte sum + shuffle reduce; the same 16-byte loads accumulate this lane's 16 columns byte-wise
// over the warp's 8 rows, flushed as exact integer-valued float atomics (only the non-zero ones: the mask is sparse).
constexpr int kMcRows = 64, kMcChunks = 8;
__global__ void __launch_bounds__(256) mask_counts_kernel(const uint8_t* __restrict__ mask, float* __restrict__ rowcnt,
                                                         float* __restrict__ colcnt, int M, int N) {
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * kMcRows, r1 = min(M, r0 + kMcRows);
  const uint8_t* mb = mask + (int64_t)b * M * N;
  uint32_t acc[kMcChunks][4];
#pragma unroll
  for (int c = 0; c < kMcChunks; ++c) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0u;
  for (int r = r0 + warp; r < r1; r += 8) {
    unsigned rs = 0u;
#pragma unroll
    for (int c = 0; c < kMcChunks; ++c) {
      const int col = c * 512 + lane * 16;
      if (col < N) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(mb + (int64_t)r * N + col));
        rs = __dp4a(v.x, 0x01010101u, __dp4a(v.y, 0x01010101u, __dp4a(v.z, 0x01010101u, __dp4a(v.w, 0x01010101u, rs))));
        acc[c][0] = __vadd4(acc[c][0], v.x);
        acc[c][1] = __vadd4(acc[c][1], v.y);
        acc[c][2] = __vadd4(acc[c][2], v.z);
        acc[c][3] = __vadd4(acc[c][3], v.w);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
    if (lane == 0) rowcnt[(int64_t)b * M + r] = (float)rs;
  }
#pragma unroll
  for (int c = 0; c < kMcChunks; ++c) {
    const int col = c * 512 + lane * 16;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (acc[c][k] == 0u) continue;
#pragma unroll
      for (int by = 0; by < 4; ++by) {
        const uint32_t n = (acc[c][k] >> (8 * by)) & 0xffu;
        if (n) atomicAdd(colcnt + (int64_t)b * N + col + 4 * k + by, (float)n);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// column sums of a tall [rows, cols] matrix: block = 32 row-lanes x 8 column-vectors (8 elements = one 128-bit load
// for bf16), row slabs across blockIdx.y, deterministic two-stage sum.  `Op` says what is summed: Op::K per-element
// terms of the row data it loads, accumulated in Op::Acc; out = [K, cols].
//   ColsumPlain  : the column sums themselves (bias gradients), fp32
//   BnStats      : sum x, sum x^2 (BatchNorm statistics), fp64, and the row count behind them
//   BnReluBwdSums: sum dy', sum dy' xhat with dy' = dy [relu output > 0] (BatchNorm + ReLU backward), fp64
// ---------------------------------------------------------------------------------------------
template <typename T>
struct ColsumPlain {
  using Acc = float;
  static constexpr int K = 1;
  const T* a;
  struct Ctx {};
  using Raw = Vec8<T>;
  __device__ Ctx ctx(int) const { return {}; }
  __device__ Raw load(int64_t r, int cols, int col0) const { return Vec8<T>::load(a + r * cols + col0); }
  __device__ Acc term(const Ctx&, const Raw& v, int, int e) const { return v.v[e]; }
  __device__ void finish(Acc*, int64_t, int) const {}
};

template <typename T>
struct BnStats {
  using Acc = double;  // exact enough for sum x^2 - n mean^2 when |mean| >> std
  static constexpr int K = 2;
  const T* x;
  struct Ctx {};
  using Raw = Vec8<T>;
  __device__ Ctx ctx(int) const { return {}; }
  __device__ Raw load(int64_t r, int cols, int col0) const { return Vec8<T>::load(x + r * cols + col0); }
  __device__ Acc term(const Ctx&, const Raw& v, int k, int e) const {
    const double d = v.v[e];
    return k == 0 ? d : d * d;
  }
  __device__ void finish(Acc* out, int64_t rows, int cols) const { out[2 * cols] = (double)rows; }
};

// normalised input and pre-activation of BatchNorm + ReLU; forward and backward evaluate the same expressions, so the
// backward's ReLU mask equals the forward's
__device__ __forceinline__ float bn_xhat(float v, float mu, float rs) { return (v - mu) * rs; }
__device__ __forceinline__ float bn_pre(float xh, float g, float b) { return fmaf(xh, g, b); }

template <typename T>
struct BnReluBwdSums {
  using Acc = double;
  static constexpr int K = 2;
  const T* dy;
  const T* x;
  const float *mean, *rstd, *gamma, *beta;
  struct Ctx {
    float mu[8], rs[8], g[8], b[8];
  };
  struct Raw {
    Vec8<T> x, g;
  };
  __device__ Ctx ctx(int col0) const {
    Ctx c;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      c.mu[e] = mean[col0 + e];
      c.rs[e] = rstd[col0 + e];
      c.g[e] = gamma[col0 + e];
      c.b[e] = beta[col0 + e];
    }
    return c;
  }
  __device__ Raw load(int64_t r, int cols, int col0) const {
    return {Vec8<T>::load(x + r * cols + col0), Vec8<T>::load(dy + r * cols + col0)};
  }
  __device__ Acc term(const Ctx& c, const Raw& v, int k, int e) const {
    const float xh = bn_xhat(v.x.v[e], c.mu[e], c.rs[e]);
    const float d = bn_pre(xh, c.g[e], c.b[e]) > 0.f ? v.g.v[e] : 0.f;
    return k == 0 ? (double)d : (double)d * (double)xh;
  }
  __device__ void finish(Acc*, int64_t, int) const {}
};

template <typename Op>
__global__ void __launch_bounds__(256) colsum_kernel(Op op, typename Op::Acc* __restrict__ part,
                                                    typename Op::Acc* __restrict__ out,
                                                    unsigned* __restrict__ counter, int64_t rows, int cols,
                                                    int rows_per_slab) {
  using Acc = typename Op::Acc;
  constexpr int K = Op::K;
  __shared__ Acc s_red[32][65];
  __shared__ bool s_last;
  const int cx = threadIdx.x & 7, ry = threadIdx.x >> 3;
  const int col0 = blockIdx.x * 64 + cx * 8;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_slab;
  const int64_t r1 = min(rows, r0 + rows_per_slab);
  Acc acc[K][8];
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[k][e] = Acc(0);
  if (col0 < cols) {
    const typename Op::Ctx c = op.ctx(col0);
    int64_t r = r0 + ry;
    for (; r + 96 < r1; r += 128) {  // four independent 16-byte loads in flight per thread
      const typename Op::Raw v0 = op.load(r, cols, col0), v1 = op.load(r + 32, cols, col0);
      const typename Op::Raw v2 = op.load(r + 64, cols, col0), v3 = op.load(r + 96, cols, col0);
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e)
          acc[k][e] += (op.term(c, v0, k, e) + op.term(c, v1, k, e)) + (op.term(c, v2, k, e) + op.term(c, v3, k, e));
    }
    for (; r < r1; r += 32) {
      const typename Op::Raw v = op.load(r, cols, col0);
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[k][e] += op.term(c, v, k, e);
    }
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (k > 0) __syncthreads();  // the previous term's slab sums have been read out of s_red
#pragma unroll
    for (int e = 0; e < 8; ++e) s_red[ry][cx * 8 + e] = acc[k][e];
    __syncthreads();
    if (threadIdx.x < 64 && blockIdx.x * 64 + threadIdx.x < cols) {
      Acc t = Acc(0);
#pragma unroll
      for (int r = 0; r < 32; ++r) t += s_red[r][threadIdx.x];
      part[((int64_t)blockIdx.y * K + k) * cols + blockIdx.x * 64 + threadIdx.x] = t;
    }
  }
  // the last CTA of this column block to finish sums the slab partials in slab order (deterministic)
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(&counter[blockIdx.x], 1u);
    s_last = (prev == gridDim.y - 1);
    if (s_last) counter[blockIdx.x] = 0u;  // self-resetting for the next call
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    const int c = blockIdx.x * 64 + (threadIdx.x & 63);
    if (threadIdx.x < 64 && c < cols) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        Acc t = Acc(0);
        for (unsigned sidx = 0; sidx < gridDim.y; ++sidx) t += __ldcg(&part[((int64_t)sidx * K + k) * cols + c]);
        out[k * cols + c] = t;
      }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) op.finish(out, rows, cols);
  }
}

template <typename Op>
static int colsum_launch(const Op& op, typename Op::Acc* out, typename Op::Acc* ws, unsigned* counters, int64_t rows,
                         int cols, cudaStream_t stream) {
  const int nslabs = lgb200_colsum_slabs(rows, cols);
  const int rps = (int)((rows + nslabs - 1) / nslabs);
  colsum_kernel<Op><<<dim3((cols + 63) / 64, nslabs), 256, 0, stream>>>(op, ws, out, counters, rows, cols, rps);
  return check_launch("colsum");
}

// ---------------------------------------------------------------------------------------------
// BatchNorm + ReLU, token-major x [ntok, C], C a power of two in [8, 512].  Thread <-> 8 consecutive channels of a
// row; the grid stride is a multiple of C / 8, so a thread keeps its channels.  Each CTA turns the per-channel
// statistics into scale / shift in shared memory first (every CTA evaluates the same expressions: identical values).
// ---------------------------------------------------------------------------------------------
constexpr int kBnMaxC = 512;

__device__ __forceinline__ int64_t bn_grid_stride() { return (int64_t)gridDim.x * blockDim.x; }

// One momentum step of the running statistics from the batch statistics in `sums` (unbiased variance).
__device__ __forceinline__ void bn_running_step(const double* __restrict__ sums, float* __restrict__ rmean,
                                                float* __restrict__ rvar, float momentum, int c, int C) {
  const double n = sums[2 * C];
  const double m = sums[c] / n;
  const double var = fmax(sums[C + c] / n - m * m, 0.0);
  rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)m;
  rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)(var * n / (n - 1.0));
}

__global__ void bn_running_update_kernel(const double* __restrict__ sums, float* __restrict__ rmean,
                                         float* __restrict__ rvar, float momentum, int C) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) bn_running_step(sums, rmean, rvar, momentum, c, C);
}

// sums = [sum x (C) | sum x^2 (C) | count] (fp64, possibly summed over ranks): training mode; NULL: eval mode with the
// running statistics.  Block 0 writes the saved mean / rstd and, in training mode, updates the running statistics
// (momentum, unbiased variance with the count in `sums`).
template <typename T>
__global__ void __launch_bounds__(256) bn_relu_fwd_kernel(const T* __restrict__ x, const double* __restrict__ sums,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float* __restrict__ rmean,
                                                         float* __restrict__ rvar, float momentum, float eps,
                                                         T* __restrict__ y, float* __restrict__ save_mean,
                                                         float* __restrict__ save_rstd, int64_t ntok, int C) {
  __shared__ float s_mu[kBnMaxC], s_rs[kBnMaxC];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mu, rs;
    if (sums) {
      const double n = sums[2 * C];
      const double m = sums[c] / n;
      const double var = fmax(sums[C + c] / n - m * m, 0.0);
      mu = (float)m;
      rs = 1.f / sqrtf((float)var + eps);
      if (blockIdx.x == 0 && rmean) bn_running_step(sums, rmean, rvar, momentum, c, C);
    } else {
      mu = rmean[c];
      rs = 1.f / sqrtf(rvar[c] + eps);
    }
    s_mu[c] = mu;
    s_rs[c] = rs;
    if (blockIdx.x == 0) {
      save_mean[c] = mu;
      save_rstd[c] = rs;
    }
  }
  __syncthreads();
  const int cv = C / 8;
  const int64_t start = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c0 = (int)(start % cv) * 8;
  float mu[8], rs[8], g[8], b[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = s_mu[c0 + e];
    rs[e] = s_rs[c0 + e];
    g[e] = gamma[c0 + e];
    b[e] = beta[c0 + e];
  }
  const int64_t n8 = ntok * cv;
  for (int64_t i = start; i < n8; i += bn_grid_stride()) {
    float v[8];
    Raw8<T>::load(x + i * 8).unpack(v);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float z = bn_pre(bn_xhat(v[e], mu[e], rs[e]), g[e], b[e]);
      v[e] = z < 0.f ? 0.f : z;  // NaN propagates like torch.relu
    }
    store8<T>(y + i * 8, v);
  }
}

// dx = gamma rstd (dy' - gsums[0:C] / n - xhat gsums[C:2C] / n), dy' = dy [pre-activation > 0], n = *count.
// gsums NULL: eval mode (the statistics are constants), dx = gamma rstd dy'.
template <typename T>
__global__ void __launch_bounds__(256) bn_relu_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta,
                                                         const float* __restrict__ mean,
                                                         const float* __restrict__ rstd,
                                                         const double* __restrict__ gsums,
                                                         const double* __restrict__ count, T* __restrict__ dx,
                                                         int64_t ntok, int C) {
  __shared__ float s_k1[kBnMaxC], s_k2[kBnMaxC];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    s_k1[c] = gsums ? (float)(gsums[c] / *count) : 0.f;
    s_k2[c] = gsums ? (float)(gsums[C + c] / *count) : 0.f;
  }
  __syncthreads();
  const int cv = C / 8;
  const int64_t start = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c0 = (int)(start % cv) * 8;
  float mu[8], rs[8], g[8], b[8], k1[8], k2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = mean[c0 + e];
    rs[e] = rstd[c0 + e];
    g[e] = gamma[c0 + e];
    b[e] = beta[c0 + e];
    k1[e] = s_k1[c0 + e];
    k2[e] = s_k2[c0 + e];
  }
  const int64_t n8 = ntok * cv;
  for (int64_t i = start; i < n8; i += bn_grid_stride()) {
    float v[8], d[8];
    Raw8<T>::load(x + i * 8).unpack(v);
    Raw8<T>::load(dy + i * 8).unpack(d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float xh = bn_xhat(v[e], mu[e], rs[e]);
      const float dd = bn_pre(xh, g[e], b[e]) > 0.f ? d[e] : 0.f;
      d[e] = (dd - k1[e] - xh * k2[e]) * (g[e] * rs[e]);
    }
    store8<T>(dx + i * 8, d);
  }
}

// x_out = x + y (fp32 residual stream) and its compute-dtype copy for the next GEMM, in one pass.  TY = element type of
// y: the compute dtype (a GEMM output added to the residual) or float (two fp32 gradient streams merged in backward).
template <typename T, typename TY = T>
__global__ void __launch_bounds__(256) residual_add_cast_kernel(const float* __restrict__ x, const TY* __restrict__ y,
                                                               float* __restrict__ xo, T* __restrict__ xc, int64_t n,
                                                               int64_t cols, int64_t cast_pitch) {
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= n) return;
  // the cast copy may be a column block of a wider matrix (row pitch cast_pitch > cols; cols % 8 == 0 then)
  if (xc && cast_pitch != cols) xc += (i0 / cols) * cast_pitch + (i0 % cols) - i0;
  if (i0 + 8 <= n) {
    Vec8<float> a = Vec8<float>::load(x + i0);
    if (y) {
      Vec8<TY> b = Vec8<TY>::load(y + i0);
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] += b.v[e];
    }
    if (xo) a.store(xo + i0);
    Vec8<T> c;
#pragma unroll
    for (int e = 0; e < 8; ++e) c.v[e] = a.v[e];
    if (xc) c.store(xc + i0);
  } else {
    for (int64_t i = i0; i < n; ++i) {
      float v = x[i] + (y ? (float)y[i] : 0.f);
      if (xo) xo[i] = v;
      if (xc) xc[i] = (T)v;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Token heads of one supervised layer (matchability lightglue.py:259-267, token confidence :74-83):
// one warp per token, lane owns 8 consecutive features per 256-column chunk.
//   fwd: zt[t] = (x.wm + bm, x.wt + bt), ls/du = log sigmoid(+-zt[t,0]), and the compute-dtype copy of x that feeds
//        final_proj -- one pass over x instead of cast + skinny GEMM + logsigmoid.
//   bwd: dx = float(dmdw) + dzt[:,0] wm  (the confidence head reads a detached x),
//        dW2[j] = sum_t dzt[t,j] x[t], db2[j] = sum_t dzt[t,j]; per-CTA partials, last CTA sums them in order.
// ---------------------------------------------------------------------------------------------
template <typename T, int NCH>
__global__ void __launch_bounds__(256) head_token_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wm,
                                                            const float* __restrict__ bm,
                                                            const float* __restrict__ wt,
                                                            const float* __restrict__ bt, T* __restrict__ xc,
                                                            float* __restrict__ zt, float* __restrict__ ls,
                                                            float* __restrict__ du, int64_t ntok, int D) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  Vec8<float> m[NCH], c[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int col = ch * 256 + lane * 8;
    if (col < D) {
      m[ch] = Vec8<float>::load(wm + col);
      c[ch] = Vec8<float>::load((wt ? wt : wm) + col);
    }
  }
  const float b0 = *bm, b1 = wt ? *bt : *bm;
  for (int64_t tok = (int64_t)blockIdx.x * 8 + warp; tok < ntok; tok += (int64_t)gridDim.x * 8) {
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int col = ch * 256 + lane * 8;
      if (col < D) {
        const Vec8<float> v = Vec8<float>::load(x + tok * D + col);
        if (xc) {
          Vec8<T> o;
#pragma unroll
          for (int e = 0; e < 8; ++e) o.v[e] = v.v[e];
          o.store(xc + tok * D + col);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          s0 = fmaf(v.v[e], m[ch].v[e], s0);
          s1 = fmaf(v.v[e], c[ch].v[e], s1);
        }
      }
    }
    s0 = warp_sum(s0) + b0;
    s1 = warp_sum(s1) + b1;
    if (lane == 0) {
      *reinterpret_cast<float2*>(zt + 2 * tok) = make_float2(s0, s1);
      const float l = log_sigmoid(s0);
      ls[tok] = l;
      du[tok] = l - s0;
    }
  }
}

constexpr int kHeadBwdParts = 592;  // 4 CTAs per SM

template <typename T, int NCH>
__global__ void __launch_bounds__(256) head_token_bwd_kernel(const float* __restrict__ x, const T* __restrict__ dmdw,
                                                            const float* __restrict__ dzt,
                                                            const float* __restrict__ wm, float* __restrict__ dx,
                                                            float* __restrict__ dW2, float* __restrict__ db2,
                                                            float* __restrict__ part, unsigned* __restrict__ counter,
                                                            int64_t ntok, int D) {
  __shared__ float s_red[8][2 * 256 * NCH + 2];
  __shared__ bool s_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  Vec8<float> m[NCH];
  float a0[NCH][8], a1[NCH][8], sb0 = 0.f, sb1 = 0.f;
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int col = ch * 256 + lane * 8;
    if (col < D) m[ch] = Vec8<float>::load(wm + col);
#pragma unroll
    for (int e = 0; e < 8; ++e) a0[ch][e] = a1[ch][e] = 0.f;
  }
  for (int64_t tok = (int64_t)blockIdx.x * 8 + warp; tok < ntok; tok += (int64_t)gridDim.x * 8) {
    const float2 dz = *reinterpret_cast<const float2*>(dzt + 2 * tok);
    sb0 += dz.x;
    sb1 += dz.y;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int col = ch * 256 + lane * 8;
      if (col < D) {
        const Vec8<float> v = Vec8<float>::load(x + tok * D + col);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          a0[ch][e] = fmaf(dz.x, v.v[e], a0[ch][e]);
          a1[ch][e] = fmaf(dz.y, v.v[e], a1[ch][e]);
        }
        if (dx) {  // null: x needs no gradient (every layer up to this head is frozen)
          const Vec8<T> g = Vec8<T>::load(dmdw + tok * D + col);
          Vec8<float> o;
#pragma unroll
          for (int e = 0; e < 8; ++e) o.v[e] = fmaf(dz.x, m[ch].v[e], g.v[e]);
          o.store(dx + tok * D + col);
        }
      }
    }
  }
  // CTA partial: [dW2 row 0 (D) | dW2 row 1 (D) | db2 (2)]
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int col = ch * 256 + lane * 8;
    if (col < D) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s_red[warp][col + e] = a0[ch][e];
        s_red[warp][D + col + e] = a1[ch][e];
      }
    }
  }
  if (lane == 0) {
    s_red[warp][2 * D] = sb0;
    s_red[warp][2 * D + 1] = sb1;
  }
  __syncthreads();
  const int width = 2 * D + 2;
  for (int c = threadIdx.x; c < width; c += 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_red[w][c];
    part[(int64_t)blockIdx.x * width + c] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(counter, 1u);
    s_last = (prev == gridDim.x - 1);
    if (s_last) *counter = 0u;  // self-resetting for the next call
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    for (int c = threadIdx.x; c < width; c += 256) {
      float t = 0.f;
      for (unsigned p = 0; p < gridDim.x; ++p) t += __ldcg(&part[(int64_t)p * width + c]);
      if (c < 2 * D) dW2[c] = t; else db2[c - 2 * D] = t;
    }
  }
}

// The kernels above read and write whole rows with 16-byte vector accesses: every such pointer must be 16-byte aligned
// (null pointers pass).  Checked on the host so a misaligned view is an LGB200_ERR_INVALID, not a device fault.
static bool aligned16(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}

}  // namespace lgb

using namespace lgb;

extern "C" {

int lgb200_colsum_slabs(int64_t rows, int cols) {
  const int cb = (cols + 63) / 64;
  int64_t want = (4 * device_sm_count() + cb - 1) / cb;  // ~4 CTAs per SM in total
  int64_t maxs = (rows + 255) / 256;                // at least 256 rows per slab
  int64_t n = want < maxs ? want : maxs;
  return (int)(n < 1 ? 1 : n);
}

int lgb200_posenc_wgrad_blocks(void) { return 2 * device_sm_count(); }
int lgb200_posenc_wgrad(const float* g, const float* kp, float* part, int64_t T, int C, int KD, cudaStream_t stream) {
  LGB_REQUIRE(g && kp && part && T > 0, kErrInvalid, "posenc_wgrad: bad arguments");
  LGB_REQUIRE((C == 32 || C == 16) && KD >= 1 && KD <= 4, kErrInvalid,
              "posenc_wgrad: C must be 32 or 16 and 1 <= KD <= 4 (got %d, %d)", C, KD);
  if (C == 32)
    posenc_wgrad_kernel<32><<<lgb200_posenc_wgrad_blocks(), 256, 0, stream>>>(g, kp, part, T, KD);
  else
    posenc_wgrad_kernel<16><<<lgb200_posenc_wgrad_blocks(), 256, 0, stream>>>(g, kp, part, T, KD);
  return check_launch("posenc_wgrad");
}

int lgb200_mask_counts(const uint8_t* mask, float* rowcnt, float* colcnt, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(mask && rowcnt && colcnt && B > 0 && M > 0 && N > 0, kErrInvalid, "mask_counts: bad arguments");
  LGB_REQUIRE(N % 16 == 0 && N <= 512 * kMcChunks && (reinterpret_cast<uintptr_t>(mask) & 15) == 0, kErrInvalid,
              "mask_counts: N must be a multiple of 16 and at most %d, mask 16-byte aligned", 512 * kMcChunks);
  cudaError_t e = cudaMemsetAsync(colcnt, 0, sizeof(float) * (size_t)B * N, stream);
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "mask_counts: memset: %s", cudaGetErrorString(e));
  mask_counts_kernel<<<dim3((M + kMcRows - 1) / kMcRows, B), 256, 0, stream>>>(mask, rowcnt, colcnt, M, N);
  return check_launch("mask_counts");
}

int lgb200_colsum(const void* a, float* out, float* ws, unsigned* counters, int64_t rows, int cols, int dtype,
                  cudaStream_t stream) {
  LGB_REQUIRE(a && out && ws && counters && rows > 0 && cols > 0, kErrInvalid, "colsum: bad arguments");
  LGB_REQUIRE(cols % 8 == 0, kErrInvalid, "colsum: cols must be a multiple of 8");
  if (dtype == LGB200_F32)
    return colsum_launch(ColsumPlain<float>{(const float*)a}, out, ws, counters, rows, cols, stream);
  if (dtype == LGB200_BF16)
    return colsum_launch(ColsumPlain<__nv_bfloat16>{(const __nv_bfloat16*)a}, out, ws, counters, rows, cols, stream);
  LGB_REQUIRE(false, kErrInvalid, "colsum: bad dtype %d", dtype);
}

static bool bn_channels_ok(int C) { return C >= 8 && C <= kBnMaxC && (C & (C - 1)) == 0; }

static unsigned bn_apply_grid(int64_t ntok, int C) {
  const int64_t blocks = (ntok * (C / 8) + 255) / 256, cap = 8 * (int64_t)device_sm_count();
  return (unsigned)(blocks < cap ? blocks : cap);
}

int lgb200_bn_stats(const void* x, double* sums, double* ws, unsigned* counters, int64_t ntok, int C, int dtype,
                    cudaStream_t stream) {
  LGB_REQUIRE(x && sums && ws && counters && ntok > 0, kErrInvalid, "bn_stats: bad arguments");
  LGB_REQUIRE(bn_channels_ok(C), kErrUnsupported, "bn_stats: C=%d is not a power of two in [8, %d]", C, kBnMaxC);
  LGB_REQUIRE(aligned16({x}), kErrInvalid, "bn_stats: misaligned pointer (16 bytes needed)");
  if (dtype == LGB200_F32) return colsum_launch(BnStats<float>{(const float*)x}, sums, ws, counters, ntok, C, stream);
  if (dtype == LGB200_BF16)
    return colsum_launch(BnStats<__nv_bfloat16>{(const __nv_bfloat16*)x}, sums, ws, counters, ntok, C, stream);
  LGB_REQUIRE(false, kErrInvalid, "bn_stats: bad dtype %d", dtype);
}

int lgb200_bn_running_update(const double* sums, float* running_mean, float* running_var, float momentum, int C,
                             cudaStream_t stream) {
  LGB_REQUIRE(sums && running_mean && running_var && C > 0, kErrInvalid, "bn_running_update: bad arguments");
  bn_running_update_kernel<<<1, 256, 0, stream>>>(sums, running_mean, running_var, momentum, C);
  return check_launch("bn_running_update");
}

int lgb200_bn_relu_fwd(const void* x, const double* sums, const float* gamma, const float* beta, float* running_mean,
                       float* running_var, float momentum, float eps, void* y, float* save_mean, float* save_rstd,
                       int64_t ntok, int C, int dtype, cudaStream_t stream) {
  LGB_REQUIRE(x && gamma && beta && y && save_mean && save_rstd && ntok > 0, kErrInvalid, "bn_relu_fwd: bad arguments");
  LGB_REQUIRE((running_mean == nullptr) == (running_var == nullptr), kErrInvalid,
              "bn_relu_fwd: running_mean / running_var must both be set or both be null");
  LGB_REQUIRE(sums || running_mean, kErrInvalid, "bn_relu_fwd: eval mode needs the running statistics");
  LGB_REQUIRE(bn_channels_ok(C), kErrUnsupported, "bn_relu_fwd: C=%d is not a power of two in [8, %d]", C, kBnMaxC);
  LGB_REQUIRE(aligned16({x, y}), kErrInvalid, "bn_relu_fwd: misaligned pointer (16 bytes needed)");
  const unsigned grid = bn_apply_grid(ntok, C);
  if (dtype == LGB200_F32)
    bn_relu_fwd_kernel<float><<<grid, 256, 0, stream>>>((const float*)x, sums, gamma, beta, running_mean, running_var,
                                                        momentum, eps, (float*)y, save_mean, save_rstd, ntok, C);
  else if (dtype == LGB200_BF16)
    bn_relu_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)x, sums, gamma, beta,
                                                                running_mean, running_var, momentum, eps,
                                                                (__nv_bfloat16*)y, save_mean, save_rstd, ntok, C);
  else
    LGB_REQUIRE(false, kErrInvalid, "bn_relu_fwd: bad dtype %d", dtype);
  return check_launch("bn_relu_fwd");
}

int lgb200_bn_relu_bwd_reduce(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                              const float* rstd, double* sums, double* ws, unsigned* counters, int64_t ntok, int C,
                              int dtype, cudaStream_t stream) {
  LGB_REQUIRE(dy && x && gamma && beta && mean && rstd && sums && ws && counters && ntok > 0, kErrInvalid,
              "bn_relu_bwd_reduce: bad arguments");
  LGB_REQUIRE(bn_channels_ok(C), kErrUnsupported, "bn_relu_bwd_reduce: C=%d is not a power of two in [8, %d]", C,
              kBnMaxC);
  LGB_REQUIRE(aligned16({dy, x}), kErrInvalid, "bn_relu_bwd_reduce: misaligned pointer (16 bytes needed)");
  if (dtype == LGB200_F32)
    return colsum_launch(BnReluBwdSums<float>{(const float*)dy, (const float*)x, mean, rstd, gamma, beta}, sums, ws,
                         counters, ntok, C, stream);
  if (dtype == LGB200_BF16)
    return colsum_launch(BnReluBwdSums<__nv_bfloat16>{(const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, mean, rstd,
                                                      gamma, beta},
                         sums, ws, counters, ntok, C, stream);
  LGB_REQUIRE(false, kErrInvalid, "bn_relu_bwd_reduce: bad dtype %d", dtype);
}

int lgb200_bn_relu_bwd(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                       const float* rstd, const double* sums, const double* count, void* dx, int64_t ntok, int C,
                       int dtype, cudaStream_t stream) {
  LGB_REQUIRE(dy && x && gamma && beta && mean && rstd && dx && ntok > 0, kErrInvalid, "bn_relu_bwd: bad arguments");
  LGB_REQUIRE((sums == nullptr) == (count == nullptr), kErrInvalid, "bn_relu_bwd: sums / count must both be set or null");
  LGB_REQUIRE(bn_channels_ok(C), kErrUnsupported, "bn_relu_bwd: C=%d is not a power of two in [8, %d]", C, kBnMaxC);
  LGB_REQUIRE(aligned16({dy, x, dx}), kErrInvalid, "bn_relu_bwd: misaligned pointer (16 bytes needed)");
  const unsigned grid = bn_apply_grid(ntok, C);
  if (dtype == LGB200_F32)
    bn_relu_bwd_kernel<float><<<grid, 256, 0, stream>>>((const float*)dy, (const float*)x, gamma, beta, mean, rstd,
                                                        sums, count, (float*)dx, ntok, C);
  else if (dtype == LGB200_BF16)
    bn_relu_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                                gamma, beta, mean, rstd, sums, count,
                                                                (__nv_bfloat16*)dx, ntok, C);
  else
    LGB_REQUIRE(false, kErrInvalid, "bn_relu_bwd: bad dtype %d", dtype);
  return check_launch("bn_relu_bwd");
}

int lgb200_residual_add_cast_pitched(const float* x, const void* y, float* x_out, void* x_cast, int64_t rows,
                                     int64_t cols, int64_t cast_pitch, int dtype, cudaStream_t stream) {
  LGB_REQUIRE(x && (x_out || x_cast) && rows > 0 && cols > 0, kErrInvalid, "residual_add_cast: bad arguments");
  LGB_REQUIRE(cast_pitch >= cols, kErrInvalid, "residual_add_cast: cast pitch %lld < cols %lld", (long long)cast_pitch,
              (long long)cols);
  LGB_REQUIRE(cast_pitch == cols || (cols % 8 == 0 && cast_pitch % 8 == 0), kErrInvalid,
              "residual_add_cast: a pitched cast output needs cols and pitch to be multiples of 8");
  LGB_REQUIRE(aligned16({x, y, x_out, x_cast}), kErrInvalid, "residual_add_cast: misaligned pointer (16 bytes needed)");
  const int64_t n = rows * cols;
  const unsigned grid = (unsigned)(((n + 7) / 8 + 255) / 256);
  if (dtype == LGB200_F32)
    residual_add_cast_kernel<float><<<grid, 256, 0, stream>>>(x, (const float*)y, x_out, (float*)x_cast, n, cols,
                                                              cast_pitch);
  else if (dtype == LGB200_BF16)
    residual_add_cast_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(x, (const __nv_bfloat16*)y, x_out,
                                                                      (__nv_bfloat16*)x_cast, n, cols, cast_pitch);
  else
    LGB_REQUIRE(false, kErrInvalid, "residual_add_cast: bad dtype %d", dtype);
  return check_launch("residual_add_cast");
}

int lgb200_add_f32_cast(const float* x, const float* y, float* x_out, void* x_cast, int64_t n, int dtype,
                        cudaStream_t stream) {
  LGB_REQUIRE(x && y && (x_out || x_cast) && n > 0, kErrInvalid, "add_f32_cast: bad arguments");
  LGB_REQUIRE(aligned16({x, y, x_out, x_cast}), kErrInvalid, "add_f32_cast: misaligned pointer (16 bytes needed)");
  const unsigned grid = (unsigned)(((n + 7) / 8 + 255) / 256);
  if (dtype == LGB200_F32)
    residual_add_cast_kernel<float, float><<<grid, 256, 0, stream>>>(x, y, x_out, (float*)x_cast, n, n, n);
  else if (dtype == LGB200_BF16)
    residual_add_cast_kernel<__nv_bfloat16, float><<<grid, 256, 0, stream>>>(x, y, x_out, (__nv_bfloat16*)x_cast, n, n, n);
  else
    LGB_REQUIRE(false, kErrInvalid, "add_f32_cast: bad dtype %d", dtype);
  return check_launch("add_f32_cast");
}

int lgb200_residual_add_cast(const float* x, const void* y, float* x_out, void* x_cast, int64_t n, int dtype,
                             cudaStream_t stream) {
  LGB_REQUIRE(n > 0, kErrInvalid, "residual_add_cast: bad arguments");
  return lgb200_residual_add_cast_pitched(x, y, x_out, x_cast, 1, n, n, dtype, stream);
}

int lgb200_rope_split_fwd_hd(const void* qkv, const float* theta, void* q, void* k, void* v, int64_t ntok, int H,
                             int dtype, int head_dim, cudaStream_t stream) {
  LGB_REQUIRE(head_dim == 32 || head_dim == 64, kErrUnsupported, "rope_split_fwd: head_dim %d (built for 32 and 64)",
              head_dim);
  LGB_REQUIRE(qkv && theta && q && k && v, kErrInvalid, "rope_split_fwd: null pointer");
  LGB_REQUIRE(ntok > 0 && H > 0, kErrInvalid, "rope_split_fwd: empty input");
  LGB_REQUIRE(aligned16({qkv, theta, q, k, v}), kErrInvalid, "rope_split_fwd: misaligned pointer (16 bytes needed)");
  LGB_REQUIRE(dtype == LGB200_F32 || dtype == LGB200_BF16, kErrInvalid, "rope_split_fwd: bad dtype %d", dtype);
  const int64_t nthr = ntok * (head_dim / 8);
  const unsigned grid = (unsigned)((nthr + 255) / 256);
  if (dtype == LGB200_F32) {
    auto kern = head_dim == 64 ? rope_split_fwd_kernel<float, 64> : rope_split_fwd_kernel<float, 32>;
    kern<<<grid, 256, 0, stream>>>((const float*)qkv, theta, (float*)q, (float*)k, (float*)v, ntok, H);
  } else {
    auto kern = head_dim == 64 ? rope_split_fwd_kernel<__nv_bfloat16, 64> : rope_split_fwd_kernel<__nv_bfloat16, 32>;
    kern<<<grid, 256, 0, stream>>>((const __nv_bfloat16*)qkv, theta, (__nv_bfloat16*)q, (__nv_bfloat16*)k,
                                   (__nv_bfloat16*)v, ntok, H);
  }
  return check_launch("rope_split_fwd");
}

int lgb200_rope_split_fwd(const void* qkv, const float* theta, void* q, void* k, void* v, int64_t ntok, int H,
                          int dtype, cudaStream_t stream) {
  return lgb200_rope_split_fwd_hd(qkv, theta, q, k, v, ntok, H, dtype, 64, stream);
}

int lgb200_rope_split_bwd_hd(const void* dq, const void* dk, const void* dv, const void* q, const void* k,
                             const float* theta, void* dqkv, float* dtheta, int64_t ntok, int H, int dtype,
                             int head_dim, cudaStream_t stream) {
  LGB_REQUIRE(head_dim == 32 || head_dim == 64, kErrUnsupported, "rope_split_bwd: head_dim %d (built for 32 and 64)",
              head_dim);
  LGB_REQUIRE(dq && dk && dv && q && k && theta && dqkv, kErrInvalid, "rope_split_bwd: null pointer");
  LGB_REQUIRE(ntok > 0 && H > 0, kErrInvalid, "rope_split_bwd: empty input");
  LGB_REQUIRE(aligned16({dq, dk, dv, q, k, theta, dqkv, dtheta}), kErrInvalid,
              "rope_split_bwd: misaligned pointer (16 bytes needed)");
  LGB_REQUIRE(dtype == LGB200_F32 || dtype == LGB200_BF16, kErrInvalid, "rope_split_bwd: bad dtype %d", dtype);
  const int64_t nthr = ntok * (head_dim / 8);
  const unsigned grid = (unsigned)((nthr + 255) / 256);
  if (dtype == LGB200_F32) {
    auto kern = head_dim == 64 ? rope_split_bwd_kernel<float, 64> : rope_split_bwd_kernel<float, 32>;
    kern<<<grid, 256, 0, stream>>>((const float*)dq, (const float*)dk, (const float*)dv, (const float*)q,
                                   (const float*)k, theta, (float*)dqkv, dtheta, ntok, H);
  } else {
    auto kern = head_dim == 64 ? rope_split_bwd_kernel<__nv_bfloat16, 64> : rope_split_bwd_kernel<__nv_bfloat16, 32>;
    kern<<<grid, 256, 0, stream>>>((const __nv_bfloat16*)dq, (const __nv_bfloat16*)dk, (const __nv_bfloat16*)dv,
                                   (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, theta, (__nv_bfloat16*)dqkv,
                                   dtheta, ntok, H);
  }
  return check_launch("rope_split_bwd");
}

int lgb200_rope_split_bwd(const void* dq, const void* dk, const void* dv, const void* q, const void* k,
                          const float* theta, void* dqkv, float* dtheta, int64_t ntok, int H, int dtype,
                          cudaStream_t stream) {
  return lgb200_rope_split_bwd_hd(dq, dk, dv, q, k, theta, dqkv, dtheta, ntok, H, dtype, 64, stream);
}

}  // extern "C"

template <typename T>
static int ln_gelu_fwd_dispatch(const void* x, const float* gamma, const float* beta, void* y, float* mean,
                                float* rstd, int64_t ntok, int W, float eps, cudaStream_t stream) {
  const unsigned grid2 = (unsigned)((ntok + 15) / 16), grid1 = (unsigned)((ntok + 7) / 8);
  switch (W) {
    case 256: ln_gelu_fwd_kernel<T, 1, 2><<<grid2, 256, 0, stream>>>((const T*)x, gamma, beta, (T*)y, mean, rstd, ntok, eps); break;
    case 512: ln_gelu_fwd_kernel<T, 2, 2><<<grid2, 256, 0, stream>>>((const T*)x, gamma, beta, (T*)y, mean, rstd, ntok, eps); break;
    case 1024: ln_gelu_fwd_kernel<T, 4, 1><<<grid1, 256, 0, stream>>>((const T*)x, gamma, beta, (T*)y, mean, rstd, ntok, eps); break;
    default: LGB_REQUIRE(false, kErrUnsupported, "ln_gelu: width %d not in {256,512,1024}", W);
  }
  return check_launch("ln_gelu_fwd");
}

extern "C" {

int lgb200_ln_gelu_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                       int64_t ntok, int W, float eps, int dtype, cudaStream_t stream) {
  LGB_REQUIRE(x && gamma && beta && y && mean && rstd, kErrInvalid, "ln_gelu_fwd: null pointer");
  LGB_REQUIRE(ntok > 0, kErrInvalid, "ln_gelu_fwd: empty input");
  LGB_REQUIRE(aligned16({x, gamma, beta, y}), kErrInvalid, "ln_gelu_fwd: misaligned pointer (16 bytes needed)");
  if (dtype == LGB200_F32) return ln_gelu_fwd_dispatch<float>(x, gamma, beta, y, mean, rstd, ntok, W, eps, stream);
  if (dtype == LGB200_BF16) return ln_gelu_fwd_dispatch<__nv_bfloat16>(x, gamma, beta, y, mean, rstd, ntok, W, eps, stream);
  LGB_REQUIRE(false, kErrInvalid, "ln_gelu_fwd: bad dtype %d", dtype);
}

int lgb200_ln_gelu_bwd_parts(int64_t ntok) {
  int64_t p = (ntok + 7) / 8;
  return (int)(p < 264 ? p : 264);  // 2 resident CTAs per SM x 132 SMs of an H100 SXM (3 per SM spills)
}

}  // extern "C"

template <typename T>
static int ln_gelu_bwd_dispatch(const void* dy, const void* x, const float* gamma, const float* beta,
                                const float* mean, const float* rstd, void* dx, float* dgp, float* dbp, float* dxp,
                                int64_t ntok, int W, cudaStream_t stream) {
  const unsigned grid = (unsigned)lgb200_ln_gelu_bwd_parts(ntok);
  switch (W) {
    case 256: ln_gelu_bwd_kernel<T, 1><<<grid, 256, 0, stream>>>((const T*)dy, (const T*)x, gamma, beta, mean, rstd, (T*)dx, dgp, dbp, dxp, ntok); break;
    case 512: ln_gelu_bwd_kernel<T, 2><<<grid, 256, 0, stream>>>((const T*)dy, (const T*)x, gamma, beta, mean, rstd, (T*)dx, dgp, dbp, dxp, ntok); break;
    case 1024: ln_gelu_bwd_kernel<T, 4><<<grid, 256, 0, stream>>>((const T*)dy, (const T*)x, gamma, beta, mean, rstd, (T*)dx, dgp, dbp, dxp, ntok); break;
    default: LGB_REQUIRE(false, kErrUnsupported, "ln_gelu: width %d not in {256,512,1024}", W);
  }
  return check_launch("ln_gelu_bwd");
}

extern "C" {

int lgb200_ln_gelu_bwd(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                       const float* rstd, void* dx, float* dgamma_part, float* dbeta_part, float* dxsum_part,
                       int64_t ntok, int W, int dtype, cudaStream_t stream) {
  LGB_REQUIRE(dy && x && gamma && beta && mean && rstd && dx && dgamma_part && dbeta_part && dxsum_part, kErrInvalid,
              "ln_gelu_bwd: null pointer");
  LGB_REQUIRE(ntok > 0, kErrInvalid, "ln_gelu_bwd: empty input");
  LGB_REQUIRE(aligned16({dy, x, gamma, beta, dx}), kErrInvalid, "ln_gelu_bwd: misaligned pointer (16 bytes needed)");
  if (dtype == LGB200_F32)
    return ln_gelu_bwd_dispatch<float>(dy, x, gamma, beta, mean, rstd, dx, dgamma_part, dbeta_part, dxsum_part, ntok, W,
                                       stream);
  if (dtype == LGB200_BF16)
    return ln_gelu_bwd_dispatch<__nv_bfloat16>(dy, x, gamma, beta, mean, rstd, dx, dgamma_part, dbeta_part, dxsum_part,
                                               ntok, W, stream);
  LGB_REQUIRE(false, kErrInvalid, "ln_gelu_bwd: bad dtype %d", dtype);
}

int lgb200_adam_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_scale_per_elem, float lr,
                     float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                     float grad_scale, const float* lr_dev, const float* loss_scale_dev, const float* found_inf_dev,
                     cudaStream_t stream) {
  LGB_REQUIRE(p && g && m && v, kErrInvalid, "adam_flat: null pointer");
  LGB_REQUIRE(n > 0 && (step >= 1 || step_dev), kErrInvalid, "adam_flat: bad n/step");
  LGB_REQUIRE((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
               reinterpret_cast<uintptr_t>(v)) % 16 == 0,
              kErrInvalid, "adam_flat: buffers must be 16-byte aligned");
  const float bc1 = step >= 1 ? 1.f - powf(beta1, (float)step) : 1.f;
  const float bc2s = step >= 1 ? sqrtf(1.f - powf(beta2, (float)step)) : 1.f;
  const AdamRule rule{beta1, beta2, eps, weight_decay, bc1, bc2s};
  flat_update_kernel<<<flat_update_grid(n), 256, 0, stream>>>(p, g, m, v, nullptr, n, lr_scale_per_elem, lr, grad_scale,
                                                              rule, AdamDev{step_dev, lr_dev, loss_scale_dev,
                                                                            found_inf_dev});
  return check_launch("adam_flat");
}

int lgb200_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_scale_per_elem,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                      float grad_scale, const float* lr_dev, const float* loss_scale_dev, const float* found_inf_dev,
                      cudaStream_t stream) {
  LGB_REQUIRE(p && g && m && v, kErrInvalid, "adamw_flat: null pointer");
  LGB_REQUIRE(n > 0 && (step >= 1 || step_dev), kErrInvalid, "adamw_flat: bad n/step");
  LGB_REQUIRE(aligned16({p, g, m, v}), kErrInvalid, "adamw_flat: buffers must be 16-byte aligned");
  AdamWRule rule;
  rule.beta1 = beta1, rule.beta2 = beta2, rule.eps = eps, rule.wd = weight_decay;
  rule.bc1 = step >= 1 ? 1.f - powf(beta1, (float)step) : 1.f;
  rule.bc2_sqrt = step >= 1 ? sqrtf(1.f - powf(beta2, (float)step)) : 1.f;
  flat_update_kernel<<<flat_update_grid(n), 256, 0, stream>>>(p, g, m, v, nullptr, n, lr_scale_per_elem, lr, grad_scale,
                                                              rule, AdamDev{step_dev, lr_dev, loss_scale_dev,
                                                                            found_inf_dev});
  return check_launch("adamw_flat");
}

int lgb200_sgd_flat(float* p, const float* g, float* momentum_buffer, int64_t n, const float* lr_scale_per_elem,
                    float lr, float momentum, float dampening, int nesterov, float weight_decay, int step,
                    const int* step_dev, float grad_scale, const float* lr_dev, const float* loss_scale_dev,
                    const float* found_inf_dev, cudaStream_t stream) {
  LGB_REQUIRE(p && g, kErrInvalid, "sgd_flat: null pointer");
  LGB_REQUIRE((momentum != 0.f) == (momentum_buffer != nullptr), kErrInvalid,
              "sgd_flat: momentum_buffer must be given exactly when momentum != 0");
  LGB_REQUIRE(!nesterov || (momentum > 0.f && dampening == 0.f), kErrInvalid,
              "sgd_flat: nesterov needs momentum > 0 and zero dampening");
  LGB_REQUIRE(n > 0 && (step >= 1 || step_dev), kErrInvalid, "sgd_flat: bad n/step");
  LGB_REQUIRE(aligned16({p, g, momentum_buffer}), kErrInvalid, "sgd_flat: buffers must be 16-byte aligned");
  const SgdRule rule{momentum, dampening, weight_decay, nesterov, step};
  flat_update_kernel<<<flat_update_grid(n), 256, 0, stream>>>(p, g, momentum_buffer, nullptr, nullptr, n,
                                                              lr_scale_per_elem, lr, grad_scale, rule,
                                                              AdamDev{step_dev, lr_dev, loss_scale_dev, found_inf_dev});
  return check_launch("sgd_flat");
}

int lgb200_rmsprop_flat(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg,
                        int64_t n, const float* lr_scale_per_elem, float lr, float alpha, float eps,
                        float weight_decay, float momentum, float grad_scale, const float* lr_dev,
                        const float* loss_scale_dev, const float* found_inf_dev, cudaStream_t stream) {
  LGB_REQUIRE(p && g && square_avg, kErrInvalid, "rmsprop_flat: null pointer");
  LGB_REQUIRE((momentum > 0.f) == (momentum_buffer != nullptr), kErrInvalid,
              "rmsprop_flat: momentum_buffer must be given exactly when momentum > 0");
  LGB_REQUIRE(n > 0, kErrInvalid, "rmsprop_flat: bad n");
  LGB_REQUIRE(aligned16({p, g, square_avg, momentum_buffer, grad_avg}), kErrInvalid,
              "rmsprop_flat: buffers must be 16-byte aligned");
  const RmspropRule rule{alpha, eps, weight_decay, momentum, grad_avg != nullptr};
  flat_update_kernel<<<flat_update_grid(n), 256, 0, stream>>>(p, g, square_avg, momentum_buffer, grad_avg, n,
                                                              lr_scale_per_elem, lr, grad_scale, rule,
                                                              AdamDev{nullptr, lr_dev, loss_scale_dev, found_inf_dev});
  return check_launch("rmsprop_flat");
}

int lgb200_flat_grad_check(const float* g, int64_t n, float* found_inf, cudaStream_t stream) {
  LGB_REQUIRE(g && found_inf && n > 0, kErrInvalid, "flat_grad_check: bad arguments");
  LGB_REQUIRE(reinterpret_cast<uintptr_t>(g) % 16 == 0, kErrInvalid, "flat_grad_check: g must be 16-byte aligned");
  cudaError_t e = cudaMemsetAsync(found_inf, 0, sizeof(float), stream);
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "flat_grad_check: memset: %s", cudaGetErrorString(e));
  int64_t blocks = (n / 4 + 255) / 256;
  const unsigned grid = (unsigned)(blocks < 1 ? 1 : (blocks > 1184 ? 1184 : blocks));
  grad_check_kernel<<<grid, 256, 0, stream>>>(g, n, found_inf);
  return check_launch("flat_grad_check");
}

}  // extern "C"

static unsigned grad_norm_ctas(int64_t n_norm) {
  const int64_t b = (n_norm / 4 + 2 * kNormThreads - 1) / (2 * kNormThreads);
  return (unsigned)(b < 1 ? 1 : (b > kNormMaxCtas ? kNormMaxCtas : b));
}

extern "C" {

size_t lgb200_flat_grad_norm_ws_bytes(int64_t n_norm) { return grad_norm_ctas(n_norm) * sizeof(double); }

int lgb200_flat_grad_norm(const float* g, int64_t n_norm, int64_t n_check, float grad_scale,
                          const float* loss_scale_dev, float max_norm, float* found_inf, float* norm_out,
                          float* adam_div_out, void* ws, cudaStream_t stream) {
  LGB_REQUIRE(g && found_inf && norm_out && adam_div_out && ws, kErrInvalid, "flat_grad_norm: null pointer");
  LGB_REQUIRE(n_norm > 0 && n_check >= n_norm, kErrInvalid, "flat_grad_norm: need 0 < n_norm <= n_check");
  LGB_REQUIRE(grad_scale > 0.f && max_norm > 0.f, kErrInvalid, "flat_grad_norm: grad_scale and max_norm must be > 0");
  LGB_REQUIRE(aligned16({g, ws}), kErrInvalid, "flat_grad_norm: g and ws must be 16-byte aligned");
  const unsigned grid = grad_norm_ctas(n_norm);
  grad_sumsq_kernel<<<grid, kNormThreads, 0, stream>>>(g, n_norm, n_check, (double*)ws);
  grad_norm_finish_kernel<<<1, kNormThreads, 0, stream>>>((const double*)ws, (int)grid, grad_scale, loss_scale_dev,
                                                          max_norm, found_inf, norm_out, adam_div_out);
  return check_launch("flat_grad_norm");
}

int lgb200_amp_update(const float* found_inf, int* step_dev, float* loss_scale, int* growth_tracker,
                      float growth_factor, float backoff_factor, int growth_interval, cudaStream_t stream) {
  LGB_REQUIRE(found_inf, kErrInvalid, "amp_update: null found_inf");
  amp_update_kernel<<<1, 1, 0, stream>>>(found_inf, step_dev, loss_scale, growth_tracker, growth_factor,
                                         backoff_factor, growth_interval);
  return check_launch("amp_update");
}

int lgb200_cast_bf16(const float* src, void* dst, int64_t n, cudaStream_t stream) {
  LGB_REQUIRE(src && dst && n > 0, kErrInvalid, "cast_bf16: bad arguments");
  LGB_REQUIRE(aligned16({src, dst}), kErrInvalid, "cast_bf16: misaligned pointer (16 bytes needed)");
  const unsigned grid = (unsigned)(((n + 7) / 8 + 255) / 256);
  cast_bf16_kernel<<<grid, 256, 0, stream>>>(src, (__nv_bfloat16*)dst, n);
  return check_launch("cast_bf16");
}

int lgb200_head_token_bwd_ws_floats(int D) { return kHeadBwdParts * (2 * D + 2); }

int lgb200_head_token_fwd(const float* x, const float* wm, const float* bm, const float* wt, const float* bt,
                          void* x_cast, float* zt, float* ls, float* du, int64_t ntok, int D, int dtype,
                          cudaStream_t stream) {
  LGB_REQUIRE(x && wm && bm && zt && ls && du && ntok > 0, kErrInvalid, "head_token_fwd: bad arguments");
  LGB_REQUIRE((wt == nullptr) == (bt == nullptr), kErrInvalid, "head_token_fwd: wt/bt must both be set or null");
  LGB_REQUIRE(D % 8 == 0 && D > 0 && D <= 512, kErrUnsupported, "head_token_fwd: D=%d not a multiple of 8 in (0,512]", D);
  int64_t g = (ntok + 7) / 8;
  const unsigned grid = (unsigned)(g < 1184 ? g : 1184);
#define LGB_HT_FWD(T, NCH) \
  head_token_fwd_kernel<T, NCH><<<grid, 256, 0, stream>>>(x, wm, bm, wt, bt, (T*)x_cast, zt, ls, du, ntok, D)
  if (dtype == LGB200_F32) { if (D <= 256) LGB_HT_FWD(float, 1); else LGB_HT_FWD(float, 2); }
  else if (dtype == LGB200_BF16) { if (D <= 256) LGB_HT_FWD(__nv_bfloat16, 1); else LGB_HT_FWD(__nv_bfloat16, 2); }
  else LGB_REQUIRE(false, kErrInvalid, "head_token_fwd: bad dtype %d", dtype);
#undef LGB_HT_FWD
  return check_launch("head_token_fwd");
}

int lgb200_head_token_bwd(const float* x, const void* dmdw, const float* dzt, const float* wm, float* dx, float* dW2,
                          float* db2, float* ws, unsigned* counter, int64_t ntok, int D, int dtype,
                          cudaStream_t stream) {
  LGB_REQUIRE(x && dzt && wm && dW2 && db2 && ws && counter && ntok > 0 && (dmdw == nullptr) == (dx == nullptr),
              kErrInvalid, "head_token_bwd: bad arguments");
  LGB_REQUIRE(D % 8 == 0 && D > 0 && D <= 512, kErrUnsupported, "head_token_bwd: D=%d not a multiple of 8 in (0,512]", D);
#define LGB_HT_BWD(T, NCH)                                                                                     \
  head_token_bwd_kernel<T, NCH><<<kHeadBwdParts, 256, 0, stream>>>(x, (const T*)dmdw, dzt, wm, dx, dW2, db2, ws, \
                                                                   counter, ntok, D)
  if (dtype == LGB200_F32) { if (D <= 256) LGB_HT_BWD(float, 1); else LGB_HT_BWD(float, 2); }
  else if (dtype == LGB200_BF16) { if (D <= 256) LGB_HT_BWD(__nv_bfloat16, 1); else LGB_HT_BWD(__nv_bfloat16, 2); }
  else LGB_REQUIRE(false, kErrInvalid, "head_token_bwd: bad dtype %d", dtype);
#undef LGB_HT_BWD
  return check_launch("head_token_bwd");
}

}  // extern "C"

namespace lgb {

// ---------------------------------------------------------------------------------------------
// LightGlue's adaptive depth / width on a batch of pairs (lightglue.py:461-526, 545-576), one layer's step.
// The tokens of pair b are two segments of the packed [T, D] state: image 0 is segment 2b, image 1 segment 2b + 1,
// described by seg [4][2B] = (offset, length, partner's offset, partner's length).
//   decide (one CTA per pair): a pair with tokens left stops when 1 - #(token confidence < thr) / (M + N) exceeds
//     depth_conf (or always, on the last layer); a stopped pair's tokens move, unpruned, to the pair's block of the
//     final buffer (b (M + N), image 1 at + M).  Otherwise a token stays when its matchability > width_thr or, with
//     early stopping on, its confidence is still <= thr; a block scan per segment gives each kept token its place,
//     and its prune counter (original keypoint index ind[t]) goes up by one.  The sigmoids are 1 / (1 + exp(-z)) in
//     fp32, as torch.sigmoid computes them, so every decision is the one the one-pair loop made.
//   gather (grid-stride, one warp per token row): every CTA scans the kept counts into the new segment offsets
//     (pair-major: pair 0 image 0, pair 0 image 1, pair 1 image 0, ...) and copies x, theta and ind of its rows; CTA 0
//     writes the new seg and status = (kept tokens, 1 if a continuing pair kept no token of a view).
// ---------------------------------------------------------------------------------------------
constexpr int kAcThreads = 1024;

__device__ __forceinline__ float sigmoid_f32(float z) { return 1.f / (1.f + expf(-z)); }

// exclusive prefix sum over the CTA (every thread calls it); *total = the sum over the CTA
__device__ __forceinline__ int block_exclusive_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nw ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    sh[lane] = w;
  }
  __syncthreads();
  const int r = (warp ? sh[warp - 1] : 0) + x - v;
  *total = sh[nw - 1];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kAcThreads)
    adaptive_decide_kernel(const int* __restrict__ ind, const float* __restrict__ zt, const int* __restrict__ seg,
                           int* __restrict__ fin_len, int* __restrict__ stop_layer, int64_t* __restrict__ prune0,
                           int64_t* __restrict__ prune1, int* __restrict__ dst_seg, int* __restrict__ dst_pos,
                           int* __restrict__ cnt, int* __restrict__ state, const float* __restrict__ conf_thr,
                           float depth_conf, float width_thr, int do_stop, int do_prune, int layer, int finish, int B,
                           int M, int N, const int* __restrict__ pair_pts) {
  __shared__ int sh[32];
  __shared__ int s_low;
  const int b = blockIdx.x, S = 2 * B;
  const int off0 = seg[2 * b], off1 = seg[2 * b + 1], n0 = seg[S + 2 * b], n1 = seg[S + 2 * b + 1];
  if (n0 == 0 && n1 == 0) {  // stopped at an earlier layer
    if (threadIdx.x == 0) {
      cnt[2 * b] = cnt[2 * b + 1] = 0;
      state[b] = 0;
    }
    return;
  }
  const bool conf = do_stop && !finish;
  const float thr = conf ? *conf_thr : 0.f;
  bool stop = finish;
  if (conf) {
    if (threadIdx.x == 0) s_low = 0;
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < n0 + n1; i += blockDim.x) {
      const int t = i < n0 ? off0 + i : off1 + i - n0;
      c += sigmoid_f32(zt[2 * t + 1]) < thr;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_low, c);
    __syncthreads();
    // relative to the pair's ORIGINAL point count (lightglue.py:489), in fp32 as the one-pair loop computes it
    stop = 1.f - (float)s_low / (float)(pair_pts ? pair_pts[b] : M + N) > depth_conf;
  }
  if (stop) {
    for (int i = threadIdx.x; i < n0 + n1; i += blockDim.x) {
      const int t = i < n0 ? off0 + i : off1 + i - n0;
      dst_seg[t] = -2;
      dst_pos[t] = b * (M + N) + (i < n0 ? i : M + i - n0);
    }
    if (threadIdx.x == 0) {
      fin_len[2 * b] = n0;
      fin_len[2 * b + 1] = n1;
      stop_layer[b] = layer;
      cnt[2 * b] = cnt[2 * b + 1] = 0;
      state[b] = 0;
    }
    return;
  }
  for (int img = 0; img < 2; ++img) {
    const int off = img ? off1 : off0, n = img ? n1 : n0;
    int64_t* prune = img ? prune1 + (int64_t)b * N : prune0 + (int64_t)b * M;
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += blockDim.x) {  // uniform trip count: every thread reaches the scan's barriers
      const int i = c0 + threadIdx.x;
      bool keep = i < n;
      if (keep && do_prune) {
        const int t = off + i;
        // low-confidence points are never pruned (lightglue.py:556-557)
        keep = sigmoid_f32(zt[2 * t]) > width_thr || (do_stop && sigmoid_f32(zt[2 * t + 1]) <= thr);
      }
      int tot;
      const int p = block_exclusive_scan(keep ? 1 : 0, sh, &tot);
      if (i < n) {
        const int t = off + i;
        dst_seg[t] = keep ? 2 * b + img : -1;
        dst_pos[t] = base + p;
        if (keep && do_prune) prune[ind[t]] += 1;
      }
      base += tot;
    }
    if (threadIdx.x == 0) cnt[2 * b + img] = base;
  }
  if (threadIdx.x == 0) state[b] = 1;
}

__global__ void __launch_bounds__(256)
    adaptive_gather_kernel(const float* __restrict__ x, const float* __restrict__ theta, const int* __restrict__ ind,
                           const int* __restrict__ dst_seg, const int* __restrict__ dst_pos,
                           const int* __restrict__ cnt, const int* __restrict__ state, float* __restrict__ x_out,
                           float* __restrict__ theta_out, int* __restrict__ ind_out, float* __restrict__ x_fin,
                           int* __restrict__ ind_fin, int* __restrict__ seg_out, int* __restrict__ status, int B, int T,
                           int D, int R) {
  extern __shared__ int s_off[];  // [2B] offsets of the new segments
  __shared__ int sh[32];
  const int S = 2 * B;
  {
    const int per = (S + blockDim.x - 1) / blockDim.x, s0 = threadIdx.x * per;
    int loc = 0;
    for (int s = s0; s < s0 + per && s < S; ++s) loc += cnt[s];
    int tot;
    int run = block_exclusive_scan(loc, sh, &tot);
    for (int s = s0; s < s0 + per && s < S; ++s) {
      s_off[s] = run;
      run += cnt[s];
    }
    __syncthreads();
    if (blockIdx.x == 0) {
      for (int s = threadIdx.x; s < S; s += blockDim.x) {
        seg_out[s] = s_off[s];
        seg_out[S + s] = cnt[s];
        seg_out[2 * S + s] = s_off[s ^ 1];
        seg_out[3 * S + s] = cnt[s ^ 1];
      }
      bool emptied = false;
      for (int b = threadIdx.x; b < B; b += blockDim.x) emptied |= state[b] && (cnt[2 * b] == 0 || cnt[2 * b + 1] == 0);
      emptied = __syncthreads_or(emptied);
      if (threadIdx.x == 0) {
        status[0] = tot;
        status[1] = emptied ? 1 : 0;
      }
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < T; t += (int64_t)gridDim.x * 8) {
    const int sg = dst_seg[t];
    if (sg == -1) continue;  // pruned
    const bool fin = sg == -2;
    const int64_t dst = fin ? (int64_t)dst_pos[t] : (int64_t)s_off[sg] + dst_pos[t];
    const float4* src = reinterpret_cast<const float4*>(x + t * D);
    float4* dx = reinterpret_cast<float4*>((fin ? x_fin : x_out) + dst * D);
    for (int c = lane; c < D / 4; c += 32) dx[c] = src[c];
    if (!fin)
      for (int c = lane; c < R; c += 32) theta_out[dst * R + c] = theta[t * R + c];
    if (lane == 0) (fin ? ind_fin : ind_out)[dst] = ind[t];
  }
}

}  // namespace lgb

extern "C" {

int64_t lgb200_adaptive_compact_ws_ints(int T, int B) { return 2 * (int64_t)T + 3 * (int64_t)B; }

int lgb200_adaptive_compact_varlen(const float* x, const float* theta, const int* ind, const float* zt, const int* seg,
                                   float* x_out, float* theta_out, int* ind_out, int* seg_out, float* x_fin,
                                   int* ind_fin, int* fin_len, int* stop_layer, int64_t* prune0, int64_t* prune1,
                                   int* status, int* ws, const float* conf_thr, const int* pair_pts, float depth_conf,
                                   float width_thr, int do_stop, int do_prune, int layer, int finish, int B, int M,
                                   int N, int T, int D, int R, cudaStream_t stream) {
  LGB_REQUIRE(x && theta && ind && seg && x_out && theta_out && ind_out && seg_out && x_fin && ind_fin && fin_len &&
                  stop_layer && prune0 && prune1 && status && ws,
              kErrInvalid, "adaptive_compact: null pointer");
  LGB_REQUIRE(finish || ((zt != nullptr) && (!do_stop || conf_thr != nullptr)), kErrInvalid,
              "adaptive_compact: the stop / prune decisions need zt (and conf_thr with early stopping)");
  LGB_REQUIRE(B > 0 && B <= 4096 && M > 0 && N > 0 && T > 0 && (int64_t)T <= (int64_t)B * (M + N), kErrInvalid,
              "adaptive_compact: bad extents B=%d M=%d N=%d T=%d", B, M, N, T);
  LGB_REQUIRE(D > 0 && D % 4 == 0 && R > 0 && aligned16({x, x_out, x_fin}), kErrInvalid,
              "adaptive_compact: D=%d must be a multiple of 4 and x / x_out / x_fin 16-byte aligned", D);
  int* dst_seg = ws;
  int* dst_pos = ws + T;
  int* cnt = ws + 2 * (int64_t)T;
  int* state = cnt + 2 * B;
  adaptive_decide_kernel<<<B, kAcThreads, 0, stream>>>(ind, zt, seg, fin_len, stop_layer, prune0, prune1, dst_seg,
                                                       dst_pos, cnt, state, conf_thr, depth_conf, width_thr, do_stop,
                                                       do_prune, layer, finish, B, M, N, pair_pts);
  int rc = check_launch("adaptive_decide");
  if (rc) return rc;
  const int64_t rows = ((int64_t)T + 7) / 8, cap = 4 * (int64_t)device_sm_count();
  adaptive_gather_kernel<<<(unsigned)(rows < cap ? rows : cap), 256, 2 * B * sizeof(int), stream>>>(
      x, theta, ind, dst_seg, dst_pos, cnt, state, x_out, theta_out, ind_out, x_fin, ind_fin, seg_out, status, B, T, D,
      R);
  return check_launch("adaptive_gather");
}

int lgb200_adaptive_compact(const float* x, const float* theta, const int* ind, const float* zt, const int* seg,
                            float* x_out, float* theta_out, int* ind_out, int* seg_out, float* x_fin, int* ind_fin,
                            int* fin_len, int* stop_layer, int64_t* prune0, int64_t* prune1, int* status, int* ws,
                            const float* conf_thr, float depth_conf, float width_thr, int do_stop, int do_prune,
                            int layer, int finish, int B, int M, int N, int T, int D, int R, cudaStream_t stream) {
  return lgb200_adaptive_compact_varlen(x, theta, ind, zt, seg, x_out, theta_out, ind_out, seg_out, x_fin, ind_fin,
                                        fin_len, stop_layer, prune0, prune1, status, ws, conf_thr, nullptr, depth_conf,
                                        width_thr, do_stop, do_prune, layer, finish, B, M, N, T, D, R, stream);
}

}  // extern "C"

