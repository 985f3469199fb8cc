// The two other assignment heads on the matcher path:
//   * log_double_softmax with a learned bin score (GlueStick, gluestick.py:772-783)
//   * log-domain Sinkhorn optimal transport with a dustbin (SuperGlue head,
//     gluefactory_nonfree/superglue.py:186-214): one persistent kernel for the iterations, one for their reverse sweep.
// Both are HBM/L2-bound sweeps over the [B,M,N] similarity; the bordered (M+1)x(N+1) coupling
// matrix is never materialised: the dustbin row/column is handled analytically.
#include <math.h>

#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

constexpr float kNInf = -INFINITY;

__device__ __forceinline__ float logaddexp_f(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == kNInf) return kNInf;
  return m + log1pf(expf(-fabsf(a - b)));
}

// scores from precomputed lse_row / lse_col of the UNBORDERED sim
__global__ void __launch_bounds__(256) lds_scores_kernel(const float* __restrict__ sim, const float* __restrict__ lse_row,
                                                        const float* __restrict__ lse_col, float beta,
                                                        const float* __restrict__ beta_dev,
                                                        float* __restrict__ scores, int M, int N) {
  if (beta_dev) beta = __ldg(beta_dev);  // the learnt bin score read from device memory (no host read-back)
  const int b = blockIdx.y;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i > M) return;
  float* orow = scores + ((int64_t)b * (M + 1) + i) * (N + 1);
  if (i == M) {
    for (int j = lane; j <= N; j += 32)
      orow[j] = j < N ? beta - logaddexp_f(lse_col[(int64_t)b * N + j], beta) : 0.f;
    return;
  }
  const float lr = logaddexp_f(lse_row[(int64_t)b * M + i], beta);
  const float* srow = sim + ((int64_t)b * M + i) * N;
  for (int j = lane; j < N; j += 32) {
    const float x = srow[j];
    const float lc = logaddexp_f(lse_col[(int64_t)b * N + j], beta);
    orow[j] = ((x - lr) + (x - lc)) * 0.5f;
  }
  if (lane == 0) orow[N] = beta - lr;
}

// ---- Sinkhorn -------------------------------------------------------------------------------------
// One persistent cooperative kernel runs all iterations (superglue.py:186-196); a second one runs the reverse sweep
// of the same iterations for the gradient.  Work item = (pair b, strip s of R consecutive rows); the CTA that owns a
// strip keeps its rows of Z in shared memory for the whole kernel when the launch has one item per CTA and the strip
// fits (B=1, N=2048: 14 rows x 8 KB), so an iteration touches HBM/L2 only for the O(M+N) potentials and the
// S x (N+1) column partials.  Two grid barriers per iteration (row phase -> column merge -> next row phase).
//   row phase    u_i = log_mu_i - LSE_j (Z_ij + v_j)   (warp per row), then, with the strip's own fresh u,
//                per-strip column partials (max, sum) of Z_ij + u_i      (thread per column)
//   merge phase  v_j = log_nu_j - LSE over the S partials and the dustbin row  (warp per column)
// The dustbin row (i = M) belongs to the last strip; the dustbin column (j = N) is an ordinary column whose Z is alpha.
struct SkGeom {
  int B, M, N, S, R, C;   // S strips per pair, R rows per strip, C columns per merge slice
  int cached;             // 1: the strip's R x N block of sim lives in shared memory
};

__device__ __forceinline__ void sk_grid_barrier(unsigned* ctr, unsigned& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(ctr, 1u);
    unsigned seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctr) : "memory");
    } while (seen < target);
  }
  __syncthreads();
}

__device__ __forceinline__ void lse4(float& m, float& s, float x0, float x1, float x2, float x3) {
  const float mn = fmaxf(fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)), m);
  s = s * __expf(m - mn) + (__expf(x0 - mn) + __expf(x1 - mn)) + (__expf(x2 - mn) + __expf(x3 - mn));
  m = mn;
}
__device__ __forceinline__ void lse1(float& m, float& s, float x) {
  const float mn = fmaxf(m, x);
  s = s * __expf(m - mn) + __expf(x - mn);
  m = mn;
}
__device__ __forceinline__ void lse_warp(float& m, float& s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mn = fmaxf(m, m2);
    s = (mn == kNInf) ? 0.f : s * __expf(m - mn) + s2 * __expf(m2 - mn);
    m = mn;
  }
}

constexpr int kSkThreads = 1024;
__host__ __device__ inline int sk_pad(int n) { return (n + 3) & ~3; }

// fill the strip cache: rows [i0, i1) of pair b
__device__ __forceinline__ void sk_fill_cache(float* zs, const float* __restrict__ sim, int b, int i0, int i1, int M,
                                              int N) {
  const float* src = sim + ((int64_t)b * M + i0) * N;
  const int n = (i1 - i0) * N;
  for (int e = threadIdx.x; e < n; e += kSkThreads) zs[e] = __ldg(src + e);
}

__global__ void __launch_bounds__(kSkThreads, 1)
sk_fwd_persistent_kernel(const float* __restrict__ sim, float alpha, const float* __restrict__ alpha_dev, int iters,
                         float* __restrict__ out, float* __restrict__ u, float* __restrict__ v, float* __restrict__ uh, float* __restrict__ vh,
                         float* __restrict__ pm, float* __restrict__ ps, unsigned* __restrict__ bar, SkGeom g) {
  extern __shared__ float sk_smem[];
  const int M = g.M, N = g.N, S = g.S, R = g.R, B = g.B;
  float* vsm = sk_smem;                 // N + 1
  float* usm = vsm + sk_pad(N + 1);     // R + 1
  float* zs = usm + sk_pad(R + 1);      // R x N when cached
  if (alpha_dev) alpha = __ldg(alpha_dev);  // the learnt bin score read from device memory (no host read-back)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int items = B * S;
  const float norm = -logf((float)(M + N));
  unsigned target = 0;
  if (g.cached) {
    const int b = blockIdx.x / S, s = blockIdx.x % S;
    sk_fill_cache(zs, sim, b, s * R, min(M, s * R + R), M, N);
    __syncthreads();
  }
  for (int it = 0; it < iters; ++it) {
    // ---- row phase
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int b = w / S, s = w % S, i0 = s * R, i1 = min(M, i0 + R);
      const int nrows = i1 - i0 + (s == S - 1 ? 1 : 0);
      for (int j = tid; j <= N; j += kSkThreads) vsm[j] = it ? __ldcg(v + (int64_t)b * (N + 1) + j) : 0.f;
      __syncthreads();
      for (int r = warp; r < nrows; r += 32) {
        const int i = i0 + r;
        float m = kNInf, sm = 0.f;
        if (i < M) {
          const float* row = g.cached ? zs + r * N : sim + ((int64_t)b * M + i) * N;
          int j = lane;
          for (; j + 224 < N; j += 256) {  // eight loads in flight per lane
            float x[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = row[j + 32 * e];
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] += vsm[j + 32 * e];
            lse4(m, sm, x[0], x[1], x[2], x[3]);
            lse4(m, sm, x[4], x[5], x[6], x[7]);
          }
          for (; j + 96 < N; j += 128)
            lse4(m, sm, row[j] + vsm[j], row[j + 32] + vsm[j + 32], row[j + 64] + vsm[j + 64], row[j + 96] + vsm[j + 96]);
          for (; j < N; j += 32) lse1(m, sm, row[j] + vsm[j]);
        } else {
          for (int j = lane; j < N; j += 32) lse1(m, sm, alpha + vsm[j]);
        }
        lse_warp(m, sm);
        if (lane == 0) {
          lse1(m, sm, alpha + vsm[N]);
          const float ui = (i < M ? norm : logf((float)N) + norm) - (m + logf(sm));
          usm[r] = ui;
          u[(int64_t)b * (M + 1) + i] = ui;
          if (uh) uh[((int64_t)it * B + b) * (M + 1) + i] = ui;
        }
      }
      __syncthreads();
      // column partials over the strip's dense rows (the dustbin row is added in the merge)
      for (int j = tid; j <= N; j += kSkThreads) {
        float m = kNInf, sm = 0.f;
        if (j < N) {
          const float* col = g.cached ? zs + j : sim + ((int64_t)b * M + i0) * N + j;
          int r = 0;
          for (; r + 7 < i1 - i0; r += 8) {
            float x[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = col[(int64_t)(r + e) * N];
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] += usm[r + e];
            lse4(m, sm, x[0], x[1], x[2], x[3]);
            lse4(m, sm, x[4], x[5], x[6], x[7]);
          }
          for (; r + 3 < i1 - i0; r += 4)
            lse4(m, sm, col[(int64_t)r * N] + usm[r], col[(int64_t)(r + 1) * N] + usm[r + 1],
                 col[(int64_t)(r + 2) * N] + usm[r + 2], col[(int64_t)(r + 3) * N] + usm[r + 3]);
          for (; r < i1 - i0; ++r) lse1(m, sm, col[(int64_t)r * N] + usm[r]);
        } else {
          for (int r = 0; r < i1 - i0; ++r) lse1(m, sm, alpha + usm[r]);
        }
        pm[(int64_t)w * (N + 1) + j] = m;
        ps[(int64_t)w * (N + 1) + j] = sm;
      }
      __syncthreads();
    }
    sk_grid_barrier(bar, target);
    // ---- merge phase: warp per column of the item's slice
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int b = w / S, s = w % S, j0 = s * g.C, j1 = min(N + 1, j0 + g.C);
      const float ubin = alpha + __ldcg(u + (int64_t)b * (M + 1) + M);
      for (int j = j0 + warp; j < j1; j += 32) {
        float m = kNInf, sm = 0.f;
        for (int p0 = 0; p0 < S; p0 += 128) {  // four partial pairs in flight per lane
          float m2[4], s2[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int p = p0 + e * 32 + lane;
            const int64_t o = ((int64_t)b * S + (p < S ? p : 0)) * (N + 1) + j;
            m2[e] = p < S ? __ldcg(pm + o) : kNInf;
            s2[e] = p < S ? __ldcg(ps + o) : 0.f;
          }
          const float mn = fmaxf(fmaxf(fmaxf(m2[0], m2[1]), fmaxf(m2[2], m2[3])), m);
          if (mn != kNInf) {
            sm = sm * __expf(m - mn);
#pragma unroll
            for (int e = 0; e < 4; ++e) sm += s2[e] * __expf(m2[e] - mn);
            m = mn;
          }
        }
        lse_warp(m, sm);
        if (lane == 0) {
          lse1(m, sm, ubin);
          const float vj = (j < N ? norm : logf((float)M) + norm) - (m + logf(sm));
          v[(int64_t)b * (N + 1) + j] = vj;
          if (vh) vh[((int64_t)it * B + b) * (N + 1) + j] = vj;
        }
      }
    }
    sk_grid_barrier(bar, target);
  }
  // ---- output: out = Z + u + v - norm
  if (!out) return;
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    const int b = w / S, s = w % S, i0 = s * R, i1 = min(M, i0 + R);
    const int nrows = i1 - i0 + (s == S - 1 ? 1 : 0);
    for (int j = tid; j <= N; j += kSkThreads) vsm[j] = iters ? __ldcg(v + (int64_t)b * (N + 1) + j) : 0.f;
    __syncthreads();
    for (int r = warp; r < nrows; r += 32) {
      const int i = i0 + r;
      const float ui = (iters ? __ldcg(u + (int64_t)b * (M + 1) + i) : 0.f) - norm;
      float* orow = out + ((int64_t)b * (M + 1) + i) * (N + 1);
      if (i < M) {
        const float* row = g.cached ? zs + r * N : sim + ((int64_t)b * M + i) * N;
        for (int j = lane; j < N; j += 32) orow[j] = row[j] + ui + vsm[j];
        if (lane == 0) orow[N] = alpha + ui + vsm[N];
      } else {
        for (int j = lane; j <= N; j += 32) orow[j] = alpha + ui + vsm[j];
      }
    }
    __syncthreads();
  }
}

// Reverse sweep (autograd of superglue.py:186-214 without its tape).  With the potentials u_k, v_k of the forward,
//   Q_k = exp(Z + u_k + v_k - log_nu) (columns sum to 1),  P_k = exp(Z + v_{k-1} + u_k - log_mu) (rows sum to 1):
//   for k = iters .. 1:  du = du0 - Q_k dv ;  dZ -= Q_k * dv + P_k * du ;  dv = -P_k^T du ;  du0 = 0
// starting from dZ = grad, du0 = rowsum(grad), dv = colsum(grad).  Row sums are local to the strip's owner, column
// sums go through per-strip partials and one merge, like the forward.  dZ lives in dsim [B,M,N] plus the dustbin
// row dzr [B,N+1] and column dzc [B,M]; every element is only ever touched by the same thread.
__global__ void __launch_bounds__(kSkThreads, 1)
sk_bwd_persistent_kernel(const float* __restrict__ sim, float alpha, const float* __restrict__ alpha_dev, int iters,
                         const float* __restrict__ grad,
                         const float* __restrict__ uh, const float* __restrict__ vh, float* __restrict__ dsim,
                         float* __restrict__ dzr, float* __restrict__ dzc, float* __restrict__ dv,
                         float* __restrict__ pw, unsigned* __restrict__ bar, SkGeom g) {
  extern __shared__ float sk_smem[];
  const int M = g.M, N = g.N, S = g.S, R = g.R, B = g.B;
  float* asm_ = sk_smem;                  // v_k - log_nu          N + 1
  float* vpm = asm_ + sk_pad(N + 1);      // v_{k-1}               N + 1
  float* dvs = vpm + sk_pad(N + 1);       // dv                    N + 1
  float* uks = dvs + sk_pad(N + 1);       // u_k                   R + 1
  float* dus = uks + sk_pad(R + 1);       // du                    R + 1
  float* zs = dus + sk_pad(R + 1);        // R x N when cached
  if (alpha_dev) alpha = __ldg(alpha_dev);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int items = B * S;
  const float norm = -logf((float)(M + N));
  unsigned target = 0;
  if (g.cached) {
    const int b = blockIdx.x / S, s = blockIdx.x % S;
    sk_fill_cache(zs, sim, b, s * R, min(M, s * R + R), M, N);
    __syncthreads();
  }
  // ---- dv = colsum(grad): per-strip partials, then merge
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    const int b = w / S, s = w % S, i0 = s * R, i1 = min(M, i0 + R);
    const int nrows = i1 - i0 + (s == S - 1 ? 1 : 0);
    for (int j = tid; j <= N; j += kSkThreads) {
      const float* col = grad + ((int64_t)b * (M + 1) + i0) * (N + 1) + j;
      float acc = 0.f;
      for (int r = 0; r < nrows; ++r) acc += __ldg(col + (int64_t)r * (N + 1));
      pw[(int64_t)w * (N + 1) + j] = acc;
    }
  }
  sk_grid_barrier(bar, target);
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    const int b = w / S, s = w % S, j0 = s * g.C, j1 = min(N + 1, j0 + g.C);
    for (int j = j0 + warp; j < j1; j += 32) {
      float acc = 0.f;
      for (int p0 = 0; p0 < S; p0 += 128) {
        float t[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int p = p0 + e * 32 + lane;
          t[e] = p < S ? __ldcg(pw + ((int64_t)b * S + p) * (N + 1) + j) : 0.f;
        }
        acc += (t[0] + t[1]) + (t[2] + t[3]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) dv[(int64_t)b * (N + 1) + j] = acc;
    }
  }
  sk_grid_barrier(bar, target);

  for (int k = iters - 1; k >= 0; --k) {
    const bool first = (k == iters - 1);
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int b = w / S, s = w % S, i0 = s * R, i1 = min(M, i0 + R);
      const int nd = i1 - i0, nrows = nd + (s == S - 1 ? 1 : 0);
      const float* vk = vh + ((int64_t)k * B + b) * (N + 1);
      const float* vp = vh + ((int64_t)(k - 1) * B + b) * (N + 1);
      for (int j = tid; j <= N; j += kSkThreads) {
        asm_[j] = __ldg(vk + j) - (j < N ? norm : logf((float)M) + norm);
        vpm[j] = k ? __ldg(vp + j) : 0.f;
        dvs[j] = __ldcg(dv + (int64_t)b * (N + 1) + j);
      }
      for (int r = tid; r < nrows; r += kSkThreads) uks[r] = __ldg(uh + ((int64_t)k * B + b) * (M + 1) + i0 + r);
      __syncthreads();
      // du_i = du0_i - sum_j Q_ij dv_j            (warp per row)
      for (int r = warp; r < nrows; r += 32) {
        const int i = i0 + r;
        const float ui = uks[r];
        float acc = 0.f, g0 = 0.f;
        if (i < M) {
          const float* row = g.cached ? zs + r * N : sim + ((int64_t)b * M + i) * N;
          for (int j = lane; j < N; j += 32) acc += __expf(row[j] + ui + asm_[j]) * dvs[j];
        } else {
          for (int j = lane; j < N; j += 32) acc += __expf(alpha + ui + asm_[j]) * dvs[j];
        }
        if (lane == 0) acc += __expf(alpha + ui + asm_[N]) * dvs[N];
        if (first) {
          const float* grow = grad + ((int64_t)b * (M + 1) + i) * (N + 1);
          for (int j = lane; j <= N; j += 32) g0 += __ldg(grow + j);
        }
        acc = g0 - acc;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) dus[r] = acc;
      }
      __syncthreads();
      // dZ -= Q dv + P du ; column partials of P du          (thread per column)
      for (int j = tid; j <= N; j += kSkThreads) {
        const float aj = asm_[j], vpj = vpm[j], dvj = dvs[j];
        float csum = 0.f;
        for (int r = 0; r < nrows; ++r) {
          const int i = i0 + r;
          const bool dense = (i < M) && (j < N);
          const float z = dense ? (g.cached ? zs[r * N + j] : __ldg(sim + ((int64_t)b * M + i) * N + j)) : alpha;
          float* dz = dense ? dsim + ((int64_t)b * M + i) * N + j
                            : (i == M ? dzr + (int64_t)b * (N + 1) + j : dzc + (int64_t)b * M + i);
          const float ui = uks[r];
          const float t = __expf(z + ui + aj) * dvj;
          const float lmu = i < M ? norm : logf((float)N) + norm;
          const float wv = __expf(z + vpj + (ui - lmu)) * dus[r];
          const float cur = first ? __ldg(grad + ((int64_t)b * (M + 1) + i) * (N + 1) + j) : *dz;
          *dz = cur - t - wv;
          csum += wv;
        }
        pw[(int64_t)w * (N + 1) + j] = csum;
      }
      __syncthreads();
    }
    sk_grid_barrier(bar, target);
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int b = w / S, s = w % S, j0 = s * g.C, j1 = min(N + 1, j0 + g.C);
      for (int j = j0 + warp; j < j1; j += 32) {
        float acc = 0.f;
        for (int p0 = 0; p0 < S; p0 += 128) {
          float t[4];
  #pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int p = p0 + e * 32 + lane;
            t[e] = p < S ? __ldcg(pw + ((int64_t)b * S + p) * (N + 1) + j) : 0.f;
          }
          acc += (t[0] + t[1]) + (t[2] + t[3]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) dv[(int64_t)b * (N + 1) + j] = -acc;
      }
    }
    sk_grid_barrier(bar, target);
  }
}

struct SkPlan {
  SkGeom g;
  int grid;
  size_t smem_fwd, smem_bwd;
};
// strips so that B * S covers the SMs once; the strip cache only when each CTA owns exactly one item and it fits
static SkPlan sk_plan(int B, int M, int N) {
  SkPlan p{};
  const int nsm = device_sm_count();
  int S = B >= nsm ? 1 : nsm / B;
  if (S > M) S = M;
  const int R = (M + S - 1) / S;
  S = (M + R - 1) / R;
  p.g = SkGeom{B, M, N, S, R, (N + 1 + S - 1) / S, 0};
  p.grid = B * S < nsm ? B * S : nsm;
  const size_t vec_f = (size_t)sk_pad(N + 1) + sk_pad(R + 1), vec_b = 3 * (size_t)sk_pad(N + 1) + 2 * sk_pad(R + 1);
  const size_t strip = (size_t)R * N;
  p.g.cached = (B * S <= nsm && (vec_b + strip) * 4 <= 200 * 1024) ? 1 : 0;
  p.smem_fwd = (vec_f + (p.g.cached ? strip : 0)) * 4;
  p.smem_bwd = (vec_b + (p.g.cached ? strip : 0)) * 4;
  return p;
}
static size_t sk_ws_floats(int B, int M, int N) {
  // u, v / dv, two partial planes of (B * S <= B + nsm) x (N + 1), barrier word (64 floats)
  const size_t parts = (size_t)(B + device_sm_count());
  return (size_t)B * (M + N + 2) + 2 * parts * (N + 1) + 64;
}

// ---- dense Sinkhorn output Z [B,M+1,N+1] (row pitch N+1): NLL head and match-filter statistics -----------------------
// SuperGlue's loss (superglue.py:322-352) and match filter (:301-311) read only the inner block and the two dustbins of
// Z: the reference builds dense fp32 copies of the mask and of mask * Z for it.  Here one pass reads the byte mask and
// touches Z only where the mask is set; every reduction runs in a fixed order (bit-identical across calls).
constexpr int kOtRows = 8;

// fixed-order sum over the block (256 threads); result valid in thread 0
__device__ __forceinline__ double ot_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) t += red[w];
  __syncthreads();
  return t;
}

// per (pair, strip of kOtRows rows): sum of Z over the positives of the strip
__global__ void __launch_bounds__(256) ot_nll_part_kernel(const float* __restrict__ Z, const uint8_t* __restrict__ mask,
                                                         float* __restrict__ part, int M, int N) {
  __shared__ double red[8];
  const int b = blockIdx.y, r0 = blockIdx.x * kOtRows, r1 = min(M, r0 + kOtRows);
  float acc = 0.f;
  for (int i = r0; i < r1; ++i) {
    const uint8_t* mrow = mask + ((int64_t)b * M + i) * N;
    const float* zrow = Z + ((int64_t)b * (M + 1) + i) * (N + 1);
    for (int j = threadIdx.x; j < N; j += 256)
      if (__ldg(mrow + j)) acc += __ldg(zrow + j);
  }
  const double t = ot_block_sum((double)acc, red);
  if (threadIdx.x == 0) part[(int64_t)b * gridDim.x + blockIdx.x] = (float)t;
}

// per pair: pos = sum of the strip partials, neg = sum_i neg0_i Z[i,N] + sum_j neg1_j Z[M,j]
__global__ void __launch_bounds__(256) ot_nll_final_kernel(const float* __restrict__ Z, const float* __restrict__ neg0,
                                                          const float* __restrict__ neg1, const float* __restrict__ part,
                                                          int nparts, float* __restrict__ pos, float* __restrict__ neg,
                                                          int M, int N) {
  __shared__ double red[8];
  const int b = blockIdx.x;
  double a = 0.0;
  for (int p = threadIdx.x; p < nparts; p += 256) a += (double)__ldg(part + (int64_t)b * nparts + p);
  const double tp = ot_block_sum(a, red);
  const float* zb = Z + (int64_t)b * (M + 1) * (N + 1);
  double c = 0.0;
  for (int i = threadIdx.x; i < M; i += 256) c += (double)__ldg(neg0 + (int64_t)b * M + i) * __ldg(zb + (int64_t)i * (N + 1) + N);
  for (int j = threadIdx.x; j < N; j += 256) c += (double)__ldg(neg1 + (int64_t)b * N + j) * __ldg(zb + (int64_t)M * (N + 1) + j);
  const double tn = ot_block_sum(c, red);
  if (threadIdx.x == 0) {
    pos[b] = (float)tp;
    neg[b] = (float)tn;
  }
}

// dZ of nll_pos = -pos / num_pos and nll_neg = -neg / num_neg for incoming per-pair gradients gpos, gneg (device)
__global__ void __launch_bounds__(256) ot_nll_bwd_kernel(const uint8_t* __restrict__ mask, const float* __restrict__ neg0,
                                                        const float* __restrict__ neg1, const float* __restrict__ num_pos,
                                                        const float* __restrict__ num_neg, const float* __restrict__ gpos,
                                                        const float* __restrict__ gneg, float* __restrict__ dZ, int M, int N) {
  const int b = blockIdx.y, r0 = blockIdx.x * kOtRows, r1 = min(M + 1, r0 + kOtRows);
  const float cp = -(__ldg(gpos + b) / __ldg(num_pos + b)), cn = -(__ldg(gneg + b) / __ldg(num_neg + b));
  for (int i = r0; i < r1; ++i) {
    float* drow = dZ + ((int64_t)b * (M + 1) + i) * (N + 1);
    if (i < M) {
      const uint8_t* mrow = mask + ((int64_t)b * M + i) * N;
      for (int j = threadIdx.x; j < N; j += 256) drow[j] = __ldg(mrow + j) ? cp : 0.f;
      if (threadIdx.x == 0) drow[N] = __ldg(neg0 + (int64_t)b * M + i) * cn;
    } else {
      for (int j = threadIdx.x; j < N; j += 256) drow[j] = __ldg(neg1 + (int64_t)b * N + j) * cn;
      if (threadIdx.x == 0) drow[N] = 0.f;
    }
  }
}

// row max / argmax of Z's inner block, first index on ties (warp per row)
__global__ void __launch_bounds__(256) ot_rowmax_kernel(const float* __restrict__ Z, float* __restrict__ rowmax,
                                                       int* __restrict__ rowarg, int M, int N) {
  const int b = blockIdx.y, i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= M) return;
  const float* zrow = Z + ((int64_t)b * (M + 1) + i) * (N + 1);
  float best = kNInf;
  int arg = lane < N ? lane : 0x7fffffff;
  for (int j = lane; j < N; j += 32) {
    const float x = __ldg(zrow + j);
    if (x > best) best = x, arg = j;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, best, o);
    const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
    if (v2 > best || (v2 == best && a2 < arg)) best = v2, arg = a2;
  }
  if (lane == 0) {
    rowmax[(int64_t)b * M + i] = best;
    rowarg[(int64_t)b * M + i] = arg;
  }
}

// column argmax of Z's inner block, first index on ties (thread per column, rows in order)
__global__ void __launch_bounds__(256) ot_colarg_kernel(const float* __restrict__ Z, int* __restrict__ colarg, int M,
                                                       int N) {
  const int b = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  const float* zc = Z + (int64_t)b * (M + 1) * (N + 1) + j;
  float best = __ldg(zc);
  int arg = 0;
  int i = 1;
  for (; i + 3 < M; i += 4) {
    float x[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) x[e] = __ldg(zc + (int64_t)(i + e) * (N + 1));
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (x[e] > best) best = x[e], arg = i + e;
  }
  for (; i < M; ++i) {
    const float x = __ldg(zc + (int64_t)i * (N + 1));
    if (x > best) best = x, arg = i;
  }
  colarg[(int64_t)b * N + j] = arg;
}

}  // namespace lgb

using namespace lgb;

extern "C" {

size_t lgb200_heads_ws_bytes(int B, int M, int N) {
  const size_t lds = (size_t)4 * B * (M + N + 2) + (size_t)8 * B * ((M + 31) / 32) * N;
  const size_t sk = 4 * sk_ws_floats(B, M, N);
  return lds > sk ? lds : sk;
}

static int log_double_softmax_impl(const float* sim, float bin_score, const float* bin_dev, float* scores, void* ws,
                                   int B, int M, int N, cudaStream_t stream);
int lgb200_log_double_softmax(const float* sim, float bin_score, float* scores, void* ws, int B, int M, int N,
                              cudaStream_t stream) {
  return log_double_softmax_impl(sim, bin_score, nullptr, scores, ws, B, M, N, stream);
}
int lgb200_log_double_softmax_dev(const float* sim, const float* bin_score_dev, float* scores, void* ws, int B, int M,
                                  int N, cudaStream_t stream) {
  LGB_REQUIRE(bin_score_dev, kErrInvalid, "log_double_softmax: null bin score pointer");
  return log_double_softmax_impl(sim, 0.f, bin_score_dev, scores, ws, B, M, N, stream);
}
static int log_double_softmax_impl(const float* sim, float bin_score, const float* bin_dev, float* scores, void* ws,
                                   int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && scores && ws, kErrInvalid, "log_double_softmax: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "log_double_softmax: empty input");
  // ws layout: [lse_row B*M][lse_col B*N][assign_lse scratch]
  float* lse_row = static_cast<float*>(ws);
  float* lse_col = lse_row + (size_t)B * M;
  void* sub = lse_col + (size_t)B * N;
  int rc = lgb200_assign_lse(sim, lse_row, lse_col, sub, B, M, N, stream);
  if (rc) return rc;
  lds_scores_kernel<<<dim3((M + 1 + 7) / 8, B), 256, 0, stream>>>(sim, lse_row, lse_col, bin_score, bin_dev, scores, M, N);
  return check_launch("log_double_softmax");
}

static int sk_launch(const void* fn, const SkPlan& p, size_t smem, void** args, cudaStream_t stream, const char* what) {
  if (int rc = ensure_dyn_smem(fn, (int)smem)) return rc;
  // cudaLaunchKernelExC with the cooperative attribute: the same co-residency guarantee as
  // cudaLaunchCooperativeKernel, and it is recorded into a CUDA graph when the stream is capturing
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(p.grid);
  cfg.blockDim = dim3(kSkThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelExC(&cfg, fn, args);
  if (e != cudaSuccess) (void)cudaGetLastError();  // do not leave the error for the next launch check to find
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "%s: cooperative launch (%d CTAs, %zu B smem): %s", what, p.grid, smem,
              cudaGetErrorString(e));
  return check_launch(what);
}

static int sinkhorn_fwd_impl(const float* sim, float alpha, const float* alpha_dev, int iters, float* out, float* uh,
                             float* vh, void* ws, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && ws, kErrInvalid, "sinkhorn: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0 && iters >= 0, kErrInvalid, "sinkhorn: bad arguments");
  LGB_REQUIRE((uh == nullptr) == (vh == nullptr), kErrInvalid, "sinkhorn: uh and vh go together");
  SkPlan p = sk_plan(B, M, N);
  float* u = static_cast<float*>(ws);
  float* v = u + (size_t)B * (M + 1);
  float* pm = v + (size_t)B * (N + 1);
  float* ps = pm + (size_t)(B + device_sm_count()) * (N + 1);
  unsigned* bar = reinterpret_cast<unsigned*>(ps + (size_t)(B + device_sm_count()) * (N + 1));
  LGB_REQUIRE(cudaMemsetAsync(bar, 0, sizeof(unsigned), stream) == cudaSuccess, kErrCuda, "sinkhorn: memset");
  void* args[] = {&sim, &alpha, &alpha_dev, &iters, &out, &u, &v, &uh, &vh, &pm, &ps, &bar, &p.g};
  return sk_launch((const void*)sk_fwd_persistent_kernel, p, p.smem_fwd, args, stream, "sinkhorn_fwd");
}

static int sinkhorn_bwd_impl(const float* sim, float alpha, const float* alpha_dev, int iters, const float* grad,
                             const float* uh, const float* vh, float* dsim, float* dzr, float* dzc, void* ws, int B,
                             int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && grad && uh && vh && dsim && dzr && dzc && ws, kErrInvalid, "sinkhorn_bwd: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0 && iters > 0, kErrInvalid, "sinkhorn_bwd: bad arguments");
  SkPlan p = sk_plan(B, M, N);
  float* dv = static_cast<float*>(ws) + (size_t)B * (M + 1);
  float* pw = dv + (size_t)B * (N + 1);
  unsigned* bar = reinterpret_cast<unsigned*>(pw + 2 * (size_t)(B + device_sm_count()) * (N + 1));
  LGB_REQUIRE(cudaMemsetAsync(bar, 0, sizeof(unsigned), stream) == cudaSuccess, kErrCuda, "sinkhorn_bwd: memset");
  void* args[] = {&sim, &alpha, &alpha_dev, &iters, &grad, &uh, &vh, &dsim, &dzr, &dzc, &dv, &pw, &bar, &p.g};
  return sk_launch((const void*)sk_bwd_persistent_kernel, p, p.smem_bwd, args, stream, "sinkhorn_bwd");
}

int lgb200_sinkhorn_fwd(const float* sim, float alpha, int iters, float* out, float* uh, float* vh, void* ws, int B,
                        int M, int N, cudaStream_t stream) {
  return sinkhorn_fwd_impl(sim, alpha, nullptr, iters, out, uh, vh, ws, B, M, N, stream);
}

int lgb200_sinkhorn_fwd_dev(const float* sim, const float* alpha_dev, int iters, float* out, float* uh, float* vh,
                            void* ws, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(alpha_dev, kErrInvalid, "sinkhorn: null bin score pointer");
  return sinkhorn_fwd_impl(sim, 0.f, alpha_dev, iters, out, uh, vh, ws, B, M, N, stream);
}

int lgb200_sinkhorn(const float* sim, float alpha, int iters, float* out, void* ws, int B, int M, int N,
                    cudaStream_t stream) {
  LGB_REQUIRE(out, kErrInvalid, "sinkhorn: null pointer");
  return lgb200_sinkhorn_fwd(sim, alpha, iters, out, nullptr, nullptr, ws, B, M, N, stream);
}

int lgb200_sinkhorn_bwd(const float* sim, float alpha, int iters, const float* grad, const float* uh, const float* vh,
                        float* dsim, float* dzr, float* dzc, void* ws, int B, int M, int N, cudaStream_t stream) {
  return sinkhorn_bwd_impl(sim, alpha, nullptr, iters, grad, uh, vh, dsim, dzr, dzc, ws, B, M, N, stream);
}

int lgb200_sinkhorn_bwd_dev(const float* sim, const float* alpha_dev, int iters, const float* grad, const float* uh,
                            const float* vh, float* dsim, float* dzr, float* dzc, void* ws, int B, int M, int N,
                            cudaStream_t stream) {
  LGB_REQUIRE(alpha_dev, kErrInvalid, "sinkhorn_bwd: null bin score pointer");
  return sinkhorn_bwd_impl(sim, 0.f, alpha_dev, iters, grad, uh, vh, dsim, dzr, dzc, ws, B, M, N, stream);
}

int lgb200_ot_nll_fwd(const float* Z, const uint8_t* mask, const float* neg0, const float* neg1, float* pos, float* neg,
                      void* ws, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(Z && mask && neg0 && neg1 && pos && neg && ws, kErrInvalid, "ot_nll_fwd: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "ot_nll_fwd: empty input");
  const int nparts = (M + kOtRows - 1) / kOtRows;
  float* part = static_cast<float*>(ws);
  ot_nll_part_kernel<<<dim3(nparts, B), 256, 0, stream>>>(Z, mask, part, M, N);
  if (int rc = check_launch("ot_nll_fwd")) return rc;
  ot_nll_final_kernel<<<B, 256, 0, stream>>>(Z, neg0, neg1, part, nparts, pos, neg, M, N);
  return check_launch("ot_nll_fwd");
}

int lgb200_ot_nll_bwd(const uint8_t* mask, const float* neg0, const float* neg1, const float* num_pos,
                      const float* num_neg, const float* gpos, const float* gneg, float* dZ, int B, int M, int N,
                      cudaStream_t stream) {
  LGB_REQUIRE(mask && neg0 && neg1 && num_pos && num_neg && gpos && gneg && dZ, kErrInvalid, "ot_nll_bwd: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "ot_nll_bwd: empty input");
  ot_nll_bwd_kernel<<<dim3((M + 1 + kOtRows - 1) / kOtRows, B), 256, 0, stream>>>(mask, neg0, neg1, num_pos, num_neg,
                                                                                 gpos, gneg, dZ, M, N);
  return check_launch("ot_nll_bwd");
}

int lgb200_ot_filter_stats(const float* Z, float* rowmax, int* rowarg, int* colarg, int B, int M, int N,
                           cudaStream_t stream) {
  LGB_REQUIRE(Z && rowmax && rowarg && colarg, kErrInvalid, "ot_filter_stats: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "ot_filter_stats: empty input");
  ot_rowmax_kernel<<<dim3((M + 7) / 8, B), 256, 0, stream>>>(Z, rowmax, rowarg, M, N);
  if (int rc = check_launch("ot_filter_stats")) return rc;
  ot_colarg_kernel<<<dim3((N + 255) / 256, B), 256, 0, stream>>>(Z, colarg, M, N);
  return check_launch("ot_filter_stats");
}

}  // extern "C"
