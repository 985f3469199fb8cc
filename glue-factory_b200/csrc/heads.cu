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

// Varlen batches (GlueStick's packed evaluation heads): pair g < G of the padded [G, M, N] sim has its own extents
// m = pairs[g] <= M, n = pairs[G + g] <= N (M and N become strides; nothing past a pair's extents is read).  Its scores
// go to batch row pairs[2G + g] of the output [*, Mo + 1, No + 1] at the same row / column indices, with its dustbin
// row and column at Mo / No; every other entry keeps its contents.  The row max / argmax of the inner block (first
// index on ties) go to rowmax / rowarg [G, M], for lgb200_filter_matches_varlen.
struct LdsVarlen {
  const int* pairs;  // [3, G]: m, n, output batch row
  float* rowmax;     // [G, M]
  int* rowarg;       // [G, M]
  int G, Mo, No;
};

// scores from precomputed lse_row / lse_col of the UNBORDERED sim
template <bool kVarlen>
__global__ void __launch_bounds__(256) lds_scores_kernel(const float* __restrict__ sim, const float* __restrict__ lse_row,
                                                        const float* __restrict__ lse_col, float beta,
                                                        const float* __restrict__ beta_dev,
                                                        float* __restrict__ scores, int M, int N, LdsVarlen vp) {
  if (beta_dev) beta = __ldg(beta_dev);  // the learnt bin score read from device memory (no host read-back)
  const int b = blockIdx.y;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  int Mb = M, Nb = N, Mp = M, Np = N;  // this pair's extents (M, N are the strides) and the output's
  int64_t ob = b;                      // output batch row
  if constexpr (kVarlen) {
    Mb = min(vp.pairs[b], M);
    Nb = min(vp.pairs[vp.G + b], N);
    Mp = vp.Mo;
    Np = vp.No;
    ob = vp.pairs[2 * vp.G + b];
  }
  if (i > Mb) return;
  float* orow = scores + (ob * (Mp + 1) + ((kVarlen && i == Mb) ? Mp : i)) * (Np + 1);
  if (i == Mb) {
    for (int j = lane; j <= Nb; j += 32)
      orow[(kVarlen && j == Nb) ? Np : j] = j < Nb ? beta - logaddexp_f(lse_col[(int64_t)b * N + j], beta) : 0.f;
    return;
  }
  const float lr = logaddexp_f(lse_row[(int64_t)b * M + i], beta);
  const float* srow = sim + ((int64_t)b * M + i) * N;
  float best = kNInf;
  int arg = 0x7fffffff;
  for (int j = lane; j < Nb; j += 32) {
    const float x = srow[j];
    const float lc = logaddexp_f(lse_col[(int64_t)b * N + j], beta);
    const float s = ((x - lr) + (x - lc)) * 0.5f;
    orow[j] = s;
    if constexpr (kVarlen) {
      if (s > best || arg == 0x7fffffff) best = s, arg = j;
    }
  }
  if (lane == 0) orow[Np] = beta - lr;
  if constexpr (kVarlen) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v2 = __shfl_xor_sync(0xffffffffu, best, o);
      const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
      if (a2 != 0x7fffffff && (arg == 0x7fffffff || v2 > best || (v2 == best && a2 < arg))) best = v2, arg = a2;
    }
    if (lane == 0) {
      vp.rowmax[(int64_t)b * M + i] = best;
      vp.rowarg[(int64_t)b * M + i] = arg;
    }
  }
}

// column argmax of a varlen pair's inner scores as written by lds_scores_kernel<true> (first row on ties; thread per
// column, rows in order)
__global__ void __launch_bounds__(256) lds_colarg_varlen_kernel(const float* __restrict__ scores, int* __restrict__ colarg,
                                                               int N, LdsVarlen vp) {
  const int b = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
  const int Mb = vp.pairs[b], Nb = min(vp.pairs[vp.G + b], N);
  if (j >= Nb) return;
  const int64_t pitch = vp.No + 1;
  const float* col = scores + (int64_t)vp.pairs[2 * vp.G + b] * (vp.Mo + 1) * pitch + j;
  float best = col[0];
  int arg = 0;
  for (int i = 1; i < Mb; ++i) {
    const float x = col[(int64_t)i * pitch];
    if (x > best) best = x, arg = i;
  }
  colarg[(int64_t)b * N + j] = arg;
}

// raw line scores (gluestick.py:348-361) of a varlen pair straight from its endpoint similarity block:
//   raw[g, i, j] = 0.5 * max(s[a0, c0] + s[a1, c1], s[a0, c1] + s[a1, c0]),
// a0 / a1 = junc0[g, 2i], [2i + 1], c0 / c1 = junc1[g, 2j], [2j + 1], s = sim[g] ([P0, P1] pitch).  Same operations
// in the same order as the torch formula (two gathers, two adds, maximum, scale).  Thread per (i, j), j fastest.
// kTrain (the training path): the maximum propagates a NaN like torch.maximum (fmaxf drops a one-sided one), and a
// junction index outside [0, P0) / [0, P1) gives NaN instead of a read outside the pair's block.
template <bool kTrain>
__global__ void __launch_bounds__(256) line_scores_varlen_kernel(const float* __restrict__ sim,
                                                                const int* __restrict__ junc0,
                                                                const int* __restrict__ junc1, float* __restrict__ raw,
                                                                const int* __restrict__ pairs, int G, int P0, int P1,
                                                                int L0, int L1) {
  const int g = blockIdx.z, i = blockIdx.y;
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int Lb0 = min(pairs[g], L0), Lb1 = min(pairs[G + g], L1);
  if (i >= Lb0 || j >= Lb1) return;
  const float* s = sim + (int64_t)g * P0 * P1;
  const int a0 = __ldg(junc0 + (int64_t)g * 2 * L0 + 2 * i), a1 = __ldg(junc0 + (int64_t)g * 2 * L0 + 2 * i + 1);
  const int c0 = __ldg(junc1 + (int64_t)g * 2 * L1 + 2 * j), c1 = __ldg(junc1 + (int64_t)g * 2 * L1 + 2 * j + 1);
  if constexpr (kTrain) {
    if ((unsigned)a0 >= (unsigned)P0 || (unsigned)a1 >= (unsigned)P0 || (unsigned)c0 >= (unsigned)P1 ||
        (unsigned)c1 >= (unsigned)P1) {
      raw[((int64_t)g * L0 + i) * L1 + j] = __int_as_float(0x7fffffff);
      return;
    }
  }
  const float* r0 = s + (int64_t)a0 * P1;
  const float* r1 = s + (int64_t)a1 * P1;
  const float straight = __fadd_rn(__ldg(r0 + c0), __ldg(r1 + c1));
  const float swapped = __fadd_rn(__ldg(r0 + c1), __ldg(r1 + c0));
  float m = fmaxf(straight, swapped);
  if constexpr (kTrain) m = isnan(straight) ? straight : isnan(swapped) ? swapped : m;
  raw[((int64_t)g * L0 + i) * L1 + j] = 0.5f * m;
}

// d sim of line_scores_varlen_kernel<true> (the autograd of the torch formula, summed in a fixed order): for each
// (r, c) of pair g, every endpoint k0 of view 0 at junction r (CSR: order0[ptr0[g, r] .. ptr0[g, r + 1]), indices into
// junc0's flat [G, 2 L0], sorted) meets every endpoint k1 of view 1 at junction c.  Their lines i = k0 / 2, j = k1 / 2
// take s[r, c] in the straight branch when k0 and k1 are the same end (k0 % 2 == k1 % 2), else in the swapped one, and
// the branch passes on 0.5 * graw[g, i, j] times torch.maximum's weight: 1 to the larger branch, 0 to the smaller
// (skipped, so a non-finite graw there does not leak), 1/2 to each on an exact tie, 1 to both when either is NaN.
// Lines past a pair's (m, n), lines with a junction index outside the block and entries of another pair are skipped.  Thread per (r, c),
// c fastest: the view-0 list is the same for the whole CTA.  Entries no line touches get 0.
__global__ void __launch_bounds__(256) line_scores_bwd_kernel(const float* __restrict__ graw,
                                                             const float* __restrict__ sim,
                                                             const int* __restrict__ junc0,
                                                             const int* __restrict__ junc1,
                                                             const int* __restrict__ order0,
                                                             const int* __restrict__ ptr0,
                                                             const int* __restrict__ order1,
                                                             const int* __restrict__ ptr1, const int* __restrict__ pairs,
                                                             float* __restrict__ dsim, int G, int P0, int P1, int L0,
                                                             int L1) {
  const int g = blockIdx.z, r = blockIdx.y;
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= P1) return;
  const int Lb0 = min(pairs[g], L0), Lb1 = min(pairs[G + g], L1);
  const float* s = sim + (int64_t)g * P0 * P1;
  const int64_t e0 = (int64_t)g * 2 * L0, e1 = (int64_t)g * 2 * L1;  // pair g's first entries of junc0 / junc1
  const int b0 = __ldg(ptr0 + (int64_t)g * (P0 + 1) + r), n0 = __ldg(ptr0 + (int64_t)g * (P0 + 1) + r + 1);
  const int b1 = __ldg(ptr1 + (int64_t)g * (P1 + 1) + c), n1 = __ldg(ptr1 + (int64_t)g * (P1 + 1) + c + 1);
  float acc = 0.f;
  for (int p = b0; p < n0; ++p) {
    const int k0 = __ldg(order0 + p) - (int)e0, i = k0 >> 1;
    if ((unsigned)i >= (unsigned)Lb0) continue;  // also an endpoint of another pair (a junction index >= n)
    const int a0 = __ldg(junc0 + e0 + 2 * i), a1 = __ldg(junc0 + e0 + 2 * i + 1);
    if ((unsigned)a0 >= (unsigned)P0 || (unsigned)a1 >= (unsigned)P0) continue;
    const float* r0 = s + (int64_t)a0 * P1;
    const float* r1 = s + (int64_t)a1 * P1;
    for (int q = b1; q < n1; ++q) {
      const int k1 = __ldg(order1 + q) - (int)e1, j = k1 >> 1;
      if ((unsigned)j >= (unsigned)Lb1) continue;
      const int c0 = __ldg(junc1 + e1 + 2 * j), c1 = __ldg(junc1 + e1 + 2 * j + 1);
      if ((unsigned)c0 >= (unsigned)P1 || (unsigned)c1 >= (unsigned)P1) continue;
      const float straight = __fadd_rn(__ldg(r0 + c0), __ldg(r1 + c1));
      const float swapped = __fadd_rn(__ldg(r0 + c1), __ldg(r1 + c0));
      const bool mine_straight = (k0 & 1) == (k1 & 1);
      const float mine = mine_straight ? straight : swapped, other = mine_straight ? swapped : straight;
      if (mine < other) continue;  // false with a NaN on either side: both branches get the gradient
      const float d = __fmul_rn(__ldg(graw + ((int64_t)g * L0 + i) * L1 + j), 0.5f);
      acc = __fadd_rn(acc, mine == other ? __fmul_rn(d, 0.5f) : d);
    }
  }
  dsim[((int64_t)g * P0 + r) * P1 + c] = acc;
}

// x[row] += mean of the endpoint updates upd[e] whose target row is `row` (the LineLayer's scatter-mean over
// junctions, gluestick.py:682-690).  order [E]: the endpoints sorted stably by target row, tgt_sorted [E] their rows;
// each run of equal rows is summed in that order (a fixed order: no atomics, and a pair's sums do not depend on the
// other pairs, whose rows differ).  Warp per sorted position; the warp at the start of a run owns the run.
// kPartnerSum: the backward of the LineLayer's endpoint gather instead, x[row] += the sum over the run of
// upd[e, :D] + upd[e ^ 1, D:2D] (endpoint e read its own junction into columns 0..D-1 and its line's other end e ^ 1
// read it into columns D..2D-1); upd has row pitch ld.
template <bool kPartnerSum>
__global__ void __launch_bounds__(256) junction_mean_kernel(float* __restrict__ x, const float* __restrict__ upd,
                                                           const int* __restrict__ order,
                                                           const int* __restrict__ tgt_sorted, int E, int D, int ld) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= E) return;
  const int row = __ldg(tgt_sorted + k);
  if (k > 0 && __ldg(tgt_sorted + k - 1) == row) return;
  int end = k + 1;
  while (end < E && __ldg(tgt_sorted + end) == row) ++end;
  const float cnt = (float)(end - k);
  for (int c = lane * 4; c < D; c += 128) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = k; e < end; ++e) {
      if constexpr (kPartnerSum) {
        const int o = __ldg(order + e);
        const float4 u = __ldg(reinterpret_cast<const float4*>(upd + (int64_t)o * ld + c));
        const float4 w = __ldg(reinterpret_cast<const float4*>(upd + (int64_t)(o ^ 1) * ld + D + c));
        s.x = __fadd_rn(s.x, u.x); s.y = __fadd_rn(s.y, u.y); s.z = __fadd_rn(s.z, u.z); s.w = __fadd_rn(s.w, u.w);
        s.x = __fadd_rn(s.x, w.x); s.y = __fadd_rn(s.y, w.y); s.z = __fadd_rn(s.z, w.z); s.w = __fadd_rn(s.w, w.w);
      } else {
        const float4 u = __ldg(reinterpret_cast<const float4*>(upd + (int64_t)__ldg(order + e) * D + c));
        s.x = __fadd_rn(s.x, u.x); s.y = __fadd_rn(s.y, u.y); s.z = __fadd_rn(s.z, u.z); s.w = __fadd_rn(s.w, u.w);
      }
    }
    float4* xr = reinterpret_cast<float4*>(x + (int64_t)row * D + c);
    float4 v = *xr;
    if constexpr (kPartnerSum) {
      v.x = __fadd_rn(v.x, s.x); v.y = __fadd_rn(v.y, s.y); v.z = __fadd_rn(v.z, s.z); v.w = __fadd_rn(v.w, s.w);
    } else {
      v.x = __fadd_rn(v.x, __fdiv_rn(s.x, cnt)); v.y = __fadd_rn(v.y, __fdiv_rn(s.y, cnt));
      v.z = __fadd_rn(v.z, __fdiv_rn(s.z, cnt)); v.w = __fadd_rn(v.w, __fdiv_rn(s.w, cnt));
    }
    *xr = v;
  }
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

// ---- packed Sinkhorn (SuperGlue's packed evaluation head): G pairs of their own sizes in one persistent launch ----
// Pair g < G of the padded sim [G, M, N] has m = pairs[g] <= M rows and n = pairs[G + g] <= N columns (M and N are
// strides: nothing past (m, n) is read).  Its strips are kSkvRows rows each, S = ceil(m / kSkvRows) of them, the last
// one owning the dustbin row; in the merge phase strip s of the pair owns the columns [s C, (s + 1) C) of its n + 1,
// C = ceil((n + 1) / S).  So a pair's strip geometry and every summation order are functions of (m, n) alone, never
// of G, the other pairs or the grid: a pair's result is bit-identical in any batch.  Work item = (pair, strip), items
// of a pair consecutive; the item table is built on the device (sk_varlen_items_kernel), so no host read sizes the
// launch.  Iterations as sk_fwd_persistent_kernel (two grid barriers each); no strip cache (a 32-row strip of a wide
// pair does not fit in shared memory, and a CTA may own several items).  Output: pair g's block goes to row
// pairs[2G + g] of out [*, Mo + 1, No + 1], its dustbin column at No, its dustbin row at Mo; other entries are kept.
constexpr int kSkvRows = 32;  // one row per warp of the 1024-thread CTA in the row phase

struct SkvGeom {
  const int* pairs;  // [3, G]: m, n, output batch row
  const int2* tab;   // [items]: (pair, strip)
  const int* start;  // [G + 1]: each pair's first item; start[G] = item count
  int G, M, N, Mo, No;
};

__device__ __forceinline__ int skv_strips(int m) { return m > 0 ? (m + kSkvRows - 1) / kSkvRows : 0; }

// one CTA: the pairs' first items (serial prefix over G, thread 0), then the table (warp per pair); resets the barrier
__global__ void __launch_bounds__(1024) sk_varlen_items_kernel(const int* __restrict__ pairs, int G, int M, int N,
                                                              int2* __restrict__ tab, int* __restrict__ start,
                                                              unsigned* __restrict__ bar) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < G; ++g) {
      start[g] = acc;
      acc += min(pairs[G + g], N) > 0 ? skv_strips(min(pairs[g], M)) : 0;
    }
    start[G] = acc;
    *bar = 0u;
  }
  __syncthreads();
  for (int g = threadIdx.x >> 5; g < G; g += 32) {
    const int s0 = start[g], S = start[g + 1] - s0;
    for (int s = threadIdx.x & 31; s < S; s += 32) tab[s0 + s] = make_int2(g, s);
  }
}

__global__ void __launch_bounds__(kSkThreads, 1)
sk_fwd_varlen_kernel(const float* __restrict__ sim, const float* __restrict__ alpha_dev, int iters,
                     float* __restrict__ out, float* __restrict__ u, float* __restrict__ v, float* __restrict__ pm,
                     float* __restrict__ ps, unsigned* __restrict__ bar, SkvGeom q) {
  extern __shared__ float sk_smem[];
  const int M = q.M, N = q.N, G = q.G;
  float* vsm = sk_smem;                  // n + 1
  float* usm = vsm + sk_pad(N + 1);      // kSkvRows + 1
  const float alpha = __ldg(alpha_dev);  // the learnt bin score read from device memory (no host read-back)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int items = __ldcg(q.start + G);
  unsigned target = 0;
  for (int it = 0; it < iters; ++it) {
    // ---- row phase
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int2 e = __ldg(q.tab + w);
      const int b = e.x, s = e.y;
      const int m = min(q.pairs[b], M), n = min(q.pairs[G + b], N), S = skv_strips(m);
      const int i0 = s * kSkvRows, i1 = min(m, i0 + kSkvRows);
      const int nrows = i1 - i0 + (s == S - 1 ? 1 : 0);
      const float norm = -logf((float)(m + n));
      for (int j = tid; j <= n; j += kSkThreads) vsm[j] = it ? __ldcg(v + (int64_t)b * (N + 1) + j) : 0.f;
      __syncthreads();
      for (int r = warp; r < nrows; r += 32) {
        const int i = i0 + r;
        float mx = kNInf, sm = 0.f;
        if (i < m) {
          const float* row = sim + ((int64_t)b * M + i) * N;
          int j = lane;
          for (; j + 224 < n; j += 256) {  // eight loads in flight per lane
            float x[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = row[j + 32 * k];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] += vsm[j + 32 * k];
            lse4(mx, sm, x[0], x[1], x[2], x[3]);
            lse4(mx, sm, x[4], x[5], x[6], x[7]);
          }
          for (; j + 96 < n; j += 128)
            lse4(mx, sm, row[j] + vsm[j], row[j + 32] + vsm[j + 32], row[j + 64] + vsm[j + 64], row[j + 96] + vsm[j + 96]);
          for (; j < n; j += 32) lse1(mx, sm, row[j] + vsm[j]);
        } else {
          for (int j = lane; j < n; j += 32) lse1(mx, sm, alpha + vsm[j]);
        }
        lse_warp(mx, sm);
        if (lane == 0) {
          lse1(mx, sm, alpha + vsm[n]);
          const float ui = (i < m ? norm : logf((float)n) + norm) - (mx + logf(sm));
          usm[r] = ui;
          u[(int64_t)b * (M + 1) + i] = ui;
        }
      }
      __syncthreads();
      // column partials over the strip's dense rows (the dustbin row is added in the merge)
      for (int j = tid; j <= n; j += kSkThreads) {
        float mx = kNInf, sm = 0.f;
        if (j < n) {
          const float* col = sim + ((int64_t)b * M + i0) * N + j;
          int r = 0;
          for (; r + 7 < i1 - i0; r += 8) {
            float x[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = col[(int64_t)(r + k) * N];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] += usm[r + k];
            lse4(mx, sm, x[0], x[1], x[2], x[3]);
            lse4(mx, sm, x[4], x[5], x[6], x[7]);
          }
          for (; r + 3 < i1 - i0; r += 4)
            lse4(mx, sm, col[(int64_t)r * N] + usm[r], col[(int64_t)(r + 1) * N] + usm[r + 1],
                 col[(int64_t)(r + 2) * N] + usm[r + 2], col[(int64_t)(r + 3) * N] + usm[r + 3]);
          for (; r < i1 - i0; ++r) lse1(mx, sm, col[(int64_t)r * N] + usm[r]);
        } else {
          for (int r = 0; r < i1 - i0; ++r) lse1(mx, sm, alpha + usm[r]);
        }
        pm[(int64_t)w * (N + 1) + j] = mx;
        ps[(int64_t)w * (N + 1) + j] = sm;
      }
      __syncthreads();
    }
    sk_grid_barrier(bar, target);
    // ---- merge phase: warp per column of the item's slice, the pair's S partials in strip order
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int2 e = __ldg(q.tab + w);
      const int b = e.x, s = e.y;
      const int m = min(q.pairs[b], M), n = min(q.pairs[G + b], N), S = skv_strips(m);
      const int C = (n + S) / S, j0 = s * C, j1 = min(n + 1, j0 + C);
      const int64_t p_first = w - s;  // item of the pair's strip 0
      const float norm = -logf((float)(m + n));
      const float ubin = alpha + __ldcg(u + (int64_t)b * (M + 1) + m);
      for (int j = j0 + warp; j < j1; j += 32) {
        float mx = kNInf, sm = 0.f;
        for (int p0 = 0; p0 < S; p0 += 128) {  // four partial pairs in flight per lane
          float m2[4], s2[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int p = p0 + k * 32 + lane;
            const int64_t o = (p_first + (p < S ? p : 0)) * (N + 1) + j;
            m2[k] = p < S ? __ldcg(pm + o) : kNInf;
            s2[k] = p < S ? __ldcg(ps + o) : 0.f;
          }
          const float mn = fmaxf(fmaxf(fmaxf(m2[0], m2[1]), fmaxf(m2[2], m2[3])), mx);
          if (mn != kNInf) {
            sm = sm * __expf(mx - mn);
#pragma unroll
            for (int k = 0; k < 4; ++k) sm += s2[k] * __expf(m2[k] - mn);
            mx = mn;
          }
        }
        lse_warp(mx, sm);
        if (lane == 0) {
          lse1(mx, sm, ubin);
          v[(int64_t)b * (N + 1) + j] = (j < n ? norm : logf((float)m) + norm) - (mx + logf(sm));
        }
      }
    }
    sk_grid_barrier(bar, target);
  }
  // ---- output: out = Z + u + v - norm, at the pair's output row with the dustbins at (Mo, No)
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    const int2 e = __ldg(q.tab + w);
    const int b = e.x, s = e.y;
    const int m = min(q.pairs[b], M), n = min(q.pairs[G + b], N), S = skv_strips(m);
    const int i0 = s * kSkvRows, i1 = min(m, i0 + kSkvRows);
    const int nrows = i1 - i0 + (s == S - 1 ? 1 : 0);
    const float norm = -logf((float)(m + n));
    const int64_t pitch = q.No + 1;
    float* ob = out + (int64_t)q.pairs[2 * G + b] * (q.Mo + 1) * pitch;
    for (int j = tid; j <= n; j += kSkThreads) vsm[j] = iters ? __ldcg(v + (int64_t)b * (N + 1) + j) : 0.f;
    __syncthreads();
    for (int r = warp; r < nrows; r += 32) {
      const int i = i0 + r;
      const float ui = (iters ? __ldcg(u + (int64_t)b * (M + 1) + i) : 0.f) - norm;
      if (i < m) {
        const float* row = sim + ((int64_t)b * M + i) * N;
        float* orow = ob + (int64_t)i * pitch;
        for (int j = lane; j < n; j += 32) orow[j] = row[j] + ui + vsm[j];
        if (lane == 0) orow[q.No] = alpha + ui + vsm[n];
      } else {
        float* orow = ob + (int64_t)q.Mo * pitch;
        for (int j = lane; j <= n; j += 32) orow[j < n ? j : q.No] = alpha + ui + vsm[j];
      }
    }
    __syncthreads();
  }
}

// the item table (two ints per item, at most G * ceil(M / kSkvRows) items), the pairs' first items (G + 1), the
// barrier word, u [G, M + 1], v [G, N + 1] and two partial planes of items x (N + 1), in 4-byte words
static size_t skv_ws_floats(int G, int M, int N) {
  const size_t items = (size_t)G * ((M + kSkvRows - 1) / kSkvRows);
  return 2 * items + G + 2 + (size_t)G * (M + N + 2) + 2 * items * (N + 1);
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

// The same two kernels with the positives given as match lists gt0 [B,M] / gt1 [B,N] (int64, one-to-one): row i's
// positive is Z[i, gt0[i]].  Thread t adds it when gt0[i] % 256 == t, so every thread sees the same entries in the same
// order as in ot_nll_part_kernel and the partials, the sums and dZ are bit-identical to the mask's.  A row whose
// partner disagrees (gt0[i] >= N, or gt1[gt0[i]] != i) adds NaN to its strip.
__global__ void __launch_bounds__(256) ot_nll_part_sparse_kernel(const float* __restrict__ Z,
                                                                const int64_t* __restrict__ gt0,
                                                                const int64_t* __restrict__ gt1,
                                                                float* __restrict__ part, int M, int N) {
  __shared__ double red[8];
  const int b = blockIdx.y, r0 = blockIdx.x * kOtRows, r1 = min(M, r0 + kOtRows);
  float acc = 0.f;
  for (int i = r0; i < r1; ++i) {
    const int64_t j = __ldg(gt0 + (int64_t)b * M + i);
    if (j < 0 || j % 256 != threadIdx.x) continue;
    if (j >= N || __ldg(gt1 + (int64_t)b * N + j) != i) acc += NAN;
    else acc += __ldg(Z + ((int64_t)b * (M + 1) + i) * (N + 1) + j);
  }
  const double t = ot_block_sum((double)acc, red);
  if (threadIdx.x == 0) part[(int64_t)b * gridDim.x + blockIdx.x] = (float)t;
}

__global__ void __launch_bounds__(256) ot_nll_bwd_sparse_kernel(const int64_t* __restrict__ gt0,
                                                               const float* __restrict__ neg0,
                                                               const float* __restrict__ neg1,
                                                               const float* __restrict__ num_pos,
                                                               const float* __restrict__ num_neg,
                                                               const float* __restrict__ gpos,
                                                               const float* __restrict__ gneg, float* __restrict__ dZ,
                                                               int M, int N) {
  const int b = blockIdx.y, r0 = blockIdx.x * kOtRows, r1 = min(M + 1, r0 + kOtRows);
  const float cp = -(__ldg(gpos + b) / __ldg(num_pos + b)), cn = -(__ldg(gneg + b) / __ldg(num_neg + b));
  for (int i = r0; i < r1; ++i) {
    float* drow = dZ + ((int64_t)b * (M + 1) + i) * (N + 1);
    if (i < M) {
      const int64_t jp = __ldg(gt0 + (int64_t)b * M + i);
      for (int j = threadIdx.x; j < N; j += 256) drow[j] = j == jp ? cp : 0.f;
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
  lds_scores_kernel<false><<<dim3((M + 1 + 7) / 8, B), 256, 0, stream>>>(sim, lse_row, lse_col, bin_score, bin_dev,
                                                                          scores, M, N, LdsVarlen{});
  return check_launch("log_double_softmax");
}

int lgb200_log_double_softmax_varlen(const float* sim, const float* bin_score_dev, float* scores, float* rowmax,
                                     int* rowarg, int* colarg, void* ws, const int* pairs, int G, int M, int N, int Mo,
                                     int No, cudaStream_t stream) {
  LGB_REQUIRE(sim && bin_score_dev && scores && rowmax && rowarg && colarg && ws && pairs, kErrInvalid,
              "log_double_softmax_varlen: null pointer");
  LGB_REQUIRE(G > 0 && G <= 65535 && M > 0 && N > 0 && Mo > 0 && No > 0, kErrInvalid,
              "log_double_softmax_varlen: bad extents G=%d M=%d N=%d Mo=%d No=%d", G, M, N, Mo, No);
  // ws layout as lgb200_log_double_softmax's: [lse_row G*M][lse_col G*N][assign_lse scratch]
  float* lse_row = static_cast<float*>(ws);
  float* lse_col = lse_row + (size_t)G * M;
  void* sub = lse_col + (size_t)G * N;
  int rc = lgb200_assign_lse_varlen(sim, lse_row, lse_col, sub, pairs, G, M, N, stream);
  if (rc) return rc;
  const LdsVarlen vp{pairs, rowmax, rowarg, G, Mo, No};
  lds_scores_kernel<true><<<dim3((M + 1 + 7) / 8, G), 256, 0, stream>>>(sim, lse_row, lse_col, 0.f, bin_score_dev,
                                                                        scores, M, N, vp);
  if ((rc = check_launch("log_double_softmax_varlen"))) return rc;
  lds_colarg_varlen_kernel<<<dim3((N + 255) / 256, G), 256, 0, stream>>>(scores, colarg, N, vp);
  return check_launch("log_double_softmax_varlen");
}

static int line_scores_launch(bool train, const float* sim, const int* junc0, const int* junc1, float* raw,
                              const int* pairs, int G, int P0, int P1, int L0, int L1, cudaStream_t stream,
                              const char* what) {
  LGB_REQUIRE(sim && junc0 && junc1 && raw && pairs, kErrInvalid, "%s: null pointer", what);
  LGB_REQUIRE(G > 0 && G <= 65535 && P0 > 0 && P1 > 0 && L0 > 0 && L0 <= 65535 && L1 > 0, kErrInvalid,
              "%s: bad extents G=%d P0=%d P1=%d L0=%d L1=%d", what, G, P0, P1, L0, L1);
  const dim3 grid((L1 + 255) / 256, L0, G);
  if (train)
    line_scores_varlen_kernel<true><<<grid, 256, 0, stream>>>(sim, junc0, junc1, raw, pairs, G, P0, P1, L0, L1);
  else
    line_scores_varlen_kernel<false><<<grid, 256, 0, stream>>>(sim, junc0, junc1, raw, pairs, G, P0, P1, L0, L1);
  return check_launch(what);
}

int lgb200_line_scores_varlen(const float* sim, const int* junc0, const int* junc1, float* raw, const int* pairs, int G,
                              int P0, int P1, int L0, int L1, cudaStream_t stream) {
  return line_scores_launch(false, sim, junc0, junc1, raw, pairs, G, P0, P1, L0, L1, stream, "line_scores_varlen");
}

int lgb200_line_scores_train(const float* sim, const int* junc0, const int* junc1, float* raw, const int* pairs, int G,
                             int P0, int P1, int L0, int L1, cudaStream_t stream) {
  return line_scores_launch(true, sim, junc0, junc1, raw, pairs, G, P0, P1, L0, L1, stream, "line_scores_train");
}

int lgb200_line_scores_bwd(const float* graw, const float* sim, const int* junc0, const int* junc1, const int* order0,
                           const int* ptr0, const int* order1, const int* ptr1, const int* pairs, float* dsim, int G,
                           int P0, int P1, int L0, int L1, cudaStream_t stream) {
  LGB_REQUIRE(graw && sim && junc0 && junc1 && order0 && ptr0 && order1 && ptr1 && pairs && dsim, kErrInvalid,
              "line_scores_bwd: null pointer");
  LGB_REQUIRE(G > 0 && G <= 65535 && P0 > 0 && P0 <= 65535 && P1 > 0 && L0 > 0 && L1 > 0, kErrInvalid,
              "line_scores_bwd: bad extents G=%d P0=%d P1=%d L0=%d L1=%d", G, P0, P1, L0, L1);
  line_scores_bwd_kernel<<<dim3((P1 + 255) / 256, P0, G), 256, 0, stream>>>(graw, sim, junc0, junc1, order0, ptr0,
                                                                             order1, ptr1, pairs, dsim, G, P0, P1, L0,
                                                                             L1);
  return check_launch("line_scores_bwd");
}

int lgb200_junction_mean_varlen(float* x, const float* upd, const int* order, const int* tgt_sorted, int E, int D,
                                cudaStream_t stream) {
  LGB_REQUIRE(x && upd && order && tgt_sorted, kErrInvalid, "junction_mean_varlen: null pointer");
  LGB_REQUIRE(E > 0 && D > 0 && D % 4 == 0, kErrInvalid, "junction_mean_varlen: bad extents E=%d D=%d", E, D);
  LGB_REQUIRE(((uintptr_t)x | (uintptr_t)upd) % 16 == 0, kErrInvalid, "junction_mean_varlen: x / upd not 16-byte aligned");
  junction_mean_kernel<false><<<(E + 7) / 8, 256, 0, stream>>>(x, upd, order, tgt_sorted, E, D, D);
  return check_launch("junction_mean_varlen");
}

int lgb200_junction_sum(float* x, const float* src, const int* order, const int* tgt_sorted, int E, int D, int ld,
                        cudaStream_t stream) {
  LGB_REQUIRE(x && src && order && tgt_sorted, kErrInvalid, "junction_sum: null pointer");
  LGB_REQUIRE(E > 0 && E % 2 == 0 && D > 0 && D % 4 == 0 && ld >= 2 * D && ld % 4 == 0, kErrInvalid,
              "junction_sum: bad extents E=%d D=%d ld=%d", E, D, ld);
  LGB_REQUIRE(((uintptr_t)x | (uintptr_t)src) % 16 == 0, kErrInvalid, "junction_sum: x / src not 16-byte aligned");
  junction_mean_kernel<true><<<(E + 7) / 8, 256, 0, stream>>>(x, src, order, tgt_sorted, E, D, ld);
  return check_launch("junction_sum");
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

size_t lgb200_sinkhorn_varlen_ws_bytes(int G, int M, int N) { return 4 * skv_ws_floats(G, M, N); }

int lgb200_sinkhorn_varlen(const float* sim, const float* alpha_dev, int iters, float* out, void* ws, const int* pairs,
                           int G, int M, int N, int Mo, int No, cudaStream_t stream) {
  LGB_REQUIRE(sim && alpha_dev && out && ws && pairs, kErrInvalid, "sinkhorn_varlen: null pointer");
  LGB_REQUIRE(G > 0 && M > 0 && N > 0 && Mo > 0 && No > 0 && iters >= 0, kErrInvalid,
              "sinkhorn_varlen: bad arguments G=%d M=%d N=%d Mo=%d No=%d iters=%d", G, M, N, Mo, No, iters);
  const size_t items = (size_t)G * ((M + kSkvRows - 1) / kSkvRows);
  // ws layout: [item table][first items G + 1][barrier][u][v][pm][ps]; the int2 table first keeps it aligned
  int2* tab = static_cast<int2*>(ws);
  int* start = reinterpret_cast<int*>(tab + items);
  unsigned* bar = reinterpret_cast<unsigned*>(start + G + 1);
  float* u = reinterpret_cast<float*>(bar + 1);
  float* v = u + (size_t)G * (M + 1);
  float* pm = v + (size_t)G * (N + 1);
  float* ps = pm + items * (N + 1);
  sk_varlen_items_kernel<<<1, 1024, 0, stream>>>(pairs, G, M, N, tab, start, bar);
  if (int rc = check_launch("sinkhorn_varlen")) return rc;
  SkPlan p{};
  const int nsm = device_sm_count();
  p.grid = items < (size_t)nsm ? (int)items : nsm;
  const size_t smem = ((size_t)sk_pad(N + 1) + sk_pad(kSkvRows + 1)) * 4;
  SkvGeom q{pairs, tab, start, G, M, N, Mo, No};
  void* args[] = {&sim, &alpha_dev, &iters, &out, &u, &v, &pm, &ps, &bar, &q};
  return sk_launch((const void*)sk_fwd_varlen_kernel, p, smem, args, stream, "sinkhorn_varlen");
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

int lgb200_ot_nll_fwd_sparse(const float* Z, const int64_t* gt0, const int64_t* gt1, const float* neg0,
                             const float* neg1, float* pos, float* neg, void* ws, int B, int M, int N,
                             cudaStream_t stream) {
  LGB_REQUIRE(Z && gt0 && gt1 && neg0 && neg1 && pos && neg && ws, kErrInvalid, "ot_nll_fwd_sparse: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "ot_nll_fwd_sparse: empty input");
  const int nparts = (M + kOtRows - 1) / kOtRows;
  float* part = static_cast<float*>(ws);
  ot_nll_part_sparse_kernel<<<dim3(nparts, B), 256, 0, stream>>>(Z, gt0, gt1, part, M, N);
  if (int rc = check_launch("ot_nll_fwd_sparse")) return rc;
  ot_nll_final_kernel<<<B, 256, 0, stream>>>(Z, neg0, neg1, part, nparts, pos, neg, M, N);
  return check_launch("ot_nll_fwd_sparse");
}

int lgb200_ot_nll_bwd_sparse(const int64_t* gt0, const float* neg0, const float* neg1, const float* num_pos,
                             const float* num_neg, const float* gpos, const float* gneg, float* dZ, int B, int M, int N,
                             cudaStream_t stream) {
  LGB_REQUIRE(gt0 && neg0 && neg1 && num_pos && num_neg && gpos && gneg && dZ, kErrInvalid,
              "ot_nll_bwd_sparse: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "ot_nll_bwd_sparse: empty input");
  ot_nll_bwd_sparse_kernel<<<dim3((M + 1 + kOtRows - 1) / kOtRows, B), 256, 0, stream>>>(gt0, neg0, neg1, num_pos,
                                                                                        num_neg, gpos, gneg, dZ, M, N);
  return check_launch("ot_nll_bwd_sparse");
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
