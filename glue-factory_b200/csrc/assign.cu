// Assignment head kernels: sigmoid_log_double_softmax, deep-supervision NLL
// terms, row/col argmax and match filtering -- the HBM-bound part of the
// LightGlue matcher (reference: gluefactory/models/matchers/lightglue.py:256-309,
// gluefactory/models/utils/losses.py:6-73).
//
// Layout: sim [B,M,N] fp32 row-major.  A CTA of 256 threads (8 warps) owns a
// strip of 32 consecutive rows and walks it in 128-column chunks; lane l of a
// warp owns 4 consecutive columns (one 128-bit load), warp w owns rows
// w, w+8, w+16, w+24 of the strip.  Row statistics stay in registers and are
// reduced with warp shuffles; column statistics are reduced across the 8 warps
// through shared memory and written as per-strip partials that a tiny second
// kernel merges in strip order (deterministic, no atomics).
#include <math.h>

#include "common.cuh"
#include "lgb200.h"

namespace lgb {

constexpr int kStripRows = 32;
constexpr int kChunk = 128;
constexpr int kWarps = 8;
constexpr int kRowsPerWarp = kStripRows / kWarps;  // 4
constexpr float kNegInf = -INFINITY;

__device__ __forceinline__ float4 ld4(const float* p, bool vec, int valid) {
  // loads up to 4 floats starting at p; lanes beyond `valid` are -inf
  float4 r;
  if (vec && valid >= 4) {
    r = *reinterpret_cast<const float4*>(p);
  } else {
    r.x = valid > 0 ? p[0] : kNegInf;
    r.y = valid > 1 ? p[1] : kNegInf;
    r.z = valid > 2 ? p[2] : kNegInf;
    r.w = valid > 3 ? p[3] : kNegInf;
  }
  return r;
}

// Varlen batches (the packed evaluation head of LightGlue's adaptive / ragged inference): the kernels below are
// instantiated a second time with kVarlen = true.  Pair g < G then has its own extents m = pairs[g] <= M and
// n = pairs[G + g] <= N inside the padded [G, M, N] operands (M and N become strides; rows / columns past a pair's
// extents are never read), and its scores, matches and scores of matches go to batch row pairs[2G + g] of the outputs
// at the original keypoint indices ind0[g * M + i] / ind1[g * N + j].  Per pair, every value is computed by the same
// instructions in the same order as a uniform call on [1, m, n].
struct VarlenPairs {
  const int* pairs;  // [3, G]: m, n, output batch row
  const int* ind0;   // [G, M]
  const int* ind1;   // [G, N]
  int G, Mo, No;     // outputs: scores [*, Mo + 1, No + 1], m0 / ms0 [*, Mo], m1 / ms1 [*, No]
};

// ---------------------------------------------------------------------------------------------
// pass 1: row LSE (final) and per-strip column (max, sumexp) partials
// ---------------------------------------------------------------------------------------------
template <bool kVarlen>
__global__ void __launch_bounds__(256) assign_lse_kernel(const float* __restrict__ sim, float* __restrict__ lse_row,
                                                        float* __restrict__ colpart_m,
                                                        float* __restrict__ colpart_s, int M, int N, int nstrips,
                                                        VarlenPairs vp) {
  __shared__ float s_cmax[2][kWarps][kChunk];
  __shared__ float s_csum[2][kWarps][kChunk];
  const int b = blockIdx.y, strip = blockIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec = (N & 3) == 0;
  const float* base = sim + (int64_t)b * M * N;
  int Mb = M, Nb = N;  // this pair's extents; M, N are the strides
  if constexpr (kVarlen) {
    Mb = min(vp.pairs[b], M);
    Nb = min(vp.pairs[vp.G + b], N);
    if (strip * kStripRows >= Mb) return;
  }

  float rm[kRowsPerWarp], rs[kRowsPerWarp];
  int rows[kRowsPerWarp];
#pragma unroll
  for (int t = 0; t < kRowsPerWarp; ++t) {
    rm[t] = kNegInf;
    rs[t] = 0.f;
    rows[t] = strip * kStripRows + w + kWarps * t;
  }
  auto load_chunk = [&](int c0, float4* dst) {
    const int col = c0 + lane * 4;
    const int valid = min(4, Nb - col);  // may be <= 0
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t)
      dst[t] = (rows[t] < Mb && valid > 0) ? ld4(base + (int64_t)rows[t] * N + col, vec, valid)
                                           : make_float4(kNegInf, kNegInf, kNegInf, kNegInf);
  };
  int buf = 0;
  float4 xn[kRowsPerWarp];
  load_chunk(0, xn);
  for (int c0 = 0; c0 < Nb; c0 += kChunk, buf ^= 1) {
    float4 x[kRowsPerWarp];
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) x[t] = xn[t];
    if (c0 + kChunk < Nb) load_chunk(c0 + kChunk, xn);  // next chunk in flight while this one is reduced
    // ---- row statistics (online, rescale only when the running max moves)
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) {
      float cm = fmaxf(fmaxf(x[t].x, x[t].y), fmaxf(x[t].z, x[t].w));
      if (cm > rm[t]) {
        rs[t] *= __expf(rm[t] - cm);  // rm=-inf -> exp(-inf)=0, rs is 0 anyway
        rm[t] = cm;
      }
      const float ref = (rm[t] == kNegInf) ? 0.f : rm[t];
      rs[t] += (__expf(x[t].x - ref) + __expf(x[t].y - ref)) + (__expf(x[t].z - ref) + __expf(x[t].w - ref));
    }
    // ---- column statistics of this strip: max first (no exp), then one exp per element
    float4 cm4;
    cm4.x = fmaxf(fmaxf(x[0].x, x[1].x), fmaxf(x[2].x, x[3].x));
    cm4.y = fmaxf(fmaxf(x[0].y, x[1].y), fmaxf(x[2].y, x[3].y));
    cm4.z = fmaxf(fmaxf(x[0].z, x[1].z), fmaxf(x[2].z, x[3].z));
    cm4.w = fmaxf(fmaxf(x[0].w, x[1].w), fmaxf(x[2].w, x[3].w));
    *reinterpret_cast<float4*>(&s_cmax[buf][w][lane * 4]) = cm4;
    __syncthreads();
    float4 mx = *reinterpret_cast<float4*>(&s_cmax[buf][0][lane * 4]);
#pragma unroll
    for (int ww = 1; ww < kWarps; ++ww) {
      float4 o = *reinterpret_cast<float4*>(&s_cmax[buf][ww][lane * 4]);
      mx.x = fmaxf(mx.x, o.x); mx.y = fmaxf(mx.y, o.y); mx.z = fmaxf(mx.z, o.z); mx.w = fmaxf(mx.w, o.w);
    }
    float4 rf;  // reference (0 when the whole strip column is -inf)
    rf.x = mx.x == kNegInf ? 0.f : mx.x; rf.y = mx.y == kNegInf ? 0.f : mx.y;
    rf.z = mx.z == kNegInf ? 0.f : mx.z; rf.w = mx.w == kNegInf ? 0.f : mx.w;
    float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) {
      cs.x += __expf(x[t].x - rf.x); cs.y += __expf(x[t].y - rf.y);
      cs.z += __expf(x[t].z - rf.z); cs.w += __expf(x[t].w - rf.w);
    }
    *reinterpret_cast<float4*>(&s_csum[buf][w][lane * 4]) = cs;
    __syncthreads();
    if (threadIdx.x < kChunk && c0 + threadIdx.x < Nb) {
      float m = s_cmax[buf][0][threadIdx.x], s = s_csum[buf][0][threadIdx.x];
#pragma unroll
      for (int ww = 1; ww < kWarps; ++ww) {
        m = fmaxf(m, s_cmax[buf][ww][threadIdx.x]);
        s += s_csum[buf][ww][threadIdx.x];
      }
      const int64_t o = ((int64_t)b * nstrips + strip) * N + c0 + threadIdx.x;
      colpart_m[o] = m;
      colpart_s[o] = s;
    }
  }
#pragma unroll
  for (int t = 0; t < kRowsPerWarp; ++t) {
    float m = rm[t], s = rs[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, m2, s2);
    }
    if (lane == 0 && rows[t] < Mb) lse_row[(int64_t)b * M + rows[t]] = m + logf(s);
  }
}

// 32 columns x 8 strip-groups per CTA: max pass (no exp), then one exp per partial; groups merged through smem
template <bool kVarlen>
__global__ void __launch_bounds__(256) assign_col_lse_merge_kernel(const float* __restrict__ colpart_m,
                                                                  const float* __restrict__ colpart_s,
                                                                  float* __restrict__ lse_col, int N, int nstrips,
                                                                  VarlenPairs vp) {
  __shared__ float s_a[8][33];
  const int b = blockIdx.y, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + tx;
  int Nb = N, ns = nstrips;  // this pair's columns and strips; N, nstrips are the strides
  if constexpr (kVarlen) {
    Nb = min(vp.pairs[vp.G + b], N);
    ns = (min(vp.pairs[b], nstrips * kStripRows) + kStripRows - 1) / kStripRows;
    if (blockIdx.x * 32 >= Nb) return;
  }
  const bool ok = j < Nb;
  const float* pm = colpart_m + (int64_t)b * nstrips * N + (ok ? j : 0);
  const float* ps = colpart_s + (int64_t)b * nstrips * N + (ok ? j : 0);
  float m = kNegInf;
  for (int st = ty; st < ns; st += 8) m = fmaxf(m, pm[(int64_t)st * N]);
  s_a[ty][tx] = m;
  __syncthreads();
  float gm = s_a[0][tx];
#pragma unroll
  for (int g = 1; g < 8; ++g) gm = fmaxf(gm, s_a[g][tx]);
  const float ref = (gm == kNegInf) ? 0.f : gm;
  float sum = 0.f;
  for (int st = ty; st < ns; st += 8) sum += ps[(int64_t)st * N] * __expf(pm[(int64_t)st * N] - ref);
  __syncthreads();
  s_a[ty][tx] = sum;
  __syncthreads();
  if (ty == 0 && ok) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) t += s_a[g][tx];  // fixed order: deterministic
    lse_col[(int64_t)b * N + j] = gm + logf(t);
  }
}

// ---------------------------------------------------------------------------------------------
// pass 2: scores (optional dense write), row/col max+argmax, positive-weighted sums
// ---------------------------------------------------------------------------------------------
struct ScoreArgs {
  const float* sim;
  const float* lse_row;
  const float* lse_col;
  const float* ls0;   // log sigmoid(z0)   [B,M]
  const float* ls1;   // log sigmoid(z1)   [B,N]
  const float* dust0; // log sigmoid(-z0)  [B,M]  (dustbin column)
  const float* dust1; // log sigmoid(-z1)  [B,N]  (dustbin row)
  const uint8_t* gt;  // [B,M,N] or null
  float* scores;      // [B,M+1,N+1] or null
  float* rowmax; int* rowarg;       // [B,M]
  float* colpart_v; int* colpart_i; // [B,nstrips,N]
  float* pos_row_sum;  // [B,M] or null : sum_j gt_ij * (2 sim_ij - lse_row_i - lse_col_j)
  float* row_expsum;   // [B,M] or null : sum_{j<=N} exp(scores_ij)
  int M, N, nstrips;
};

__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

template <bool kVarlen>
__global__ void __launch_bounds__(256) assign_scores_kernel(ScoreArgs a, VarlenPairs vp) {
  __shared__ float s_v[2][kWarps][kChunk];
  __shared__ int s_i[2][kWarps][kChunk];
  const int b = blockIdx.y, strip = blockIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int M = a.M, N = a.N;
  const bool vec = (N & 3) == 0;
  const float* base = a.sim + (int64_t)b * M * N;
  const uint8_t* gbase = a.gt ? a.gt + (int64_t)b * M * N : nullptr;
  int Mb = M, Nb = N;  // this pair's extents; M, N are the strides
  float* sbase = nullptr;  // varlen: row 0 of this pair's scores in the output batch
  if constexpr (kVarlen) {
    Mb = min(vp.pairs[b], M);
    Nb = min(vp.pairs[vp.G + b], N);
    if (strip * kStripRows >= Mb) return;
    if (a.scores) sbase = a.scores + (int64_t)vp.pairs[2 * vp.G + b] * (vp.Mo + 1) * (vp.No + 1);
  }

  int rows[kRowsPerWarp];
  float lr[kRowsPerWarp], l0[kRowsPerWarp], bestv[kRowsPerWarp], psum[kRowsPerWarp], esum[kRowsPerWarp];
  int besti[kRowsPerWarp];
  int64_t orow[kRowsPerWarp];  // varlen: offset of the row's original index in the output scores
#pragma unroll
  for (int t = 0; t < kRowsPerWarp; ++t) {
    rows[t] = strip * kStripRows + w + kWarps * t;
    const bool ok = rows[t] < Mb;
    lr[t] = ok ? a.lse_row[(int64_t)b * M + rows[t]] : 0.f;
    l0[t] = ok ? a.ls0[(int64_t)b * M + rows[t]] : 0.f;
    bestv[t] = kNegInf;
    besti[t] = 0x7fffffff;
    psum[t] = 0.f;
    esum[t] = 0.f;
    if constexpr (kVarlen) orow[t] = ok ? (int64_t)vp.ind0[(int64_t)b * M + rows[t]] * (vp.No + 1) : 0;
  }
  auto load_chunk = [&](int c0, float4* dx, uint32_t* dg) {
    const int col = c0 + lane * 4;
    const int valid = min(4, Nb - col);
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) {
      dx[t] = make_float4(kNegInf, kNegInf, kNegInf, kNegInf);
      dg[t] = 0;
      if (rows[t] >= Mb || valid <= 0) continue;
      const int64_t roff = (int64_t)rows[t] * N + col;
      dx[t] = ld4(base + roff, vec, valid);
      if (gbase) {
        if (vec && valid >= 4) dg[t] = *reinterpret_cast<const uint32_t*>(gbase + roff);
        else
          for (int e = 0; e < valid; ++e) dg[t] |= (uint32_t)gbase[roff + e] << (8 * e);
      }
    }
  };
  int buf = 0;
  float4 xn[kRowsPerWarp];
  uint32_t gn[kRowsPerWarp];
  load_chunk(0, xn, gn);
  for (int c0 = 0; c0 < Nb; c0 += kChunk, buf ^= 1) {
    const int col = c0 + lane * 4;
    const int valid = min(4, Nb - col);
    float4 xc[kRowsPerWarp];
    uint32_t gc[kRowsPerWarp];
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) { xc[t] = xn[t]; gc[t] = gn[t]; }
    if (c0 + kChunk < Nb) load_chunk(c0 + kChunk, xn, gn);  // next chunk in flight while this one is processed
    float lc[4], l1[4];
    int ocol[4];  // varlen: the columns' original indices
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      lc[e] = e < valid ? a.lse_col[(int64_t)b * N + col + e] : 0.f;
      l1[e] = e < valid ? a.ls1[(int64_t)b * N + col + e] : 0.f;
      if constexpr (kVarlen) ocol[e] = e < valid ? vp.ind1[(int64_t)b * N + col + e] : 0;
    }
    float cbv[4];
    int cbi[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) { cbv[e] = kNegInf; cbi[e] = 0x7fffffff; }
#pragma unroll
    for (int t = 0; t < kRowsPerWarp; ++t) {
      if (rows[t] >= Mb || valid <= 0) continue;
      const float x[4] = {xc[t].x, xc[t].y, xc[t].z, xc[t].w};
      const uint32_t g = gc[t];
      float sc[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // same association as the reference: (log_softmax_row + log_softmax_col) + (lsig0 + lsig1)
        sc[e] = ((x[e] - lr[t]) + (x[e] - lc[e])) + (l0[t] + l1[e]);
        if (e < valid) {
          if (sc[e] > bestv[t]) { bestv[t] = sc[e]; besti[t] = col + e; }
          if (better(sc[e], rows[t], cbv[e], cbi[e])) { cbv[e] = sc[e]; cbi[e] = rows[t]; }
          if ((g >> (8 * e)) & 0xffu) psum[t] += (x[e] - lr[t]) + (x[e] - lc[e]);
          if (a.row_expsum) esum[t] += __expf(sc[e]);
        }
      }
      if constexpr (kVarlen) {
        if (sbase) {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (e < valid) sbase[orow[t] + ocol[e]] = sc[e];
        }
      } else if (a.scores) {
        float* o = a.scores + ((int64_t)b * (M + 1) + rows[t]) * (N + 1) + col;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (e < valid) o[e] = sc[e];
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) { s_v[buf][w][lane * 4 + e] = cbv[e]; s_i[buf][w][lane * 4 + e] = cbi[e]; }
    __syncthreads();
    if (threadIdx.x < kChunk && c0 + threadIdx.x < Nb) {
      float v = s_v[buf][0][threadIdx.x];
      int i = s_i[buf][0][threadIdx.x];
#pragma unroll
      for (int ww = 1; ww < kWarps; ++ww) {
        float v2 = s_v[buf][ww][threadIdx.x];
        int i2 = s_i[buf][ww][threadIdx.x];
        if (better(v2, i2, v, i)) { v = v2; i = i2; }
      }
      const int64_t o = ((int64_t)b * a.nstrips + strip) * N + c0 + threadIdx.x;
      a.colpart_v[o] = v;
      a.colpart_i[o] = i;
    }
    // s_v/s_i[buf] are rewritten two chunks later, after the next __syncthreads
  }
#pragma unroll
  for (int t = 0; t < kRowsPerWarp; ++t) {
    float v = bestv[t];
    int i = besti[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float v2 = __shfl_xor_sync(0xffffffffu, v, o);
      int i2 = __shfl_xor_sync(0xffffffffu, i, o);
      if (better(v2, i2, v, i)) { v = v2; i = i2; }
    }
    float ps = warp_sum(psum[t]);
    float es = a.row_expsum ? warp_sum(esum[t]) : 0.f;
    if (lane == 0 && rows[t] < Mb) {
      const int64_t r = (int64_t)b * M + rows[t];
      a.rowmax[r] = v;
      a.rowarg[r] = i;
      if (a.pos_row_sum) a.pos_row_sum[r] = ps;
      const float d0 = a.dust0[r];
      if (a.row_expsum) a.row_expsum[r] = es + __expf(d0);
      if constexpr (kVarlen) {
        if (sbase) sbase[orow[t] + vp.No] = d0;
      } else if (a.scores) {
        a.scores[((int64_t)b * (M + 1) + rows[t]) * (N + 1) + N] = d0;
      }
    }
  }
}

template <bool kVarlen>
__global__ void __launch_bounds__(256) assign_col_arg_merge_kernel(const float* __restrict__ colpart_v,
                                                                  const int* __restrict__ colpart_i,
                                                                  const float* __restrict__ dust1,
                                                                  float* __restrict__ colmax, int* __restrict__ colarg,
                                                                  float* __restrict__ scores, int M, int N,
                                                                  int nstrips, VarlenPairs vp) {
  __shared__ float s_v[8][33];
  __shared__ int s_i[8][33];
  const int b = blockIdx.y, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + tx;
  int Nb = N, ns = nstrips;  // this pair's columns and strips; N, nstrips are the strides
  if constexpr (kVarlen) {
    Nb = min(vp.pairs[vp.G + b], N);
    ns = (min(vp.pairs[b], M) + kStripRows - 1) / kStripRows;
    if (blockIdx.x * 32 > Nb) return;
  }
  float v = kNegInf;
  int i = 0x7fffffff;
  if (j < Nb) {
    for (int st = ty; st < ns; st += 8) {
      const int64_t o = ((int64_t)b * nstrips + st) * N + j;
      const float v2 = colpart_v[o];
      const int i2 = colpart_i[o];
      if (better(v2, i2, v, i)) { v = v2; i = i2; }
    }
  }
  s_v[ty][tx] = v;
  s_i[ty][tx] = i;
  __syncthreads();
  if (ty != 0 || j > Nb) return;
  float* srow = scores;  // varlen: the dustbin row of this pair in the output batch
  if constexpr (kVarlen) {
    if (scores) srow = scores + ((int64_t)vp.pairs[2 * vp.G + b] * (vp.Mo + 1) + vp.Mo) * (vp.No + 1);
  }
  if (j == Nb) {
    if constexpr (kVarlen) {
      if (scores) srow[vp.No] = 0.f;
    } else if (scores) {
      scores[((int64_t)b * (M + 1) + M) * (N + 1) + N] = 0.f;
    }
    return;
  }
#pragma unroll
  for (int g = 1; g < 8; ++g)
    if (better(s_v[g][tx], s_i[g][tx], v, i)) { v = s_v[g][tx]; i = s_i[g][tx]; }
  colmax[(int64_t)b * N + j] = v;
  colarg[(int64_t)b * N + j] = i;
  if constexpr (kVarlen) {
    if (scores) srow[vp.ind1[(int64_t)b * N + j]] = dust1[(int64_t)b * N + j];
  } else if (scores) {
    scores[((int64_t)b * (M + 1) + M) * (N + 1) + j] = dust1[(int64_t)b * N + j];
  }
}

// ---------------------------------------------------------------------------------------------
// backward of S_pos(sim) = sum_ij gt_ij (2 sim_ij - lse_row_i - lse_col_j):
//   dsim_ij = 2 c_b gt_ij - exp(sim_ij - lse_row_i) a_row_i - exp(sim_ij - lse_col_j) a_col_j
// (SURVEY.md Appendix A.4; here a_row_i = c_b * rowcount_i(gt), a_col_j = c_b * colcount_j(gt): the
//  kernel takes the counts and applies c_b itself)
// GtT = uint8_t: gt is the [B,M,N] byte mask.  GtT = int64_t: gt is the match list gt_matches0 [B,M] (one-to-one
// labels), and gt_ij = (gt[i] == j); every other instruction is the same, so dsim is bit-identical to the mask's.
// ---------------------------------------------------------------------------------------------
template <typename OutT, typename GtT>
__global__ void __launch_bounds__(256) assign_bwd_kernel(const float* __restrict__ sim,
                                                        const float* __restrict__ lse_row,
                                                        const float* __restrict__ lse_col,
                                                        const GtT* __restrict__ gt, const float* __restrict__ gcoef,
                                                        const float* __restrict__ a_row,
                                                        const float* __restrict__ a_col, OutT* __restrict__ dsim, int M,
                                                        int N) {
  const int b = blockIdx.y;
  const int row = blockIdx.x * kWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const bool vec = (N & 3) == 0;
  const float gc = gcoef[b];
  const float c2 = 2.f * gc;
  const float lr = lse_row[(int64_t)b * M + row];
  const float ar = gc * a_row[(int64_t)b * M + row];
  const int64_t roff = ((int64_t)b * M + row) * N;
  int64_t jpos = -1;
  if constexpr (sizeof(GtT) == 8) jpos = gt[(int64_t)b * M + row];
  for (int col = lane * 4; col < N; col += 128) {
    const int valid = min(4, N - col);
    float4 x4 = ld4(sim + roff + col, vec, valid);
    float x[4] = {x4.x, x4.y, x4.z, x4.w};
    uint32_t g = 0;
    if constexpr (sizeof(GtT) == 8) {
      if (jpos >= col && jpos < col + valid) g = 0xffu << (8 * (int)(jpos - col));
    } else {
      if (vec && valid >= 4) g = *reinterpret_cast<const uint32_t*>(gt + roff + col);
      else
        for (int e = 0; e < valid; ++e) g |= (uint32_t)gt[roff + col + e] << (8 * e);
    }
    float d[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      d[e] = 0.f;
      if (e < valid) {
        const float ac = gc * a_col[(int64_t)b * N + col + e];
        float v = ((g >> (8 * e)) & 0xffu) ? c2 : 0.f;
        if (ar != 0.f) v -= __expf(x[e] - lr) * ar;
        if (ac != 0.f) v -= __expf(x[e] - lse_col[(int64_t)b * N + col + e]) * ac;
        d[e] = v;
      }
    }
    OutT* o = dsim + roff + col;
    if constexpr (sizeof(OutT) == 4) {
      if (vec && valid >= 4) *reinterpret_cast<float4*>(o) = make_float4(d[0], d[1], d[2], d[3]);
      else
        for (int e = 0; e < valid; ++e) o[e] = d[e];
    } else {
      if (vec && valid >= 4) {
        uint2 p;
        p.x = pack_bf16(d[0], d[1]);
        p.y = pack_bf16(d[2], d[3]);
        *reinterpret_cast<uint2*>(o) = p;
      } else {
        for (int e = 0; e < valid; ++e) o[e] = __float2bfloat16(d[e]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Positive term from match lists: with one-to-one labels row i has its only positive at j = gt0[i] >= 0, so the
// positive part of the NLL is one entry per row and its gradient one rank-1 update per row and per column
// (no [B,M,N] mask is read).  One warp per row; every sum runs in a fixed order.
// ---------------------------------------------------------------------------------------------
// pos_row_sum_i = 2 alpha md0_i . md1_j - lse_row_i - lse_col_j   (kSim = false: bf16 operands, fp32 accumulate)
//              = (sim_ij - lse_row_i) + (sim_ij - lse_col_j)     (kSim = true: assign_scores' arithmetic, so the result
//                                                                 is bit-identical to the mask's on consistent lists)
// 0 when the row has no positive, NaN when j >= N or gt1[j] != i (the two lists disagree).
template <bool kSim>
__global__ void __launch_bounds__(256) assign_pos_fwd_kernel(const __nv_bfloat16* __restrict__ md0,
                                                            const __nv_bfloat16* __restrict__ md1,
                                                            const float* __restrict__ sim, float alpha,
                                                            const float* __restrict__ lse_row,
                                                            const float* __restrict__ lse_col,
                                                            const int64_t* __restrict__ gt0,
                                                            const int64_t* __restrict__ gt1,
                                                            float* __restrict__ pos_row_sum, int M, int N, int D) {
  const int b = blockIdx.y, i = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= M) return;
  const int64_t r = (int64_t)b * M + i;
  const int64_t j = gt0[r];  // warp-uniform: every branch below is taken by the whole warp
  float v = 0.f;
  if (j >= 0) {
    if (j >= N || gt1[(int64_t)b * N + j] != i) {
      v = NAN;
    } else {
      const float lr = lse_row[r], lc = lse_col[(int64_t)b * N + j];
      if constexpr (kSim) {
        const float x = sim[r * N + j];
        v = (x - lr) + (x - lc);
      } else {
        const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(md0 + r * D);
        const __nv_bfloat162* c = reinterpret_cast<const __nv_bfloat162*>(md1 + ((int64_t)b * N + j) * D);
        float s = 0.f;
        for (int k = lane; k < D / 2; k += 32) {
          const float2 x = __bfloat1622float2(a[k]), y = __bfloat1622float2(c[k]);
          s = fmaf(x.x, y.x, s);
          s = fmaf(x.y, y.y, s);
        }
        v = fmaf(warp_sum(s), 2.f * alpha, -lr) - lc;
      }
    }
  }
  if (lane == 0) pos_row_sum[r] = v;
}

// dmd0_i += 2 gcoef_b md1_{gt0[i]} and dmd1_j += 2 gcoef_b md0_{gt1[j]} (bf16 in place, fp32 arithmetic): the dsim =
// 2 gcoef entries at the positives, which the mask-free fused backward leaves out.  Warps [0, M) of a pair take the
// rows of image 0, warps [M, M + N) the columns of image 1; an index outside the other image adds nothing.
__global__ void __launch_bounds__(256) assign_pos_bwd_kernel(const __nv_bfloat16* __restrict__ md0,
                                                            const __nv_bfloat16* __restrict__ md1,
                                                            const float* __restrict__ gcoef,
                                                            const int64_t* __restrict__ gt0,
                                                            const int64_t* __restrict__ gt1,
                                                            __nv_bfloat16* __restrict__ dmd0,
                                                            __nv_bfloat16* __restrict__ dmd1, int M, int N, int D) {
  const int b = blockIdx.y, w = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= M + N) return;
  const bool side1 = w >= M;
  const int64_t r = side1 ? (int64_t)b * N + (w - M) : (int64_t)b * M + w;
  const int64_t k = side1 ? gt1[r] : gt0[r];
  if (k < 0 || k >= (side1 ? M : N)) return;
  const __nv_bfloat162* src =
      reinterpret_cast<const __nv_bfloat162*>(side1 ? md0 + ((int64_t)b * M + k) * D : md1 + ((int64_t)b * N + k) * D);
  __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>((side1 ? dmd1 : dmd0) + r * D);
  const float c = 2.f * gcoef[b];
  for (int e = lane; e < D / 2; e += 32) {
    const float2 s = __bfloat1622float2(src[e]), d = __bfloat1622float2(dst[e]);
    dst[e] = __floats2bfloat162_rn(fmaf(c, s.x, d.x), fmaf(c, s.y, d.y));
  }
}

template <typename GtT>
static int launch_assign_bwd(const float* sim, const float* lse_row, const float* lse_col, const GtT* gt,
                             const float* gcoef, const float* a_row, const float* a_col, void* dsim, int out_dtype,
                             int B, int M, int N, cudaStream_t stream, const char* what) {
  dim3 grid((M + kWarps - 1) / kWarps, B);
  if (out_dtype == LGB200_F32)
    assign_bwd_kernel<float, GtT><<<grid, 256, 0, stream>>>(sim, lse_row, lse_col, gt, gcoef, a_row, a_col,
                                                            static_cast<float*>(dsim), M, N);
  else if (out_dtype == LGB200_BF16)
    assign_bwd_kernel<__nv_bfloat16, GtT><<<grid, 256, 0, stream>>>(sim, lse_row, lse_col, gt, gcoef, a_row, a_col,
                                                                    static_cast<__nv_bfloat16*>(dsim), M, N);
  else
    LGB_REQUIRE(false, kErrInvalid, "%s: bad out_dtype %d", what, out_dtype);
  return check_launch(what);
}

// ---------------------------------------------------------------------------------------------
// filter_matches (lightglue.py:293-309) from the row/col argmax of pass 2
// ---------------------------------------------------------------------------------------------
template <bool kVarlen>
__global__ void filter_matches_kernel(const float* __restrict__ rowmax, const int* __restrict__ rowarg,
                                      const int* __restrict__ colarg, float th, int64_t* __restrict__ m0,
                                      int64_t* __restrict__ m1, float* __restrict__ ms0, float* __restrict__ ms1,
                                      int M, int N, VarlenPairs vp) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int* ra = rowarg + (int64_t)b * M;
  const int* ca = colarg + (int64_t)b * N;
  const float* rm = rowmax + (int64_t)b * M;
  int Mb = M, Nb = N;  // this pair's extents; M, N are the strides
  if constexpr (kVarlen) {
    Mb = min(vp.pairs[b], M);
    Nb = min(vp.pairs[vp.G + b], N);
  }
  if (t < Mb) {
    const int j = ra[t];
    const bool mutual = (j >= 0 && j < Nb) && ca[j] == t;
    const float s = mutual ? expf(rm[t]) : 0.f;
    const bool valid = mutual && s > th;
    if constexpr (kVarlen) {  // original indices of both points
      const int64_t o = (int64_t)vp.pairs[2 * vp.G + b] * vp.Mo + vp.ind0[(int64_t)b * M + t];
      m0[o] = valid ? vp.ind1[(int64_t)b * N + j] : -1;
      ms0[o] = s;
    } else {
      m0[(int64_t)b * M + t] = valid ? j : -1;
      ms0[(int64_t)b * M + t] = s;
    }
  }
  if (t < Nb) {
    const int i = ca[t];
    const bool mutual1 = (i >= 0 && i < Mb) && ra[i] == t;
    float s = 0.f;
    bool valid = false;
    if (mutual1) {
      // mutual1 implies mutual0 of row i (ca[ra[i]] == i)
      s = expf(rm[i]);
      valid = s > th;
    }
    if constexpr (kVarlen) {
      const int64_t o = (int64_t)vp.pairs[2 * vp.G + b] * vp.No + vp.ind1[(int64_t)b * N + t];
      m1[o] = valid ? vp.ind0[(int64_t)b * M + i] : -1;
      ms1[o] = s;
    } else {
      m1[(int64_t)b * N + t] = valid ? i : -1;
      ms1[(int64_t)b * N + t] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// O(M+N) terms of one supervised layer, fused: matchability log-sigmoids, the NLL of losses.py:6-25
// (given the similarity part sum_j gt_ij(2 sim - lse_r - lse_c) per row from pass 2), and the
// TokenConfidence BCE of lightglue.py:81-94.  zt holds [matchability logit, token logit] per token,
// tokens ordered [image0 (B*M); image1 (B*N)].  One CTA per pair; deterministic block reduction.
// ---------------------------------------------------------------------------------------------
struct HeadArgs {
  const float* zt;           // [T, 2]
  const float* pos_row_sum;  // [B,M]
  const float* rowcnt; const float* colcnt; const float* neg0; const float* neg1;
  const float* rowmax; const int* rowarg; const float* colmax; const int* colarg;
  const int* fin0; const int* fin1;  // final-layer argmax incl. dustbin, or null (no confidence term)
  const float* num_pos; const float* num_neg;  // [B]
  float bal;
  int B, M, N;
  float* nll; float* nll_pos; float* nll_neg; float* conf;  // [B]
};

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

// grid (chunks of 256 tokens over [side-0 rows | side-1 columns], B); per-chunk partial sums, then the last
// CTA of each pair to finish adds the partials in chunk order (deterministic) and writes the four outputs.
__global__ void __launch_bounds__(256) head_terms_fwd_kernel(HeadArgs a, float* __restrict__ part,
                                                            unsigned* __restrict__ counter) {
  __shared__ float red[8];
  __shared__ bool s_last;
  const int b = blockIdx.y, M = a.M, N = a.N;
  const int64_t t0 = (int64_t)a.B * M;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  float pos = 0.f, neg = 0.f, c0 = 0.f, c1 = 0.f;
  if (idx < M) {
    const int64_t r = (int64_t)b * M + idx;
    const float2 z = *reinterpret_cast<const float2*>(a.zt + 2 * r);
    const float ls = log_sigmoid(z.x), du = ls - z.x;
    pos = a.pos_row_sum[r] + a.rowcnt[r] * ls;
    neg = a.neg0[r] * du;
    if (a.fin0) {
      const int arg = du > a.rowmax[r] ? N : a.rowarg[r];
      const float y = (a.fin0[r] == arg) ? 1.f : 0.f;
      c0 = fmaxf(z.y, 0.f) - z.y * y + log1pf(expf(-fabsf(z.y)));
    }
  } else if (idx < M + N) {
    const int64_t r = (int64_t)b * N + (idx - M);
    const float2 z = *reinterpret_cast<const float2*>(a.zt + 2 * (t0 + r));
    const float ls = log_sigmoid(z.x), du = ls - z.x;
    pos = a.colcnt[r] * ls;
    neg = a.neg1[r] * du;
    if (a.fin1) {
      const int arg = du > a.colmax[r] ? M : a.colarg[r];
      const float y = (a.fin1[r] == arg) ? 1.f : 0.f;
      c1 = fmaxf(z.y, 0.f) - z.y * y + log1pf(expf(-fabsf(z.y)));
    }
  }
  pos = block_sum_256(pos, red);
  neg = block_sum_256(neg, red);
  c0 = block_sum_256(c0, red);
  c1 = block_sum_256(c1, red);
  const int nchunk = gridDim.x;
  if (threadIdx.x == 0) {
    float4* dst = reinterpret_cast<float4*>(part) + (int64_t)b * nchunk + blockIdx.x;
    *dst = make_float4(pos, neg, c0, c1);
    __threadfence();
    const unsigned prev = atomicAdd(&counter[b], 1u);
    s_last = (prev == (unsigned)nchunk - 1);
    if (s_last) counter[b] = 0u;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    float sp = 0.f, sn = 0.f, s0 = 0.f, s1 = 0.f;
    for (int c = 0; c < nchunk; ++c) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(part) + (int64_t)b * nchunk + c);
      sp += v.x; sn += v.y; s0 += v.z; s1 += v.w;
    }
    const float np = -sp / a.num_pos[b], nn = -sn / a.num_neg[b];
    a.nll_pos[b] = np;
    a.nll_neg[b] = nn;
    a.nll[b] = a.bal * np + (1.f - a.bal) * nn;
    a.conf[b] = a.fin0 ? 0.5f * (s0 / M + s1 / N) : 0.f;
  }
}

// d(zt) for upstream gradients g_nll[b], g_conf[b]
__global__ void __launch_bounds__(256) head_terms_bwd_kernel(HeadArgs a, const float* __restrict__ g_nll,
                                                            const float* __restrict__ g_conf,
                                                            float* __restrict__ dzt) {
  const int M = a.M, N = a.N;
  const int64_t t0 = (int64_t)a.B * M, T = t0 + (int64_t)a.B * N;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const bool side1 = t >= t0;
  const int64_t r = side1 ? t - t0 : t;
  const int L = side1 ? N : M;
  const int b = (int)(r / L);
  const float2 z = *reinterpret_cast<const float2*>(a.zt + 2 * t);
  const float g = g_nll[b];
  const float gpos = -a.bal * g / a.num_pos[b];
  const float gneg = -(1.f - a.bal) * g / a.num_neg[b];
  const float sg = 1.f / (1.f + expf(-z.x));
  const float cnt = side1 ? a.colcnt[r] : a.rowcnt[r];
  const float ng = side1 ? a.neg1[r] : a.neg0[r];
  float2 d;
  d.x = gpos * cnt * (1.f - sg) - gneg * ng * sg;
  d.y = 0.f;
  const int* fin = side1 ? a.fin1 : a.fin0;
  if (fin) {
    const float ls = log_sigmoid(z.x), du = ls - z.x;
    const float mx = side1 ? a.colmax[r] : a.rowmax[r];
    const int ag = side1 ? a.colarg[r] : a.rowarg[r];
    const int arg = du > mx ? (side1 ? M : N) : ag;
    const float y = (fin[r] == arg) ? 1.f : 0.f;
    d.y = g_conf[b] * (0.5f / L) * (1.f / (1.f + expf(-z.y)) - y);
  }
  *reinterpret_cast<float2*>(dzt + 2 * t) = d;
}

// ls = log sigmoid(z), du = log sigmoid(-z) from the strided logits (feeds pass 2)
__global__ void __launch_bounds__(256) logsig_kernel(const float* __restrict__ zt, float* __restrict__ ls,
                                                    float* __restrict__ du, int64_t T) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const float z = zt[2 * t];
  const float l = log_sigmoid(z);
  ls[t] = l;
  du[t] = l - z;
}

}  // namespace lgb

using namespace lgb;

extern "C" {

int lgb200_head_logsig(const float* zt, float* ls, float* du, int64_t T, cudaStream_t stream) {
  LGB_REQUIRE(zt && ls && du && T > 0, kErrInvalid, "head_logsig: bad arguments");
  logsig_kernel<<<(unsigned)((T + 255) / 256), 256, 0, stream>>>(zt, ls, du, T);
  return check_launch("head_logsig");
}

static int fill_head_args(HeadArgs& a, const float* zt, const float* pos_row_sum, const float* rowcnt,
                          const float* colcnt, const float* neg0, const float* neg1, const float* rowmax,
                          const int* rowarg, const float* colmax, const int* colarg, const int* fin0, const int* fin1,
                          const float* num_pos, const float* num_neg, float bal, int B, int M, int N) {
  LGB_REQUIRE(zt && pos_row_sum && rowcnt && colcnt && neg0 && neg1 && rowmax && rowarg && colmax && colarg &&
                  num_pos && num_neg,
              kErrInvalid, "head_terms: null pointer");
  LGB_REQUIRE((fin0 == nullptr) == (fin1 == nullptr), kErrInvalid, "head_terms: fin0/fin1 must both be set or null");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "head_terms: empty input");
  a.zt = zt; a.pos_row_sum = pos_row_sum; a.rowcnt = rowcnt; a.colcnt = colcnt; a.neg0 = neg0; a.neg1 = neg1;
  a.rowmax = rowmax; a.rowarg = rowarg; a.colmax = colmax; a.colarg = colarg; a.fin0 = fin0; a.fin1 = fin1;
  a.num_pos = num_pos; a.num_neg = num_neg; a.bal = bal; a.B = B; a.M = M; a.N = N;
  a.nll = a.nll_pos = a.nll_neg = a.conf = nullptr;
  return 0;
}

int lgb200_head_terms_fwd(const float* zt, const float* pos_row_sum, const float* rowcnt, const float* colcnt,
                          const float* neg0, const float* neg1, const float* rowmax, const int* rowarg,
                          const float* colmax, const int* colarg, const int* fin0, const int* fin1,
                          const float* num_pos, const float* num_neg, float bal, float* nll, float* nll_pos,
                          float* nll_neg, float* conf, float* ws, unsigned* counters, int B, int M, int N,
                          cudaStream_t stream) {
  HeadArgs a;
  int rc = fill_head_args(a, zt, pos_row_sum, rowcnt, colcnt, neg0, neg1, rowmax, rowarg, colmax, colarg, fin0, fin1,
                          num_pos, num_neg, bal, B, M, N);
  if (rc) return rc;
  LGB_REQUIRE(nll && nll_pos && nll_neg && conf && ws && counters, kErrInvalid, "head_terms_fwd: null output");
  a.nll = nll; a.nll_pos = nll_pos; a.nll_neg = nll_neg; a.conf = conf;
  head_terms_fwd_kernel<<<dim3((M + N + 255) / 256, B), 256, 0, stream>>>(a, ws, counters);
  return check_launch("head_terms_fwd");
}

int lgb200_head_terms_bwd(const float* zt, const float* rowcnt, const float* colcnt, const float* neg0,
                          const float* neg1, const float* rowmax, const int* rowarg, const float* colmax,
                          const int* colarg, const int* fin0, const int* fin1, const float* num_pos,
                          const float* num_neg, float bal, const float* g_nll, const float* g_conf, float* dzt, int B,
                          int M, int N, cudaStream_t stream) {
  HeadArgs a;
  int rc = fill_head_args(a, zt, rowcnt /*unused*/, rowcnt, colcnt, neg0, neg1, rowmax, rowarg, colmax, colarg, fin0,
                          fin1, num_pos, num_neg, bal, B, M, N);
  if (rc) return rc;
  LGB_REQUIRE(g_nll && g_conf && dzt, kErrInvalid, "head_terms_bwd: null pointer");
  const int64_t T = (int64_t)B * (M + N);
  head_terms_bwd_kernel<<<(unsigned)((T + 255) / 256), 256, 0, stream>>>(a, g_nll, g_conf, dzt);
  return check_launch("head_terms_bwd");
}

size_t lgb200_assign_ws_bytes(int B, int M, int N) {
  const int nstrips = (M + kStripRows - 1) / kStripRows;
  return (size_t)B * nstrips * N * 8;
}

int lgb200_assign_lse(const float* sim, float* lse_row, float* lse_col, void* ws, int B, int M, int N,
                      cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && ws, kErrInvalid, "assign_lse: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_lse: empty input B=%d M=%d N=%d", B, M, N);
  const int nstrips = (M + kStripRows - 1) / kStripRows;
  float* pm = static_cast<float*>(ws);
  float* ps = pm + (size_t)B * nstrips * N;
  assign_lse_kernel<false><<<dim3(nstrips, B), 256, 0, stream>>>(sim, lse_row, pm, ps, M, N, nstrips, VarlenPairs{});
  assign_col_lse_merge_kernel<false><<<dim3((N + 31) / 32, B), 256, 0, stream>>>(pm, ps, lse_col, N, nstrips,
                                                                                 VarlenPairs{});
  return check_launch("assign_lse");
}

int lgb200_assign_scores(const float* sim, const float* lse_row, const float* lse_col, const float* ls0,
                         const float* ls1, const float* dust0, const float* dust1, const uint8_t* gt, float* scores,
                         float* rowmax, int* rowarg, float* colmax, int* colarg, float* pos_row_sum,
                         float* row_expsum, void* ws, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && ls0 && ls1 && dust0 && dust1 && rowmax && rowarg && colmax && colarg && ws,
              kErrInvalid, "assign_scores: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_scores: empty input");
  LGB_REQUIRE(!pos_row_sum || gt, kErrInvalid, "assign_scores: pos_row_sum requested without gt");
  const int nstrips = (M + kStripRows - 1) / kStripRows;
  ScoreArgs a;
  a.sim = sim; a.lse_row = lse_row; a.lse_col = lse_col; a.ls0 = ls0; a.ls1 = ls1; a.dust0 = dust0; a.dust1 = dust1;
  a.gt = gt; a.scores = scores; a.rowmax = rowmax; a.rowarg = rowarg;
  a.colpart_v = static_cast<float*>(ws);
  a.colpart_i = reinterpret_cast<int*>(a.colpart_v + (size_t)B * nstrips * N);
  a.pos_row_sum = pos_row_sum; a.row_expsum = row_expsum; a.M = M; a.N = N; a.nstrips = nstrips;
  assign_scores_kernel<false><<<dim3(nstrips, B), 256, 0, stream>>>(a, VarlenPairs{});
  assign_col_arg_merge_kernel<false><<<dim3((N + 1 + 31) / 32, B), 256, 0, stream>>>(
      a.colpart_v, a.colpart_i, dust1, colmax, colarg, scores, M, N, nstrips, VarlenPairs{});
  return check_launch("assign_scores");
}

int lgb200_assign_bwd(const float* sim, const float* lse_row, const float* lse_col, const uint8_t* gt,
                      const float* gcoef, const float* a_row, const float* a_col, void* dsim, int out_dtype, int B,
                      int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && gt && gcoef && a_row && a_col && dsim, kErrInvalid,
              "assign_bwd: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_bwd: empty input");
  return launch_assign_bwd(sim, lse_row, lse_col, gt, gcoef, a_row, a_col, dsim, out_dtype, B, M, N, stream,
                           "assign_bwd");
}

int lgb200_assign_bwd_sparse(const float* sim, const float* lse_row, const float* lse_col, const int64_t* gt0,
                             const float* gcoef, const float* a_row, const float* a_col, void* dsim, int out_dtype,
                             int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && gt0 && gcoef && a_row && a_col && dsim, kErrInvalid,
              "assign_bwd_sparse: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_bwd_sparse: empty input");
  return launch_assign_bwd(sim, lse_row, lse_col, gt0, gcoef, a_row, a_col, dsim, out_dtype, B, M, N, stream,
                           "assign_bwd_sparse");
}

int lgb200_assign_pos_fwd(const void* md0, const void* md1, const float* sim, float alpha, const float* lse_row,
                          const float* lse_col, const int64_t* gt0, const int64_t* gt1, float* pos_row_sum, int B,
                          int M, int N, int D, cudaStream_t stream) {
  LGB_REQUIRE(lse_row && lse_col && gt0 && gt1 && pos_row_sum, kErrInvalid, "assign_pos_fwd: null pointer");
  LGB_REQUIRE((sim != nullptr) != (md0 != nullptr && md1 != nullptr) && (md0 == nullptr) == (md1 == nullptr),
              kErrInvalid, "assign_pos_fwd: pass either sim or both descriptor matrices");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_pos_fwd: empty input B=%d M=%d N=%d", B, M, N);
  dim3 grid((M + kWarps - 1) / kWarps, B);
  if (sim) {
    assign_pos_fwd_kernel<true><<<grid, 256, 0, stream>>>(nullptr, nullptr, sim, alpha, lse_row, lse_col, gt0, gt1,
                                                          pos_row_sum, M, N, 0);
  } else {
    LGB_REQUIRE(D > 0 && D % 2 == 0 && ((reinterpret_cast<uintptr_t>(md0) | reinterpret_cast<uintptr_t>(md1)) & 3) == 0,
                kErrInvalid, "assign_pos_fwd: descriptor width %d must be even, rows 4-byte aligned", D);
    assign_pos_fwd_kernel<false><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(md0),
                                                           static_cast<const __nv_bfloat16*>(md1), nullptr, alpha,
                                                           lse_row, lse_col, gt0, gt1, pos_row_sum, M, N, D);
  }
  return check_launch("assign_pos_fwd");
}

int lgb200_assign_pos_bwd(const void* md0, const void* md1, const float* gcoef, const int64_t* gt0, const int64_t* gt1,
                          void* dmd0, void* dmd1, int B, int M, int N, int D, cudaStream_t stream) {
  LGB_REQUIRE(md0 && md1 && gcoef && gt0 && gt1 && dmd0 && dmd1, kErrInvalid, "assign_pos_bwd: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "assign_pos_bwd: empty input B=%d M=%d N=%d", B, M, N);
  LGB_REQUIRE(D > 0 && D % 2 == 0 &&
                  ((reinterpret_cast<uintptr_t>(md0) | reinterpret_cast<uintptr_t>(md1) |
                    reinterpret_cast<uintptr_t>(dmd0) | reinterpret_cast<uintptr_t>(dmd1)) & 3) == 0,
              kErrInvalid, "assign_pos_bwd: descriptor width %d must be even, rows 4-byte aligned", D);
  assign_pos_bwd_kernel<<<dim3((M + N + kWarps - 1) / kWarps, B), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(md0), static_cast<const __nv_bfloat16*>(md1), gcoef, gt0, gt1,
      static_cast<__nv_bfloat16*>(dmd0), static_cast<__nv_bfloat16*>(dmd1), M, N, D);
  return check_launch("assign_pos_bwd");
}

int lgb200_filter_matches(const float* rowmax, const int* rowarg, const int* colarg, float th, int64_t* m0,
                          int64_t* m1, float* ms0, float* ms1, int B, int M, int N, cudaStream_t stream) {
  LGB_REQUIRE(rowmax && rowarg && colarg && m0 && m1 && ms0 && ms1, kErrInvalid, "filter_matches: null pointer");
  LGB_REQUIRE(B > 0 && M > 0 && N > 0, kErrInvalid, "filter_matches: empty input");
  const int L = M > N ? M : N;
  filter_matches_kernel<false><<<dim3((L + 255) / 256, B), 256, 0, stream>>>(rowmax, rowarg, colarg, th, m0, m1, ms0,
                                                                             ms1, M, N, VarlenPairs{});
  return check_launch("filter_matches");
}

static int varlen_pairs(VarlenPairs& vp, const int* pairs, const int* ind0, const int* ind1, int G, int M, int N, int Mo,
                        int No, const char* what) {
  LGB_REQUIRE(pairs, kErrInvalid, "%s: null pairs", what);
  LGB_REQUIRE(G > 0 && G <= 65535 && M > 0 && N > 0 && Mo > 0 && No > 0, kErrInvalid,
              "%s: bad extents G=%d M=%d N=%d Mo=%d No=%d", what, G, M, N, Mo, No);
  vp.pairs = pairs; vp.ind0 = ind0; vp.ind1 = ind1; vp.G = G; vp.Mo = Mo; vp.No = No;
  return 0;
}

int lgb200_assign_lse_varlen(const float* sim, float* lse_row, float* lse_col, void* ws, const int* pairs, int G, int M,
                             int N, cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && ws, kErrInvalid, "assign_lse_varlen: null pointer");
  VarlenPairs vp;
  int rc = varlen_pairs(vp, pairs, nullptr, nullptr, G, M, N, 1, 1, "assign_lse_varlen");
  if (rc) return rc;
  const int nstrips = (M + kStripRows - 1) / kStripRows;
  float* pm = static_cast<float*>(ws);
  float* ps = pm + (size_t)G * nstrips * N;
  assign_lse_kernel<true><<<dim3(nstrips, G), 256, 0, stream>>>(sim, lse_row, pm, ps, M, N, nstrips, vp);
  assign_col_lse_merge_kernel<true><<<dim3((N + 31) / 32, G), 256, 0, stream>>>(pm, ps, lse_col, N, nstrips, vp);
  return check_launch("assign_lse_varlen");
}

int lgb200_assign_scores_varlen(const float* sim, const float* lse_row, const float* lse_col, const float* ls0,
                                const float* ls1, const float* dust0, const float* dust1, float* scores, float* rowmax,
                                int* rowarg, float* colmax, int* colarg, float* row_expsum, void* ws, const int* pairs,
                                const int* ind0, const int* ind1, int G, int M, int N, int Mo, int No,
                                cudaStream_t stream) {
  LGB_REQUIRE(sim && lse_row && lse_col && ls0 && ls1 && dust0 && dust1 && rowmax && rowarg && colmax && colarg && ws,
              kErrInvalid, "assign_scores_varlen: null pointer");
  LGB_REQUIRE(!scores || (ind0 && ind1), kErrInvalid, "assign_scores_varlen: scores need the index maps");
  VarlenPairs vp;
  int rc = varlen_pairs(vp, pairs, ind0, ind1, G, M, N, Mo, No, "assign_scores_varlen");
  if (rc) return rc;
  const int nstrips = (M + kStripRows - 1) / kStripRows;
  ScoreArgs a;
  a.sim = sim; a.lse_row = lse_row; a.lse_col = lse_col; a.ls0 = ls0; a.ls1 = ls1; a.dust0 = dust0; a.dust1 = dust1;
  a.gt = nullptr; a.scores = scores; a.rowmax = rowmax; a.rowarg = rowarg;
  a.colpart_v = static_cast<float*>(ws);
  a.colpart_i = reinterpret_cast<int*>(a.colpart_v + (size_t)G * nstrips * N);
  a.pos_row_sum = nullptr; a.row_expsum = row_expsum; a.M = M; a.N = N; a.nstrips = nstrips;
  assign_scores_kernel<true><<<dim3(nstrips, G), 256, 0, stream>>>(a, vp);
  assign_col_arg_merge_kernel<true><<<dim3((N + 1 + 31) / 32, G), 256, 0, stream>>>(
      a.colpart_v, a.colpart_i, dust1, colmax, colarg, scores, M, N, nstrips, vp);
  return check_launch("assign_scores_varlen");
}

int lgb200_filter_matches_varlen(const float* rowmax, const int* rowarg, const int* colarg, float th, int64_t* m0,
                                 int64_t* m1, float* ms0, float* ms1, const int* pairs, const int* ind0,
                                 const int* ind1, int G, int M, int N, int Mo, int No, cudaStream_t stream) {
  LGB_REQUIRE(rowmax && rowarg && colarg && m0 && m1 && ms0 && ms1 && ind0 && ind1, kErrInvalid,
              "filter_matches_varlen: null pointer");
  VarlenPairs vp;
  int rc = varlen_pairs(vp, pairs, ind0, ind1, G, M, N, Mo, No, "filter_matches_varlen");
  if (rc) return rc;
  const int L = M > N ? M : N;
  filter_matches_kernel<true><<<dim3((L + 255) / 256, G), 256, 0, stream>>>(rowmax, rowarg, colarg, th, m0, m1, ms0,
                                                                            ms1, M, N, vp);
  return check_launch("filter_matches_varlen");
}

}  // extern "C"
