// Ground-truth LINE correspondences on the device: the O(L0 L1 npts) part of gt_line_matches_from_homography /
// gt_line_matches_from_pose_depth (gluefactory/geometry/gt_generation.py:207-558) and the per-pair linear assignment
// the reference solves on the host with scipy.optimize.linear_sum_assignment (:366-367, :515-516).
//
// The caller (ops.gt_line_matches_*) clamps the segments, projects the sampled points into the other view and passes
// [B, L, npts, 2] point arrays; this file then
//   1. samples the points of each segment (gt_line_sample_kernel; sample_pts, :164-170),
//   2. derives per-line flags: mostly outside the other image, ignored, overlap threshold (:290-302, :345-352, :460-470),
//   3. counts, for every segment pair, the sampled points of one segment that lie within dist_th of the other segment
//      and overlap it, both ways (torch_perp_dist, :173-204), without the reference's dense [B, L0, L1, npts] tensors,
//      and writes the assignment cost -c0 c1 (1e6 on unmatched / ignored rows and columns) plus mask_close,
//   4. solves the rectangular assignment per pair exactly as scipy does (one CTA per pair),
//   5. writes line_assignment and line_matches0/1 (:374-400, :524-552).
// Elementwise steps use explicitly rounded operations, so that every comparison sees the value torch's CPU ops produce.
// The perpendicular rotation follows the reference's CPU arithmetic (fma(R[j,1], c1, R[j,0] c0), torch.einsum's
// result there); on CUDA the reference rounds `centered` and `R` to fp16 first (:194-195) to save memory for its
// dense tensor, which this file does not reproduce.
#include <cuda_fp16.h>

#include "common.cuh"
#include "lgb200.h"

namespace lgb {

constexpr int kLineTile = 16;   // segments per side of a count tile (16 x 16 pairs, one per thread)
constexpr int kLsapThreads = 256;
constexpr int kFlagOut = 1, kFlagIgnore = 2, kFlagClose = 4;  // per-line flag bits

__global__ void __launch_bounds__(256) gt_line_sample_kernel(const float4* __restrict__ lines, float2* __restrict__ pts,
                                                            int64_t total, int npts) {
  const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (t >= total) return;
  const float4 s = lines[t / npts];
  const float k = (float)(t % npts), den = (float)(npts - 1);
  // lines[..., :2] + ((lines[..., 2:4] - lines[..., :2]) / (npts - 1)) * k
  const float dx = __fdiv_rn(__fsub_rn(s.z, s.x), den), dy = __fdiv_rn(__fsub_rn(s.w, s.y), den);
  pts[t] = make_float2(__fadd_rn(s.x, __fmul_rn(dx, k)), __fadd_rn(s.y, __fmul_rn(dy, k)));
}

// One thread per line of either view (view-0 lines first).  flags: kFlagOut when at least (1 - min_visibility_th) of
// the line's projected points leave the other image; kFlagIgnore for an invalid line or (depth variant) one whose
// points have valid depth less often than min_visibility_th.  thr: the count a pair must exceed (overlap_th times the
// number of visible points in the depth variant, npts * overlap_th in the homography variant).
__global__ void __launch_bounds__(256) gt_line_flags_kernel(
    const float2* __restrict__ pts0_1, const float2* __restrict__ pts1_0, const uint8_t* __restrict__ vis0,
    const uint8_t* __restrict__ vis1, const uint8_t* __restrict__ vpts0, const uint8_t* __restrict__ vpts1,
    const uint8_t* __restrict__ vline0, const uint8_t* __restrict__ vline1, float w0, float h0, float w1, float h1,
    int npts, float out_th, float min_vis, float overlap, float fixed_th, float* __restrict__ thr0,
    float* __restrict__ thr1, int* __restrict__ flags0, int* __restrict__ flags1, int L0, int L1) {
  const int b = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
  if (t >= L0 + L1) return;
  const bool side1 = t >= L0;
  const int l = side1 ? t - L0 : t;
  const int64_t line = (int64_t)b * (side1 ? L1 : L0) + l;
  const float2* p = (side1 ? pts1_0 : pts0_1) + line * npts;
  const uint8_t* vis = side1 ? vis1 : vis0;
  const uint8_t* vpts = side1 ? vpts1 : vpts0;
  const float w = side1 ? w0 : w1, h = side1 ? h0 : h1;  // the image the points were projected into
  int nout = 0, nvis = 0, nvalid = 0;
  for (int k = 0; k < npts; ++k) {
    const float2 q = p[k];
    nout += (q.x < 0.f || q.y < 0.f || q.x >= w || q.y >= h) ? 1 : 0;
    if (vis) nvis += vis[line * npts + k] ? 1 : 0;
    if (vpts) nvalid += vpts[line * npts + k] ? 1 : 0;
  }
  const float n = (float)npts;
  int f = __fdiv_rn((float)nout, n) >= out_th ? kFlagOut : 0;  // float mean (sum / n) against the fp32 threshold
  bool ignore = !(side1 ? vline1 : vline0)[line];
  if (vpts) ignore = ignore || __fdiv_rn((float)nvalid, n) < min_vis;
  f |= ignore ? kFlagIgnore : 0;
  (side1 ? flags1 : flags0)[line] = f;
  (side1 ? thr1 : thr0)[line] = vis ? __fmul_rn((float)nvis, overlap) : fixed_th;
}

struct SegFrame {
  float ex, ey, n0, n1, size;  // end point, direction / fp16(|dir|), fp16(|dir|) as float
};

__device__ __forceinline__ SegFrame seg_frame(float4 s) {
  SegFrame f;
  const float dx = __fsub_rn(s.z, s.x), dy = __fsub_rn(s.w, s.y);
  f.size = __half2float(__float2half_rn(sqrtf(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)))));  // torch.norm(dir).half()
  f.n0 = __fdiv_rn(dx, f.size);
  f.n1 = __fdiv_rn(dy, f.size);
  f.ex = s.z;
  f.ey = s.w;
  return f;
}

// point q within dist_th of the segment's line, on the segment side of its end point and not beyond its start
__device__ __forceinline__ bool close_to(const SegFrame& f, float2 q, float dist_th) {
  const float c0 = __fsub_rn(q.x, f.ex), c1 = __fsub_rn(q.y, f.ey);
  const float r0 = __fmaf_rn(f.n1, c1, __fmul_rn(f.n0, c0));
  const float r1 = __fmaf_rn(f.n0, c1, __fmul_rn(-f.n1, c0));
  return fabsf(r1) < dist_th && r0 <= 0.f && fabsf(r0) <= f.size;
}

// One 16 x 16 tile of segment pairs per CTA, one pair per thread.  c0 = points of segment l1 (projected into view 0)
// close to segment l0, c1 = points of segment l0 (projected into view 1) close to segment l1, each weighted by the
// point's visibility in the depth variant.  Writes cost = -(c0 c1) and mask_close; rows / columns with any close pair
// get kFlagClose.  Dynamic shared memory: the tile's points, point-major so that the 16 lanes of a row read 16
// consecutive float2.
__global__ void __launch_bounds__(256) gt_line_count_kernel(
    const float4* __restrict__ lines0, const float4* __restrict__ lines1, const float2* __restrict__ pts0_1,
    const float2* __restrict__ pts1_0, const uint8_t* __restrict__ vis0, const uint8_t* __restrict__ vis1,
    const float* __restrict__ thr0, const float* __restrict__ thr1, int* __restrict__ flags0, int* __restrict__ flags1,
    float dist_th, int npts, int L0, int L1, double* __restrict__ cost, uint8_t* __restrict__ mask) {
  extern __shared__ float2 s_pts[];
  float2* s_p10 = s_pts;                              // [npts][16]: points of this tile's view-1 segments, in view 0
  float2* s_p01 = s_pts + npts * kLineTile;           // [npts][16]: points of this tile's view-0 segments, in view 1
  uint8_t* s_v1 = reinterpret_cast<uint8_t*>(s_pts + 2 * npts * kLineTile);
  uint8_t* s_v0 = s_v1 + npts * kLineTile;
  const int b = blockIdx.z, base1 = blockIdx.x * kLineTile, base0 = blockIdx.y * kLineTile;
  const int tx = threadIdx.x & (kLineTile - 1), ty = threadIdx.x / kLineTile;
  const bool depth = vis0 != nullptr;
  for (int idx = threadIdx.x; idx < npts * kLineTile; idx += 256) {
    const int line = idx / npts, k = idx - line * npts;
    const int l1 = base1 + line, l0 = base0 + line;
    const int64_t o1 = ((int64_t)b * L1 + l1) * npts + k, o0 = ((int64_t)b * L0 + l0) * npts + k;
    s_p10[k * kLineTile + line] = l1 < L1 ? pts1_0[o1] : make_float2(0.f, 0.f);
    s_p01[k * kLineTile + line] = l0 < L0 ? pts0_1[o0] : make_float2(0.f, 0.f);
    s_v1[k * kLineTile + line] = depth && l1 < L1 ? vis1[o1] : 1;
    s_v0[k * kLineTile + line] = depth && l0 < L0 ? vis0[o0] : 1;
  }
  __syncthreads();
  const int l0 = base0 + ty, l1 = base1 + tx;
  if (l0 >= L0 || l1 >= L1) return;
  const SegFrame f0 = seg_frame(lines0[(int64_t)b * L0 + l0]);
  const SegFrame f1 = seg_frame(lines1[(int64_t)b * L1 + l1]);
  int c0 = 0, c1 = 0;
  for (int k = 0; k < npts; ++k) {
    c0 += (close_to(f0, s_p10[k * kLineTile + tx], dist_th) && s_v1[k * kLineTile + tx]) ? 1 : 0;
    c1 += (close_to(f1, s_p01[k * kLineTile + ty], dist_th) && s_v0[k * kLineTile + ty]) ? 1 : 0;
  }
  const int64_t r0 = (int64_t)b * L0 + l0, r1 = (int64_t)b * L1 + l1;
  bool close = (float)c1 > thr0[r0] && (float)c0 > thr1[r1];
  if (!depth) close = close && !((flags0[r0] | flags1[r1]) & kFlagOut);  // homography variant (:491-496)
  const int64_t o = r0 * L1 + l1;
  cost[o] = -(double)(c0 * c1);
  mask[o] = close ? 1 : 0;
  if (close) {
    atomicOr(flags0 + r0, kFlagClose);
    atomicOr(flags1 + r1, kFlagClose);
  }
}

// unmatched (no close partner, or mostly outside the other image) or ignored
__device__ __forceinline__ bool line_excluded(int f) { return !(f & kFlagClose) || (f & (kFlagOut | kFlagIgnore)); }

__global__ void __launch_bounds__(256) gt_line_cost_kernel(double* __restrict__ cost, const int* __restrict__ flags0,
                                                          const int* __restrict__ flags1, int L0, int L1,
                                                          int64_t total) {
  const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (t >= total) return;
  const int64_t row = t / L1;                           // b * L0 + l0
  const int64_t col = (row / L0) * L1 + (t - row * L1);  // b * L1 + l1
  if (line_excluded(flags0[row]) || line_excluded(flags1[col])) cost[t] = 1e6;
}

__device__ __forceinline__ bool lsap_better(double s, int k, double bs, int bk) { return s < bs || (s == bs && k < bk); }

// Shortest-augmenting-path rectangular assignment with scipy's (linear_sum_assignment) tie rules, one CTA per pair.
// Solves the transpose when rows > cols.  Per augmenting step every thread scans its columns of `remaining`; the
// column picked is the minimum of shortest[], preferring among equal values the last unassigned column in
// `remaining` order, else the first one -- a lexicographic minimum of (shortest, key) with
// key = -1 - position (unassigned) or position (assigned), so the reduction gives that answer in any order.
// Costs must be finite.  Shared memory: duals, path and the `remaining` permutation (see lsap_smem_bytes).
__global__ void __launch_bounds__(kLsapThreads) lsap_kernel(const double* __restrict__ cost, int rows, int cols,
                                                           int* __restrict__ row2col, int* __restrict__ col2row) {
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kWarps = kLsapThreads / 32;
  const bool tr = rows > cols;
  const int nr = tr ? cols : rows, nc = tr ? rows : cols;
  const double* C = cost + (int64_t)b * rows * cols;
  const int64_t rs = tr ? 1 : cols, cs = tr ? cols : 1;  // element (i, j) of the solved matrix at C[i rs + j cs]
  extern __shared__ double s_lsap[];
  double* v = s_lsap;             // [nc]
  double* shortest = v + nc;      // [nc]
  double* u = shortest + nc;      // [nr]
  int* path = reinterpret_cast<int*>(u + nr);  // [nc]
  int* pos = path + nc;           // [nc]: position of column j in `remaining`
  int* remaining = pos + nc;      // [nc]
  int* row4col = remaining + nc;  // [nc]
  int* col4row = row4col + nc;    // [nr]
  uint8_t* SC = reinterpret_cast<uint8_t*>(col4row + nr);  // [nc]
  uint8_t* SR = SC + nc;          // [nr]
  __shared__ double s_ws[kWarps], s_min;
  __shared__ int s_wk[kWarps], s_i, s_nrem, s_sink;
  for (int j = tid; j < nc; j += kLsapThreads) { v[j] = 0.0; row4col[j] = -1; }
  for (int i = tid; i < nr; i += kLsapThreads) { u[i] = 0.0; col4row[i] = -1; }
  for (int cur = 0; cur < nr; ++cur) {
    for (int j = tid; j < nc; j += kLsapThreads) {
      shortest[j] = INFINITY; path[j] = -1; SC[j] = 0;
      pos[j] = nc - 1 - j; remaining[j] = nc - 1 - j;
    }
    for (int i = tid; i < nr; i += kLsapThreads) SR[i] = i == cur;
    if (tid == 0) { s_i = cur; s_min = 0.0; s_nrem = nc; s_sink = -1; }
    __syncthreads();
    while (true) {
      const int i = s_i, nrem = s_nrem;
      const double minv = s_min, ui = u[i];
      double bs = INFINITY;
      int bk = 0x7fffffff;
      for (int j = tid; j < nc; j += kLsapThreads) {
        if (SC[j]) continue;
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minv, C[i * rs + j * cs]), ui), v[j]);
        double sh = shortest[j];
        if (r < sh) { sh = r; shortest[j] = r; path[j] = i; }
        const int key = row4col[j] < 0 ? -1 - pos[j] : pos[j];
        if (lsap_better(sh, key, bs, bk)) { bs = sh; bk = key; }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, bs, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (lsap_better(os, ok, bs, bk)) { bs = os; bk = ok; }
      }
      if (lane == 0) { s_ws[warp] = bs; s_wk[warp] = bk; }
      __syncthreads();
      if (warp == 0) {
        bs = lane < kWarps ? s_ws[lane] : INFINITY;
        bk = lane < kWarps ? s_wk[lane] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          const double os = __shfl_xor_sync(0xffffffffu, bs, o);
          const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
          if (lsap_better(os, ok, bs, bk)) { bs = os; bk = ok; }
        }
        if (lane == 0) {
          const int p = bk < 0 ? -1 - bk : bk, j = remaining[p], last = remaining[nrem - 1];
          s_min = bs;
          SC[j] = 1;
          remaining[p] = last;  // remove: move the last entry into the freed slot
          pos[last] = p;
          s_nrem = nrem - 1;
          if (row4col[j] < 0) {
            s_sink = j;
          } else {
            s_i = row4col[j];
            SR[row4col[j]] = 1;
          }
        }
      }
      __syncthreads();
      if (s_sink >= 0) break;
    }
    const double minv = s_min;
    for (int i = tid; i < nr; i += kLsapThreads)
      if (i == cur) u[i] = __dadd_rn(u[i], minv);
      else if (SR[i]) u[i] = __dadd_rn(u[i], __dsub_rn(minv, shortest[col4row[i]]));
    for (int j = tid; j < nc; j += kLsapThreads)
      if (SC[j]) v[j] = __dsub_rn(v[j], __dsub_rn(minv, shortest[j]));
    __syncthreads();
    if (tid == 0) {  // augment along the path back to `cur`
      int j = s_sink;
      while (true) {
        const int i = path[j];
        row4col[j] = i;
        const int prev = col4row[i];
        col4row[i] = j;
        j = prev;
        if (i == cur) break;
      }
    }
    __syncthreads();
  }
  int* r2c = row2col + (int64_t)b * rows;
  int* c2r = col2row + (int64_t)b * cols;
  if (!tr) {
    for (int i = tid; i < nr; i += kLsapThreads) r2c[i] = col4row[i];
    for (int j = tid; j < nc; j += kLsapThreads) c2r[j] = row4col[j];
  } else {  // solved rows are the original columns
    for (int j = tid; j < nc; j += kLsapThreads) r2c[j] = row4col[j];
    for (int i = tid; i < nr; i += kLsapThreads) c2r[i] = col4row[i];
  }
}

size_t lsap_smem_bytes(int rows, int cols) {
  const size_t nr = rows < cols ? rows : cols, nc = rows < cols ? cols : rows;
  return nc * (2 * sizeof(double) + 4 * sizeof(int) + 1) + nr * (sizeof(double) + sizeof(int) + 1);
}

// step 8 of the reference (:374-400, :524-552): positives are assigned pairs that are close and neither unmatched nor
// ignored; matches: partner, -1 (unmatched, or no positive), -2 (ignored)
__global__ void __launch_bounds__(256) gt_line_label_kernel(const int* __restrict__ row2col,
                                                           const int* __restrict__ col2row,
                                                           const uint8_t* __restrict__ mask,
                                                           const int* __restrict__ flags0, const int* __restrict__ flags1,
                                                           int64_t* __restrict__ m0, int64_t* __restrict__ m1,
                                                           uint8_t* __restrict__ assignment, int L0, int L1) {
  const int b = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
  const int* f0 = flags0 + (int64_t)b * L0;
  const int* f1 = flags1 + (int64_t)b * L1;
  const uint8_t* mk = mask + (int64_t)b * L0 * L1;
  if (t < L0) {
    const int c = row2col[(int64_t)b * L0 + t];
    const bool pos = c >= 0 && mk[(int64_t)t * L1 + c] && !line_excluded(f0[t]) && !line_excluded(f1[c]);
    m0[(int64_t)b * L0 + t] = (f0[t] & kFlagIgnore) ? -2 : pos ? c : -1;
    if (pos && assignment) assignment[((int64_t)b * L0 + t) * L1 + c] = 1;
  }
  if (t < L1) {
    const int r = col2row[(int64_t)b * L1 + t];
    const bool pos = r >= 0 && mk[(int64_t)r * L1 + t] && !line_excluded(f0[r]) && !line_excluded(f1[t]);
    m1[(int64_t)b * L1 + t] = (f1[t] & kFlagIgnore) ? -2 : pos ? r : -1;
  }
}

int launch_lsap(const double* cost, int* row2col, int* col2row, int B, int rows, int cols, cudaStream_t stream) {
  const size_t smem = lsap_smem_bytes(rows, cols);
  LGB_REQUIRE(smem <= 227 * 1024, kErrUnsupported, "lsap: %d x %d needs %zu bytes of shared memory", rows, cols, smem);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(lsap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    LGB_REQUIRE(e == cudaSuccess, kErrCuda, "lsap: %s", cudaGetErrorString(e));
  }
  lsap_kernel<<<B, kLsapThreads, smem, stream>>>(cost, rows, cols, row2col, col2row);
  return check_launch("lsap");
}

}  // namespace lgb

using namespace lgb;

namespace {
// workspace: cost [B,L0,L1] f64 | mask [B,L0,L1] u8 | thr0, flags0, row2col [B,L0] | thr1, flags1, col2row [B,L1]
size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }
}  // namespace

extern "C" {

size_t lgb200_gt_lines_ws_bytes(int B, int L0, int L1) {
  const size_t n = (size_t)B * L0 * L1;
  return align16(n * 8) + align16(n) + align16((size_t)B * L0 * 12) + align16((size_t)B * L1 * 12);
}

int lgb200_gt_line_sample(const float* lines, float* pts, int B, int L, int npts, cudaStream_t stream) {
  LGB_REQUIRE(lines && pts, kErrInvalid, "gt_line_sample: null pointer");
  LGB_REQUIRE(B > 0 && L > 0 && npts >= 2, kErrInvalid, "gt_line_sample: B=%d L=%d npts=%d", B, L, npts);
  LGB_REQUIRE(((reinterpret_cast<uintptr_t>(lines) & 15) | (reinterpret_cast<uintptr_t>(pts) & 7)) == 0, kErrInvalid,
              "gt_line_sample: lines must be 16-byte and pts 8-byte aligned");
  const int64_t total = (int64_t)B * L * npts;
  gt_line_sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(lines),
                                                                             reinterpret_cast<float2*>(pts), total, npts);
  return check_launch("gt_line_sample");
}

int lgb200_lsap(const double* cost, int* row2col, int* col2row, int B, int rows, int cols, cudaStream_t stream) {
  LGB_REQUIRE(cost && row2col && col2row, kErrInvalid, "lsap: null pointer");
  LGB_REQUIRE(B > 0 && rows > 0 && cols > 0, kErrInvalid, "lsap: empty input B=%d rows=%d cols=%d", B, rows, cols);
  return launch_lsap(cost, row2col, col2row, B, rows, cols, stream);
}

int lgb200_gt_line_matches(const float* lines0, const float* lines1, const float* pts0_1, const float* pts1_0,
                           const uint8_t* visible0, const uint8_t* visible1, const uint8_t* valid_pts0,
                           const uint8_t* valid_pts1, const uint8_t* valid_lines0, const uint8_t* valid_lines1, int w0,
                           int h0, int w1, int h1, int npts, double dist_th, double overlap_th,
                           double min_visibility_th, int64_t* m0, int64_t* m1, uint8_t* assignment, void* ws, int B,
                           int L0, int L1, cudaStream_t stream) {
  LGB_REQUIRE(lines0 && lines1 && pts0_1 && pts1_0 && valid_lines0 && valid_lines1 && m0 && m1 && ws, kErrInvalid,
              "gt_line_matches: null pointer");
  LGB_REQUIRE(B > 0 && L0 > 0 && L1 > 0 && npts >= 2, kErrInvalid, "gt_line_matches: B=%d L0=%d L1=%d npts=%d", B, L0,
              L1, npts);
  const bool depth = visible0 != nullptr;
  LGB_REQUIRE((visible1 != nullptr) == depth && (valid_pts0 != nullptr) == depth && (valid_pts1 != nullptr) == depth,
              kErrInvalid, "gt_line_matches: the four point masks are all given (depth variant) or all null");
  LGB_REQUIRE(((reinterpret_cast<uintptr_t>(lines0) | reinterpret_cast<uintptr_t>(lines1)) & 15) == 0 &&
                  ((reinterpret_cast<uintptr_t>(pts0_1) | reinterpret_cast<uintptr_t>(pts1_0)) & 7) == 0,
              kErrInvalid, "gt_line_matches: lines must be 16-byte and points 8-byte aligned");
  const size_t smem = (size_t)npts * kLineTile * (2 * sizeof(float2) + 2);
  LGB_REQUIRE(smem <= 227 * 1024, kErrUnsupported, "gt_line_matches: npts=%d too large", npts);
  const size_t n = (size_t)B * L0 * L1;
  char* p = static_cast<char*>(ws);
  double* cost = reinterpret_cast<double*>(p);
  uint8_t* mask = reinterpret_cast<uint8_t*>(p + align16(n * 8));
  char* q0 = p + align16(n * 8) + align16(n);
  float* thr0 = reinterpret_cast<float*>(q0);
  int* flags0 = reinterpret_cast<int*>(thr0 + (size_t)B * L0);
  int* row2col = flags0 + (size_t)B * L0;
  float* thr1 = reinterpret_cast<float*>(q0 + align16((size_t)B * L0 * 12));
  int* flags1 = reinterpret_cast<int*>(thr1 + (size_t)B * L1);
  int* col2row = flags1 + (size_t)B * L1;
  // thresholds as torch evaluates them: python-float expressions rounded to fp32 at the comparison
  const float out_th = (float)(1.0 - min_visibility_th), min_vis = (float)min_visibility_th;
  const float fixed_th = (float)(npts * overlap_th);
  gt_line_flags_kernel<<<dim3((L0 + L1 + 255) / 256, B), 256, 0, stream>>>(
      reinterpret_cast<const float2*>(pts0_1), reinterpret_cast<const float2*>(pts1_0), visible0, visible1, valid_pts0,
      valid_pts1, valid_lines0, valid_lines1, (float)w0, (float)h0, (float)w1, (float)h1, npts, out_th, min_vis,
      (float)overlap_th, fixed_th, thr0, thr1, flags0, flags1, L0, L1);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(gt_line_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    LGB_REQUIRE(e == cudaSuccess, kErrCuda, "gt_line_matches: %s", cudaGetErrorString(e));
  }
  gt_line_count_kernel<<<dim3((L1 + kLineTile - 1) / kLineTile, (L0 + kLineTile - 1) / kLineTile, B), 256, smem,
                         stream>>>(reinterpret_cast<const float4*>(lines0), reinterpret_cast<const float4*>(lines1),
                                   reinterpret_cast<const float2*>(pts0_1), reinterpret_cast<const float2*>(pts1_0),
                                   visible0, visible1, thr0, thr1, flags0, flags1, (float)dist_th, npts, L0, L1, cost,
                                   mask);
  gt_line_cost_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(cost, flags0, flags1, L0, L1, (int64_t)n);
  int rc = check_launch("gt_line_matches");
  if (rc) return rc;
  rc = launch_lsap(cost, row2col, col2row, B, L0, L1, stream);
  if (rc) return rc;
  if (assignment) {
    cudaError_t e = cudaMemsetAsync(assignment, 0, n, stream);
    LGB_REQUIRE(e == cudaSuccess, kErrCuda, "gt_line_matches: memset: %s", cudaGetErrorString(e));
  }
  const int L = L0 > L1 ? L0 : L1;
  gt_line_label_kernel<<<dim3((L + 255) / 256, B), 256, 0, stream>>>(row2col, col2row, mask, flags0, flags1, m0, m1,
                                                                     assignment, L0, L1);
  return check_launch("gt_line_matches");
}

}  // extern "C"
