// Assignment head fused with its similarity GEMM (SURVEY K8+K9; lightglue.py:256-290, losses.py:6-25):
// sim = mdesc0 . mdesc1^T is produced tile by tile in registers and consumed there -- it is never written to HBM.
//
// Three passes over the same skeleton (persistent CTAs, one per SM):
//   work item = (direction, pair b, 128-row panel).  direction 0: panel rows = keypoints of image 0, columns = all
//   keypoints of image 1 (everything per ROW of sim); direction 1: the transposed problem (everything per COLUMN).
//   Running both directions doubles the (cheap, tensor-core) contraction but makes every reduction a per-row running
//   value: no column partials, no merge kernels, no atomics, deterministic.
//   The panel (A, 128 x D bf16) stays resident in shared memory for the item; 64-column tiles of the other image
//   (B, 64 x D) stream through a 3-stage ring.  Two consumer warpgroups own 64 panel rows each and form
//   S = A B^T (64 x 64 per warpgroup, D/16 wgmma m64n64k16) in registers; a row is shared by the four lanes of a
//   quad (16 of the tile's columns each), whose running values are merged at the end of the item.
//   A producer warpgroup fills each stage: the B tile by TMA and, for STATS / BWD, the tile's side data next to it --
//   the 128 x 64 mask tile (gt for direction 0, gt_t for direction 1) and the two per-column fp32 vectors the
//   elementwise work reads -- so the consumers' inner loop makes no global loads.  Without a mask (labels given as
//   match lists) no mask tile is staged and STATS / BWD have no positive term: lgb200_assign_pos_fwd / _bwd
//   (assign.cu) supply it, one entry per row.
//
//   LSE  : running (max, sum exp2) per row -> lse_row [B,M] (dir 0), lse_col [B,N] (dir 1).
//   STATS: scores in the reference's association order ((s - lse_r) + (s - lse_c)) + (lsig0 + lsig1); running
//          max / first argmax per row -> rowmax/rowarg (dir 0), colmax/colarg (dir 1); dir 0 also gathers
//          sum_j gt_ij (2 s_ij - lse_r_i - lse_c_j) from the boolean assignment.  No MUFU work at all.
//   BWD  : dsim = gc (2 gt - softmax_row rowcnt - softmax_col colcnt) recomputed from S and the two LSE vectors,
//          rounded to bf16 into register A fragments, then
//          d(mdesc) panel (64 x D fp32 per warpgroup, registers) += dsim . B tile (the same smem bytes, MN-major):
//          dir 0 yields d(mdesc0) = dsim mdesc1, dir 1 yields d(mdesc1) = dsim^T mdesc0.  dsim never exists in HBM.
// All three are exact restatements of assign_lse / assign_scores / assign_bwd (assign.cu) on the fp32 accumulator.
#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

constexpr int AT_R = 128;                  // panel rows
constexpr int AT_C = 64;                   // columns per tile
constexpr int AT_KBLK = 64;                // K elements per smem block (one 128-byte swizzle row)
constexpr int AT_ABLK = AT_R * AT_KBLK * 2; // 16 KiB
constexpr int AT_BBLK = AT_C * AT_KBLK * 2; // 8 KiB
constexpr int AT_MAXKB = 4;                // D <= 256
constexpr int AT_STAGES = 3;
constexpr int AT_GBLK = AT_R * AT_C;       // 8 KiB: a stage's mask tile, one 64-byte row per panel row
constexpr int AT_VBLK = 2 * AT_C;          // a stage's two per-column fp32 vectors (512 B)
// A whole producer warpgroup, so that setmaxnreg can move registers from it to the two consumer warpgroups: a BWD
// consumer holds its 64 x 256 fp32 d(mdesc) panel (128 registers) next to S and the dsim fragments, which does not fit
// in the 168 registers a thread gets at 288 or 384 threads per CTA.  Its 128 threads also copy the side data.
constexpr int AT_THREADS = 3 * 128;
constexpr int AT_PRODUCER_WG = 2;
constexpr int AT_PRODUCER_REGS = 56, AT_CONSUMER_REGS = 224;
constexpr float kLog2e_at = 1.4426950408889634f;
constexpr int AT_OFF_G = AT_MAXKB * AT_ABLK + AT_STAGES * AT_MAXKB * AT_BBLK;
constexpr int AT_OFF_V = AT_OFF_G + AT_STAGES * AT_GBLK;
constexpr int AT_SMEM = AT_OFF_V + AT_STAGES * AT_VBLK * 4 + 256;

enum { AT_LSE = 0, AT_STATS = 1, AT_BWD = 2 };

struct AssignTcArgs {
  float alpha;                         // sim = alpha * (md0 . md1^T)
  int B, M, N, D;
  float* lse_row; float* lse_col;      // [B,M], [B,N]   (LSE: out; STATS / BWD: in)
  const float* ls0; const float* ls1;  // STATS: log sigmoid(z0) [B,M], log sigmoid(z1) [B,N]
  const uint8_t* gt;                   // [B,M,N] bool (STATS: optional; BWD: required)
  const uint8_t* gt_t;                 // [B,N,M] bool, the transposed copy (BWD, dir 1)
  float* rowmax; int* rowarg; float* colmax; int* colarg; float* pos_row_sum;  // STATS out
  const float* gcoef;                  // BWD: [B]
  const float* rowcnt; const float* colcnt;  // BWD: [B,M], [B,N]
  __nv_bfloat16* dmd0; __nv_bfloat16* dmd1;  // BWD out: [B*M, D], [B*N, D]
};

// cp.async (generic proxy, read by ordinary shared loads): src_size 0 writes zeros and reads nothing
__device__ __forceinline__ void cp_async_16(void* dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_4(void* dst, const void* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 4 : 0)
               : "memory");
}
// one arrival on `bar` once every cp.async this thread has issued so far has landed (counted in the barrier's init)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(AT_THREADS, 1)
    assign_tc_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1, AssignTcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;
  uint8_t* sB = smem + AT_MAXKB * AT_ABLK;
  uint8_t* sG = smem + AT_OFF_G;
  float* sV = reinterpret_cast<float*>(smem + AT_OFF_V);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AT_SMEM - 256);
  uint64_t* a_full = bars;                   // 1
  uint64_t* a_empty = bars + 1;              // 1
  uint64_t* b_full = bars + 2;               // [AT_STAGES]
  uint64_t* b_empty = b_full + AT_STAGES;    // [AT_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int B = a.B, M = a.M, N = a.N, D = a.D;
  const int KB = D / AT_KBLK;
  const int PM = (M + AT_R - 1) / AT_R, PN = (N + AT_R - 1) / AT_R;
  const int nitems = B * (PM + PN);

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    mbar_init(a_full, 1);
    mbar_init(a_empty, 2);
    for (int s = 0; s < AT_STAGES; ++s) {
      mbar_init(&b_full[s], MODE == AT_LSE ? 1 : 1 + 128);  // the TMA bytes + each producer thread's side data
      mbar_init(&b_empty[s], 8);                           // every consumer warp has read the stage
    }
    mbar_fence_init();
  }
  if (threadIdx.x == AT_PRODUCER_WG * 128) {
    tma_prefetch_desc(&tm0);
    tma_prefetch_desc(&tm1);
  }
  __syncthreads();

  // item -> (dir, b, panel); items of one pair are consecutive so its tiles are shared through L2
  auto decode = [&](int item, int& dir, int& b, int& p) {
    b = item / (PM + PN);
    const int r = item - b * (PM + PN);
    dir = r >= PM;
    p = dir ? r - PM : r;
  };
  // the mask an item reads, rows = its panel's rows (null: none)
  auto mask_of = [&](int dir) -> const uint8_t* {
    return MODE == AT_BWD ? (dir ? a.gt_t : a.gt) : (MODE == AT_STATS && !dir) ? a.gt : nullptr;
  };

  if (wg == AT_PRODUCER_WG) {
    // ------------------------------------------------------------------ producer: TMA (thread 0) + side data
    setmaxnreg_dec<AT_PRODUCER_REGS>();
    const int pt = threadIdx.x & 127;
    if (MODE == AT_LSE && pt != 0) return;
    int it = 0, g = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++it) {
      int dir, b, p;
      decode(item, dir, b, p);
      const CUtensorMap* tA = dir ? &tm1 : &tm0;
      const CUtensorMap* tB = dir ? &tm0 : &tm1;
      const int nrows = dir ? N : M, ncols = dir ? M : N;
      const int ntiles = (ncols + AT_C - 1) / AT_C;
      if (pt == 0) {
        mbar_wait(a_empty, (it & 1) ^ 1);
        mbar_expect_tx(a_full, KB * AT_ABLK);
        for (int kb = 0; kb < KB; ++kb)
          for (int hf = 0; hf < 2; ++hf)  // two 64-row boxes per block: the same bytes as one 128-row box
            tma_load_3d(sA + kb * AT_ABLK + hf * AT_BBLK, tA, a_full, kb * AT_KBLK, p * AT_R + hf * AT_C, b);
      }
      const uint8_t* gm = mask_of(dir);
      const uint8_t* gpanel = gm ? gm + ((int64_t)b * nrows + p * AT_R) * ncols : nullptr;
      // 16-byte copies need 16-byte aligned rows; ragged widths take the byte-wise path
      const bool direct = !gm || (ncols % 16 == 0 && (reinterpret_cast<uintptr_t>(gm) & 15) == 0);
      const int prows = min(AT_R, nrows - p * AT_R);
      const float* va = nullptr;
      const float* vb = nullptr;
      if (MODE != AT_LSE) {  // STATS: lse_other, ls_other; BWD: lse_other, cnt_other
        va = (dir ? a.lse_row : a.lse_col) + (int64_t)b * ncols;
        vb = (MODE == AT_STATS ? (dir ? a.ls0 : a.ls1) : (dir ? a.rowcnt : a.colcnt)) + (int64_t)b * ncols;
      }
      for (int t = 0; t < ntiles; ++t, ++g) {
        const int s = g % AT_STAGES;
        mbar_wait(&b_empty[s], ((g / AT_STAGES) & 1) ^ 1);
        if (pt == 0) {
          mbar_expect_tx(&b_full[s], KB * AT_BBLK);
          for (int kb = 0; kb < KB; ++kb)
            tma_load_3d(sB + (s * AT_MAXKB + kb) * AT_BBLK, tB, &b_full[s], kb * AT_KBLK, t * AT_C, b);
        }
        if (MODE != AT_LSE) {
          const int c0 = t * AT_C;
          const int jv = c0 + (pt & 63);  // thread pt copies entry pt % 64 of vector pt / 64; zeros past the end
          const float* vsrc = (pt < 64 ? va : vb) + (jv < ncols ? jv : 0);
          float* vdst = sV + s * AT_VBLK + pt;
          uint8_t* gdst = sG + s * AT_GBLK;
          if (direct) {
            cp_async_4(vdst, vsrc, jv < ncols);
            if (gpanel) {
#pragma unroll
              for (int u = 0; u < 4; ++u) {  // 16-byte piece q: panel row q / 4, columns c0 + 16 (q % 4) + [0, 16)
                const int q = pt + 128 * u, r = q >> 2, c = c0 + 16 * (q & 3);
                const bool ok = r < prows && c < ncols;
                cp_async_16(gdst + 16 * q, gpanel + (ok ? (int64_t)r * ncols + c : 0), ok);
              }
            }
            cp_async_mbar_arrive(&b_full[s]);
          } else {
            *vdst = jv < ncols ? *vsrc : 0.f;
#pragma unroll 1
            for (int u = 0; u < 4; ++u) {
              const int q = pt + 128 * u, r = q >> 2, c = c0 + 16 * (q & 3);
              const uint8_t* src = gpanel + (int64_t)r * ncols + c;
              const int n = r < prows ? min(16, ncols - c) : 0;
#pragma unroll 1
              for (int k = 0; k < 16; ++k) gdst[16 * q + k] = k < n ? src[k] : 0;
            }
            mbar_arrive(&b_full[s]);
          }
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumer warpgroups
  setmaxnreg_inc<AT_CONSUMER_REGS>();
  const int t4 = lane & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint64_t dA = make_smem_desc(smem_u32(sA) + wg * 8192, 8192, 1024);
  const uint64_t dB = make_smem_desc(smem_u32(sB), 8192, 1024);
  const float c2 = a.alpha * kLog2e_at;
  int rl[2];  // this thread's two rows within the panel
#pragma unroll
  for (int i = 0; i < 2; ++i) rl[i] = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
  int it = 0, g = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++it) {
    int dir, b, p;
    decode(item, dir, b, p);
    const int nrows = dir ? N : M, ncols = dir ? M : N;
    const int ntiles = (ncols + AT_C - 1) / AT_C;
    const bool has_mask = mask_of(dir) != nullptr;
    // per-row constants of this thread's two rows
    bool rok[2];
    int64_t ro[2];
    float lse_mine[2] = {0.f, 0.f}, ls_mine[2] = {0.f, 0.f}, coef_mine[2] = {0.f, 0.f};
    const float gc = MODE == AT_BWD ? a.gcoef[b] : 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = p * AT_R + rl[i];
      rok[i] = row < nrows;
      ro[i] = (int64_t)b * nrows + (rok[i] ? row : 0);
      if (MODE != AT_LSE) lse_mine[i] = (dir ? a.lse_col : a.lse_row)[ro[i]];
      if (MODE == AT_STATS) ls_mine[i] = (dir ? a.ls1 : a.ls0)[ro[i]];
      if (MODE == AT_BWD) {
        coef_mine[i] = rok[i] ? gc * (dir ? a.colcnt : a.rowcnt)[ro[i]] : 0.f;
        lse_mine[i] *= kLog2e_at;
      }
    }
    // running values (this lane's 16 columns of every tile)
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // LSE (log2 domain)
    float best[2] = {-INFINITY, -INFINITY}, psum[2] = {0.f, 0.f};    // STATS
    int besti[2] = {0x7fffffff, 0x7fffffff};
    float acc[AT_MAXKB][32];                                         // BWD: d(mdesc) rows, 64 channels per block
    if (MODE == AT_BWD) {
#pragma unroll
      for (int c = 0; c < AT_MAXKB; ++c)
#pragma unroll
        for (int e = 0; e < 32; ++e) acc[c][e] = 0.f;
    }
    mbar_wait(a_full, it & 1);
    for (int t = 0; t < ntiles; ++t, ++g) {
      const int s = g % AT_STAGES;
      const uint64_t sb = dB + (uint64_t)((s * AT_MAXKB * AT_BBLK) >> 4);
      const uint8_t* sg = sG + s * AT_GBLK;  // mask tile: row r at sg + 64 r
      const float* sv_a = sV + s * AT_VBLK;  // lse_other[64] | ls_other or cnt_other[64]
      mbar_wait(&b_full[s], (g / AT_STAGES) & 1);
      float sv[32];
      wgmma_fence();
      for (int kb = 0; kb < KB; ++kb) {
#pragma unroll
        for (int kk = 0; kk < AT_KBLK / 16; ++kk)
          wgmma_m64n64_ss<0, 0>(sv, dA + (uint64_t)((kb * AT_ABLK) >> 4) + kk * 2,
                                sb + (uint64_t)((kb * AT_BBLK) >> 4) + kk * 2, (kb | kk) != 0);
      }
      wgmma_commit();
      // does this row hold a positive in the tile?  Each lane of the quad tests 16 of the row's 64 bytes (a warp
      // reads 512 contiguous bytes: no bank conflicts); nearly every row is all zero and skips the positive term.
      bool pos[2] = {false, false};
      if (MODE != AT_LSE && has_mask) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const uint4 w = *reinterpret_cast<const uint4*>(sg + 64 * rl[i] + 16 * t4);
          uint32_t u = w.x | w.y | w.z | w.w;
          u |= __shfl_xor_sync(0xffffffffu, u, 1);
          u |= __shfl_xor_sync(0xffffffffu, u, 2);
          pos[i] = u != 0u;
        }
      }
      wgmma_wait<0>();
      wgmma_hold(sv);
      if (MODE == AT_LSE && lane == 0) mbar_arrive(&b_empty[s]);  // S is in registers: the tile's stage is free
      const int j0 = t * AT_C + 2 * t4;  // column of sv[0]; sv[4jj + 2i + e] is column j0 + 8jj + e of row i
      if (MODE == AT_LSE) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float mx = -INFINITY;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float& x = sv[4 * jj + 2 * i + e];
              if (j0 + 8 * jj + e >= ncols) x = -INFINITY;
              mx = fmaxf(mx, x);
            }
          // alpha > 0: max commutes with the scale.  All-masked columns: mx = -inf, contributes nothing.
          const float m_new = fmaxf(m_run[i], mx * c2);
          if (m_new > -INFINITY) {
            float sum = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int e = 0; e < 2; ++e) sum += fast_exp2(fmaf(sv[4 * jj + 2 * i + e], c2, -m_new));
            l_run[i] = l_run[i] * fast_exp2(m_run[i] - m_new) + sum;
            m_run[i] = m_new;
          }
        }
      } else if (MODE == AT_STATS) {
        // score_ij = (2 alpha S_ij + [lsig - lse]_other(j)) + [lsig - lse]_mine: the second bracket is constant along
        // the row, so the running max / first argmax is taken over the first term only and the constant is added
        // when the result is written.  (assign_scores in assign.cu keeps the reference's association order for the
        // fp32 parity path; the two agree to fp32 rounding.)
        const float a2 = 2.f * a.alpha;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float2 lc2 = *reinterpret_cast<const float2*>(sv_a + 8 * jj + 2 * t4);
          const float2 ls2 = *reinterpret_cast<const float2*>(sv_a + AT_C + 8 * jj + 2 * t4);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * jj + 2 * t4 + e, j = t * AT_C + c;
            const bool cok = j < ncols;
            const float lc = cok ? (e ? lc2.y : lc2.x) : 0.f;
            const float cv = cok ? (e ? ls2.y : ls2.x) - lc : -INFINITY;  // -inf masks the tail
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float x = fmaf(sv[4 * jj + 2 * i + e], a2, cv);
              if (x > best[i]) {  // columns are visited in increasing order: the first maximum stays
                best[i] = x;
                besti[i] = j;
              }
              if (pos[i] && sg[64 * rl[i] + c]) psum[i] += (x - cv) - lse_mine[i] - lc;  // zeros past the end
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[s]);
      } else {  // AT_BWD
        const float two_gc = 2.f * gc;
        float ds[32];  // dsim, in S's layout (written apart from S: S's registers belong to the MMA pipeline)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float2 lc2 = *reinterpret_cast<const float2*>(sv_a + 8 * jj + 2 * t4);
          const float2 cn2 = *reinterpret_cast<const float2*>(sv_a + AT_C + 8 * jj + 2 * t4);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * jj + 2 * t4 + e, j = t * AT_C + c;
            const bool cok = j < ncols;
            const float lc = cok ? (e ? lc2.y : lc2.x) * kLog2e_at : INFINITY;  // exp2(x - inf) = 0 past the end
            const float cc = cok ? (e ? cn2.y : cn2.x) * gc : 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float x = sv[4 * jj + 2 * i + e];
              float v = (pos[i] && sg[64 * rl[i] + c]) ? two_gc : 0.f;  // zeros past the end
              v = fmaf(-fast_exp2(fmaf(x, c2, -lse_mine[i])), coef_mine[i], v);
              if (cc != 0.f) v = fmaf(-fast_exp2(fmaf(x, c2, -lc)), cc, v);
              ds[4 * jj + 2 * i + e] = cok ? v : 0.f;
            }
          }
        }
        uint32_t da[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) acc_to_afrag(ds, kk, da[kk]);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < AT_MAXKB; ++c) {
          if (c < KB) {
#pragma unroll
            for (int kk = 0; kk < AT_C / 16; ++kk)  // 16 columns per step; block c holds channels [64c, 64c + 64)
              wgmma_m64n64_rs<1>(acc[c], da[kk], sb + (uint64_t)((c * AT_BBLK) >> 4) + kk * 128, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int c = 0; c < AT_MAXKB; ++c) wgmma_hold(acc[c]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[s]);
      }
    }
    if (signal) mbar_arrive(a_empty);  // every MMA that reads the panel has retired

    // ---- end of item: merge the four lanes of each row (LSE / STATS) or store the panel gradient (BWD)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (MODE == AT_LSE) {
        float m = m_run[i], l = l_run[i];
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {  // (max, sum exp2) of two lanes, log2 domain; -inf partials add nothing
          const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
          const float mn = fmaxf(m, m2);
          l = (m == mn ? l : l * fast_exp2(m - mn)) + (m2 == mn ? l2 : l2 * fast_exp2(m2 - mn));
          m = mn;
        }
        if (t4 == 0 && rok[i]) (dir ? a.lse_col : a.lse_row)[ro[i]] = (m + log2f(l)) * 0.6931471805599453f;
      } else if (MODE == AT_STATS) {
        float bv = best[i], ps = psum[i];
        int bi = besti[i];
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float b2 = __shfl_xor_sync(0xffffffffu, bv, o);
          const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
          if (b2 > bv || (b2 == bv && i2 < bi)) { bv = b2; bi = i2; }  // on equal values the lower index stays
          ps += __shfl_xor_sync(0xffffffffu, ps, o);
        }
        if (t4 == 0 && rok[i]) {
          (dir ? a.colmax : a.rowmax)[ro[i]] = bv + (ls_mine[i] - lse_mine[i]);
          (dir ? a.colarg : a.rowarg)[ro[i]] = bi;
          if (!dir && a.pos_row_sum) a.pos_row_sum[ro[i]] = ps;
        }
      } else if (rok[i]) {
        __nv_bfloat16* out = (dir ? a.dmd1 : a.dmd0) + ro[i] * D + 2 * t4;
#pragma unroll
        for (int c = 0; c < AT_MAXKB; ++c) {
          if (c < KB) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              *reinterpret_cast<__nv_bfloat162*>(out + c * 64 + 8 * jj) =
                  __floats2bfloat162_rn(acc[c][4 * jj + 2 * i], acc[c][4 * jj + 2 * i + 1]);
          }
        }
      }
    }
  }
}

static int make_md_map(CUtensorMap* tm, const void* base, int B, int rows, int D) {
  const uint64_t dims[3] = {(uint64_t)D, (uint64_t)rows, (uint64_t)B};
  const uint64_t str[2] = {(uint64_t)D * 2, (uint64_t)rows * D * 2};
  const uint32_t box[3] = {AT_KBLK, AT_C, 1};
  return make_tmap_bf16(tm, base, 3, dims, str, box);
}

template <int MODE>
static int launch_assign_tc(const void* md0, const void* md1, const AssignTcArgs& a, cudaStream_t stream) {
  LGB_REQUIRE(md0 && md1, kErrInvalid, "assign_fused: null mdesc pointer");
  LGB_REQUIRE(a.B > 0 && a.M > 0 && a.N > 0, kErrInvalid, "assign_fused: empty input B=%d M=%d N=%d", a.B, a.M, a.N);
  LGB_REQUIRE(a.D % 64 == 0 && a.D >= 64 && a.D <= 256, kErrUnsupported,
              "assign_fused: descriptor width %d not a multiple of 64 in [64, 256]", a.D);
  LGB_REQUIRE(a.alpha > 0.f, kErrInvalid, "assign_fused: alpha must be positive");
  CUtensorMap t0, t1;
  int rc;
  if ((rc = make_md_map(&t0, md0, a.B, a.M, a.D))) return rc;
  if ((rc = make_md_map(&t1, md1, a.B, a.N, a.D))) return rc;
  auto kern = assign_tc_kernel<MODE>;
  if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), AT_SMEM))) return rc;
  const int items = a.B * ((a.M + AT_R - 1) / AT_R + (a.N + AT_R - 1) / AT_R);
  const int sms = device_sm_count();
  kern<<<items < sms ? items : sms, AT_THREADS, AT_SMEM, stream>>>(t0, t1, a);
  return check_launch("assign_fused");
}

}  // namespace lgb

using namespace lgb;

extern "C" {

int lgb200_assign_fused_lse(const void* md0, const void* md1, float alpha, float* lse_row, float* lse_col, int B, int M,
                            int N, int D, cudaStream_t stream) {
  LGB_REQUIRE(lse_row && lse_col, kErrInvalid, "assign_fused_lse: null pointer");
  AssignTcArgs a = {};
  a.alpha = alpha; a.B = B; a.M = M; a.N = N; a.D = D;
  a.lse_row = lse_row; a.lse_col = lse_col;
  return launch_assign_tc<AT_LSE>(md0, md1, a, stream);
}

int lgb200_assign_fused_stats(const void* md0, const void* md1, float alpha, const float* lse_row, const float* lse_col,
                              const float* ls0, const float* ls1, const uint8_t* gt, float* rowmax, int* rowarg,
                              float* colmax, int* colarg, float* pos_row_sum, int B, int M, int N, int D,
                              cudaStream_t stream) {
  LGB_REQUIRE(lse_row && lse_col && ls0 && ls1 && rowmax && rowarg && colmax && colarg, kErrInvalid,
              "assign_fused_stats: null pointer");
  LGB_REQUIRE((gt == nullptr) == (pos_row_sum == nullptr), kErrInvalid,
              "assign_fused_stats: gt and pos_row_sum must both be set or both be null");
  AssignTcArgs a = {};
  a.alpha = alpha; a.B = B; a.M = M; a.N = N; a.D = D;
  a.lse_row = const_cast<float*>(lse_row); a.lse_col = const_cast<float*>(lse_col);
  a.ls0 = ls0; a.ls1 = ls1; a.gt = gt;
  a.rowmax = rowmax; a.rowarg = rowarg; a.colmax = colmax; a.colarg = colarg; a.pos_row_sum = pos_row_sum;
  return launch_assign_tc<AT_STATS>(md0, md1, a, stream);
}

int lgb200_assign_fused_bwd(const void* md0, const void* md1, float alpha, const float* lse_row, const float* lse_col,
                            const uint8_t* gt, const uint8_t* gt_t, const float* gcoef, const float* rowcnt,
                            const float* colcnt, void* dmd0, void* dmd1, int B, int M, int N, int D,
                            cudaStream_t stream) {
  LGB_REQUIRE(lse_row && lse_col && gcoef && rowcnt && colcnt && dmd0 && dmd1, kErrInvalid,
              "assign_fused_bwd: null pointer");
  // both masks NULL: no mask tile is staged and dsim has no positive term (lgb200_assign_pos_bwd adds it)
  LGB_REQUIRE((gt == nullptr) == (gt_t == nullptr), kErrInvalid,
              "assign_fused_bwd: gt and gt_t must both be set or both be null");
  AssignTcArgs a = {};
  a.alpha = alpha; a.B = B; a.M = M; a.N = N; a.D = D;
  a.lse_row = const_cast<float*>(lse_row); a.lse_col = const_cast<float*>(lse_col);
  a.gt = gt; a.gt_t = gt_t; a.gcoef = gcoef; a.rowcnt = rowcnt; a.colcnt = colcnt;
  a.dmd0 = static_cast<__nv_bfloat16*>(dmd0); a.dmd1 = static_cast<__nv_bfloat16*>(dmd1);
  return launch_assign_tc<AT_BWD>(md0, md1, a, stream);
}

}  // extern "C"
