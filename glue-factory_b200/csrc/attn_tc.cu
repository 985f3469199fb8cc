// Flash attention on the Hopper tensor cores (sm_90a): out = softmax(scale * q k^T) v
// for head_dim 64 or 32, bf16 operands, fp32 accumulation, never materialising the N x N similarity.
// (reference: lightglue.py:118-121 self-attention; :207-216 cross-attention; gluestick.py:524-529.)
//
// The description below is for head_dim D = 64.  The forward, dQ and dK / dV kernels are templates on D; at D = 32
// (GlueStick with 128-channel descriptors, 4 heads) a q / k / v row is 64 bytes, so the tiles use the 64-byte swizzle,
// Q K^T takes two k-steps instead of four, and the products with a D-wide output (P V, dQ, dK, dV) are m64n32k16.  At
// D = 32 a 64 x 64 tile costs half the tensor-core time of D = 64 but the same 4096 exponentials, so the forward is
// bound by the exponentials there.  The shared-qk backward is built for D = 64 only.
//
// FORWARD.  One CTA = one (batch, head, 128-query tile): two consumer warpgroups of 64 query rows each and one TMA
// producer warp.  Q/K/V tiles are brought in by TMA (4-D tensor map over the token-major [B,N,H,64] layout, 128-byte
// swizzle) and consumed straight from shared memory by wgmma:
//     S_j (64 x 64 fp32, registers) = Q K_j^T      4 wgmma m64n64k16 (both operands K-major in smem)
//     O   (64 x 64 fp32, registers) += P_j V_j     4 wgmma m64n64k16 (P_j from registers, V_j MN-major in smem)
// The softmax runs on the S_j accumulators in place (online maximum, rows shared by the four lanes of a quad) and
// P_j is re-packed to bf16 A fragments without leaving the registers.  For one 64 x 64 tile the wgmma work and the
// 4096 exponentials cost about the same SM time, so they are overlapped: a warpgroup issues S_{j+1} with P_j V_j and
// runs the softmax of S_{j+1} while P_j V_j executes.  106 registers, so two CTAs (four consumer warpgroups) share an
// SM and fill each other's gaps; making the two warpgroups of a CTA take turns (named-barrier ping-pong) measured
// slower at that occupancy.  Tile order and per-element arithmetic are those of the unpipelined loop, so out and lse
// do not depend on the overlap.
// BACKWARD: one CTA owns 128 keys (K, V resident in smem) and walks the queries in tiles of 64 (dK, dV accumulated in
// registers); dQ comes from a second kernel that owns the queries and recomputes S / dP.  No atomics: every sum has
// a fixed order, so eager steps and CUDA-graph replays of a training step agree bit for bit.
// Cross-attention with one shared q = k projection (LightGlue's to_qk) has its own kernel: both directions share the
// similarity, so one sweep per image yields dV and dq + dk (attn_bwd_shared_qk_kernel, below).
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

constexpr int FA_BM = 128;     // queries per CTA
constexpr int FA_BN = 64;      // keys per iteration
constexpr int FA_STAGES = 4;
constexpr int FA_THREADS = 2 * 128 + 32;      // two consumer warpgroups + the producer warp

// Tile geometry at head dim D: a q / k / v row is one head of D bf16, 2D bytes, which is also the swizzle span of the
// TMA tiles and of the wgmma descriptors (128 B at D = 64, 64 B at D = 32).
template <int D>
struct Hd {
  static_assert(D == 32 || D == 64, "head_dim 32 or 64");
  static constexpr int ROW = 2 * D;                    // bytes per row = swizzle span
  static constexpr int SBO = 8 * ROW;                  // 8-row swizzle atom
  static constexpr int WG = 64 * ROW;                  // a warpgroup's 64 rows of a resident tile
  static constexpr int MN_KSTEP = (16 * ROW) >> 4;     // descriptor step of one K=16 slice of an MN-major operand
  static constexpr int NACC = D / 2;                   // fp32 accumulators per thread of a 64 x D tile
  static constexpr int QBYTES = FA_BM * ROW;           // forward: Q tile (16 KiB at D = 64)
  static constexpr int KBYTES = FA_BN * ROW;           // forward: one K or V stage (8 KiB at D = 64)
  static constexpr int SMEM = QBYTES + FA_STAGES * 2 * KBYTES + 256;
};

// wgmma with a D-wide output (P V, dS K, P^T dO, dS^T Q)
template <int D, int TB>
__device__ __forceinline__ void wgmma_m64nD_rs(float (&d)[D / 2], const uint32_t (&a)[4], uint64_t db, int acc) {
  if constexpr (D == 64)
    wgmma_m64n64_rs<TB>(d, a, db, acc);
  else
    wgmma_m64n32_rs<TB>(d, a, db, acc);
}
constexpr int FA_PRODUCER = 8;
constexpr float kLn2 = 0.6931471805599453f, kLog2e = 1.4426950408889634f;

// max / sum over the four lanes of a quad (they share the rows of an accumulator fragment)
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// bf16 store of a 64 x D accumulator (the warpgroup's rows row_base.., valid while < nrows) into the token-major
// [.., N, H, D] layout at (batch, head)
template <int D>
__device__ __forceinline__ void store_acc_rows(const float (&d)[D / 2], __nv_bfloat16* __restrict__ dst, int bat,
                                               int N, int H, int h, int row_base, float mul) {
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = row_base + wq * 16 + (lane >> 2) + 8 * i;
    if (row >= N) continue;
    __nv_bfloat16* o = dst + (((int64_t)bat * N + row) * H + h) * D + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<__nv_bfloat162*>(o + 8 * j) = __floats2bfloat162_rn(d[4 * j + 2 * i] * mul, d[4 * j + 2 * i + 1] * mul);
  }
}

// One CTA of the forward: query tile q0 of head h.  Uniform batches (VARLEN false): TMA coordinates (.., q0, b) and
// (.., key row, kb) of the 4-D maps, rows past Nq / keys past Nk are the map's zero fill.  Packed sequences (VARLEN
// true): 3-D maps over [T, H, D], the sequence's queries start at token row b and its keys at row kb; Nq / Nk are
// the sequence's lengths and Tq the query map's token count (row pitch of lse [H, Tq]).  Rows of the tiles past a
// sequence's end hold the next sequence's tokens: their keys are masked out like the padding, their queries are not
// stored.
template <int D, bool VARLEN>
__device__ __forceinline__ void attn_fwd_tc_cta(const CUtensorMap* tmQ, const CUtensorMap* tmK, const CUtensorMap* tmV,
                                                __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int q0,
                                                int h, int b, int kb, int Nq, int Nk, int H, int Tq,
                                                float scale_log2) {
  using G = Hd<D>;
  constexpr int FA_QBYTES = G::QBYTES, FA_KBYTES = G::KBYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + FA_QBYTES;
  uint8_t* sV = sK + FA_STAGES * FA_KBYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + FA_STAGES * FA_KBYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;               // [FA_STAGES]
  uint64_t* kv_empty = kv_full + FA_STAGES;   // [FA_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = (Nk + FA_BN - 1) / FA_BN;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    mbar_init(q_full, 1);
    for (int s = 0; s < FA_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);
    }
    mbar_fence_init();
  }
  if (warp == FA_PRODUCER && lane == 0) {
    tma_prefetch_desc(tmQ);
    tma_prefetch_desc(tmK);
    tma_prefetch_desc(tmV);
  }
  __syncthreads();

  if (warp == FA_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(q_full, FA_QBYTES);
      if constexpr (VARLEN)
        tma_load_3d(sQ, tmQ, q_full, 0, h, b + q0);
      else
        tma_load_4d(sQ, tmQ, q_full, 0, h, q0, b);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j % FA_STAGES;
        mbar_wait(&kv_empty[s], ((j / FA_STAGES) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 2 * FA_KBYTES);
        if constexpr (VARLEN) {
          tma_load_3d(sK + s * FA_KBYTES, tmK, &kv_full[s], 0, h, kb + j * FA_BN);
          tma_load_3d(sV + s * FA_KBYTES, tmV, &kv_full[s], 0, h, kb + j * FA_BN);
        } else {
          tma_load_4d(sK + s * FA_KBYTES, tmK, &kv_full[s], 0, h, j * FA_BN, kb);
          tma_load_4d(sV + s * FA_KBYTES, tmV, &kv_full[s], 0, h, j * FA_BN, kb);
        }
      }
    }
    return;
  }
  const int wg = threadIdx.x >> 7, t4 = lane & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint64_t dQ0 = make_smem_desc(smem_u32(sQ) + wg * G::WG, 8192, G::SBO, G::ROW);
  const uint64_t dK0 = make_smem_desc(smem_u32(sK), 8192, G::SBO, G::ROW);
  const uint64_t dV0 = make_smem_desc(smem_u32(sV), 8192, G::SBO, G::ROW);
  float o[G::NACC], sv[32], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, alpha[2];
  uint32_t pa[4][4];
#pragma unroll
  for (int e = 0; e < G::NACC; ++e) o[e] = 0.f;
  auto issue_s = [&](int s) {  // S = Q K^T of stage s into sv (the caller waits for the stage, fences and commits)
    const uint64_t so = (uint64_t)((s * FA_KBYTES) >> 4);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64_ss<0, 0>(sv, dQ0 + kk * 2, dK0 + so + kk * 2, kk != 0);
  };
  // online softmax of S_j in place (sv becomes P_j); O is not touched: its rescale by alpha waits until the P V
  // product that is in flight meanwhile has retired
  auto softmax = [&](int j) {
    const int kbase = j * FA_BN;
    if (kbase + FA_BN > Nk) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * jj + 2 * t4 + e >= Nk) sv[4 * jj + e] = sv[4 * jj + 2 + e] = -INFINITY;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * i], sv[4 * jj + 2 * i + 1]));
      const float m_new = fmaxf(m[i], quad_max(mx) * scale_log2);  // every key tile holds at least one valid key
      alpha[i] = fast_exp2(m[i] - m_new);                          // first tile: exp2(-inf) = 0
      float rs = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jj + 2 * i + e;
          sv[x] = fast_exp2(fmaf(sv[x], scale_log2, -m_new));  // masked keys: exp2(-inf) = 0
          rs += sv[x];
        }
      l[i] = l[i] * alpha[i] + rs;  // this lane's partial row sum; the quad is summed at the end
      m[i] = m_new;
    }
  };
  auto rescale_pack = [&]() {  // O *= alpha, P_j -> bf16 A fragments
#pragma unroll
    for (int x = 0; x < G::NACC; ++x) o[x] *= alpha[(x >> 1) & 1];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_afrag(sv, kk, pa[kk]);
  };
  // Pipeline per warpgroup: S_{j+1} is issued together with P_j V_j, and its softmax runs while P_j V_j is still on
  // the tensor cores.  K/V stage j is released once P_j V_j has retired.
  mbar_wait(q_full, 0);
  mbar_wait(&kv_full[0], 0);
  wgmma_fence();
  issue_s(0);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_hold(sv);
  softmax(0);
  rescale_pack();
  for (int j = 0; j + 1 < ntiles; ++j) {
    const int s = j % FA_STAGES;
    const uint64_t so = (uint64_t)((s * FA_KBYTES) >> 4);
    const int s1 = (j + 1) % FA_STAGES;
    mbar_wait(&kv_full[s1], ((j + 1) / FA_STAGES) & 1);
    wgmma_fence();
    issue_s(s1);
    wgmma_commit();
#pragma unroll
    for (int kk = 0; kk < FA_BN / 16; ++kk) wgmma_m64nD_rs<D, 1>(o, pa[kk], dV0 + so + kk * G::MN_KSTEP, 1);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(sv);
    softmax(j + 1);
    wgmma_wait<0>();
    wgmma_hold(o);
    if (signal) mbar_arrive(&kv_empty[s]);
    rescale_pack();
  }
  {  // last tile: P V only
    const int s = (ntiles - 1) % FA_STAGES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FA_BN / 16; ++kk)
      wgmma_m64nD_rs<D, 1>(o, pa[kk], dV0 + (uint64_t)((s * FA_KBYTES) >> 4) + kk * G::MN_KSTEP, 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(o);
  }
  const int rbase = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] = quad_sum(l[i]);
    const float inv = 1.f / l[i];
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj) {
      o[4 * jj + 2 * i] *= inv;
      o[4 * jj + 2 * i + 1] *= inv;
    }
    const int row = rbase + 8 * i;
    if constexpr (VARLEN) {
      if (t4 == 0 && row < Nq) lse[(int64_t)h * Tq + b + row] = (m[i] + log2f(l[i])) * kLn2;
    } else {
      if (t4 == 0 && row < Nq) lse[((int64_t)b * H + h) * Nq + row] = (m[i] + log2f(l[i])) * kLn2;
    }
  }
  if constexpr (VARLEN)
    store_acc_rows<D>(o, out + (int64_t)b * H * D, 0, Nq, H, h, q0 + wg * 64, 1.f);
  else
    store_acc_rows<D>(o, out, b, Nq, H, h, q0 + wg * 64, 1.f);
}

template <int D>
__global__ void __launch_bounds__(FA_THREADS, 1)
    attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, __nv_bfloat16* __restrict__ out,
                       float* __restrict__ lse, int B, int Nq, int Nk, int H, int kv_shift, float scale_log2) {
  const int b = blockIdx.z;
  attn_fwd_tc_cta<D, false>(&tmQ, &tmK, &tmV, out, lse, blockIdx.x * FA_BM, blockIdx.y, b, (b + kv_shift) % B, Nq, Nk,
                            H, 0, scale_log2);
}

// Packed sequences: sequence s = blockIdx.z has queries [q_off[s], q_off[s] + q_len[s]) and keys / values
// [k_off[s], k_off[s] + k_len[s]) of the token-major [T, H, D] buffers.  The grid covers the longest sequence; the
// CTAs of query tiles past a sequence's length, and every CTA of a sequence without queries or keys, exit at once.
template <int D>
__global__ void __launch_bounds__(FA_THREADS, 1)
    attn_fwd_varlen_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                              const __grid_constant__ CUtensorMap tmV, __nv_bfloat16* __restrict__ out,
                              float* __restrict__ lse, const int* __restrict__ q_off, const int* __restrict__ q_len,
                              const int* __restrict__ k_off, const int* __restrict__ k_len, int Tq, int H,
                              float scale_log2) {
  const int s = blockIdx.z, q0 = blockIdx.x * FA_BM;
  const int nq = q_len[s], nk = k_len[s];
  if (q0 >= nq || nk <= 0) return;
  attn_fwd_tc_cta<D, true>(&tmQ, &tmK, &tmV, out, lse, q0, blockIdx.y, q_off[s], k_off[s], nq, nk, H, Tq, scale_log2);
}

// 4-D tensor map over the token-major [B, N, H, D] layout: boxes of box_rows tokens of one head, swizzled by the row
template <int D>
static int make_qkv_tmap(CUtensorMap* tm, const void* base, int B, int N, int H, int box_rows) {
  const uint64_t dims[4] = {D, (uint64_t)H, (uint64_t)N, (uint64_t)B};
  const uint64_t str[3] = {D * 2, (uint64_t)H * D * 2, (uint64_t)N * H * D * 2};
  const uint32_t box[4] = {D, 1, (uint32_t)box_rows, 1};
  return make_tmap_bf16(tm, base, 4, dims, str, box, Hd<D>::ROW);
}

template <int D>
static int attn_fwd_tc_hd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk,
                          int H, int kv_shift, float scale, cudaStream_t stream) {
  constexpr int FA_SMEM = Hd<D>::SMEM;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_qkv_tmap<D>(&tq, q, B, Nq, H, FA_BM))) return rc;  // K/V boxes: FA_BN rows
  if ((rc = make_qkv_tmap<D>(&tk, k, B, Nk, H, FA_BN))) return rc;
  if ((rc = make_qkv_tmap<D>(&tv, v, B, Nk, H, FA_BN))) return rc;
  if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_tc_kernel<D>), FA_SMEM))) return rc;
  dim3 grid((Nq + FA_BM - 1) / FA_BM, H, B);
  attn_fwd_tc_kernel<D><<<grid, FA_THREADS, FA_SMEM, stream>>>(tq, tk, tv, static_cast<__nv_bfloat16*>(out), lse, B, Nq,
                                                               Nk, H, kv_shift, scale * kLog2e);
  return check_launch("attn_fwd_tc");
}

int attn_fwd_tc(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                int kv_shift, float scale, int head_dim, cudaStream_t stream) {
  return head_dim == 32 ? attn_fwd_tc_hd<32>(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, stream)
                        : attn_fwd_tc_hd<64>(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, stream);
}

// 3-D tensor map over a packed token-major [T, H, D] buffer: boxes of box_rows tokens of one head
template <int D>
static int make_packed_tmap(CUtensorMap* tm, const void* base, int T, int H, int box_rows) {
  const uint64_t dims[3] = {D, (uint64_t)H, (uint64_t)T};
  const uint64_t str[2] = {D * 2, (uint64_t)H * D * 2};
  const uint32_t box[3] = {D, 1, (uint32_t)box_rows};
  return make_tmap_bf16(tm, base, 3, dims, str, box, Hd<D>::ROW);
}

template <int D>
static int attn_fwd_varlen_tc_hd(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                                 const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq,
                                 int Tk, int H, float scale, cudaStream_t stream) {
  constexpr int FA_SMEM = Hd<D>::SMEM;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_packed_tmap<D>(&tq, q, Tq, H, FA_BM))) return rc;
  if ((rc = make_packed_tmap<D>(&tk, k, Tk, H, FA_BN))) return rc;
  if ((rc = make_packed_tmap<D>(&tv, v, Tk, H, FA_BN))) return rc;
  if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_varlen_tc_kernel<D>), FA_SMEM))) return rc;
  dim3 grid((max_q_len + FA_BM - 1) / FA_BM, H, S);
  attn_fwd_varlen_tc_kernel<D><<<grid, FA_THREADS, FA_SMEM, stream>>>(tq, tk, tv, static_cast<__nv_bfloat16*>(out), lse,
                                                                      q_off, q_len, k_off, k_len, Tq, H,
                                                                      scale * kLog2e);
  return check_launch("attn_fwd_varlen_tc");
}

int attn_fwd_varlen_tc(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                       const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int Tk,
                       int H, float scale, int head_dim, cudaStream_t stream) {
  return head_dim == 32 ? attn_fwd_varlen_tc_hd<32>(q, k, v, out, lse, q_off, q_len, k_off, k_len, S, max_q_len, Tq,
                                                    Tk, H, scale, stream)
                        : attn_fwd_varlen_tc_hd<64>(q, k, v, out, lse, q_off, q_len, k_off, k_len, S, max_q_len, Tq,
                                                    Tk, H, scale, stream);
}

// ---------------------------------------------------------------------------------------------
// BACKWARD.  dKV kernel: a CTA owns 128 keys (K, V resident in smem; warpgroup w owns keys 64w..64w+63) and walks the
// queries in tiles of 64:
//     S^T  = K Q_i^T,  dP^T = V dO_i^T            (64 x 64 per warpgroup, wgmma from smem)
//     P^T  = exp2(c S^T - lse2_i),  dS^T = P^T (dP^T scale - delta_i scale)   (in registers; lse2 / delta are
//            per-COLUMN values here and come as two 64-float vectors with every query tile)
//     dV  += P^T dO_i,   dK += dS^T Q_i           (P^T / dS^T as register A operands, dO_i / Q_i MN-major from smem)
// dQ kernel: a CTA owns 128 queries (Q, dO resident) and walks the keys in tiles of 64:
//     S = Q K_j^T, dP = dO V_j^T, dS = exp2(c S - lse2) (dP scale - delta scale), dQ += dS K_j.
// Queries past Nq load as zeros and carry lse2 = +inf (p = 0); keys past Nk load as zeros, so their dS meets a zero
// row of K and adds nothing to dQ, and their dK / dV rows are not stored.
// ---------------------------------------------------------------------------------------------
constexpr int FB_R = 128;            // rows owned by the CTA
constexpr int FB_C = 64;             // inner tile
constexpr int FF_STAGES = 3;
constexpr int FQ_STAGES = 4;
template <int D>
struct HdB {
  static constexpr int RBYTES = FB_R * Hd<D>::ROW;        // a resident tile (16 KiB at D = 64)
  static constexpr int CBYTES = FB_C * Hd<D>::ROW;        // a streamed tile (8 KiB at D = 64)
  static constexpr int FF_STAGE_BYTES = 2 * CBYTES + 1024;  // Q | dO | lse2 256 B | delta 256 B (| pad to 1 KiB)
  static constexpr int FF_OFF_STAGE = 2 * RBYTES;         // after the resident K and V tiles
  static constexpr int FF_SMEM = FF_OFF_STAGE + FF_STAGES * FF_STAGE_BYTES + 256;
  static constexpr int FQ_SMEM = 2 * RBYTES + FQ_STAGES * 2 * CBYTES + 256;
};

__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// delta = rowsum(dout * out) * scale; lse2 = lse * log2(e); both written token-tile padded: [B*H][nq_pad] with +inf / 0 in the pad
// (8 lanes per row, D / 8 channels each)
template <int D>
__global__ void __launch_bounds__(256)
    attn_bwd_prep_fused_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                               const float* __restrict__ lse, float* __restrict__ lse2p, float* __restrict__ deltap,
                               int64_t nrows_pad /* B * nq_pad * H */, int N, int nq_pad, int H, float scale) {
  using Vec = std::conditional_t<D == 64, uint4, uint2>;  // D / 8 bf16
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = gid >> 3;  // (b, n_pad, h)
  const int sub = (int)(gid & 7);
  const bool live = r < nrows_pad;  // no early return: the shuffles below are full-warp
  const int64_t rr = live ? r : 0;
  const int h = (int)(rr % H);
  const int64_t bn = rr / H;
  const int n = (int)(bn % nq_pad);
  const int64_t b = bn / nq_pad;
  float acc = 0.f;
  if (live && n < N) {
    const int64_t src = ((b * N + n) * H + h) * D + sub * (D / 8);
    const Vec a = *reinterpret_cast<const Vec*>(out + src);
    const Vec g = *reinterpret_cast<const Vec*>(dout + src);
    const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
    const __nv_bfloat162* pg = reinterpret_cast<const __nv_bfloat162*>(&g);
#pragma unroll
    for (int e = 0; e < D / 16; ++e) {
      const float2 fa = __bfloat1622float2(pa[e]), fg = __bfloat1622float2(pg[e]);
      acc = fmaf(fa.x, fg.x, acc);
      acc = fmaf(fa.y, fg.y, acc);
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (live && sub == 0) {
    const int64_t o = (b * H + h) * nq_pad + n;
    deltap[o] = n < N ? acc * scale : 0.f;  // pre-multiplied: dS = P (dP scale - delta scale)
    lse2p[o] = n < N ? lse[(b * H + h) * N + n] * 1.4426950408889634f : INFINITY;  // pad: p = exp2(-inf) = 0
  }
}

template <int D>
__global__ void __launch_bounds__(FA_THREADS, 1)
    attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                        const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                        const float* __restrict__ lse2p, const float* __restrict__ deltap,
                        __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv, int B, int Nq, int nq_pad,
                        int Nk, int H, int kv_shift, float scale, float scale_log2) {
  using G = Hd<D>;
  constexpr int FB_CBYTES = HdB<D>::CBYTES, FF_STAGE_BYTES = HdB<D>::FF_STAGE_BYTES, FF_SMEM = HdB<D>::FF_SMEM;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sK = smem;
  uint8_t* sV = smem + HdB<D>::RBYTES;
  uint8_t* sStage = smem + HdB<D>::FF_OFF_STAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FF_SMEM - 256);
  uint64_t* kv_full = bars;
  uint64_t* in_full = bars + 1;               // [FF_STAGES]
  uint64_t* in_empty = in_full + FF_STAGES;   // [FF_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * FB_R, h = blockIdx.y, kb = blockIdx.z;
  const int qb = ((kb - kv_shift) % B + B) % B;
  const int ntiles = (Nq + FB_C - 1) / FB_C;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    mbar_init(kv_full, 1);
    for (int s = 0; s < FF_STAGES; ++s) {
      mbar_init(&in_full[s], 1);
      mbar_init(&in_empty[s], 2);
    }
    mbar_fence_init();
  }
  if (warp == FA_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();

  if (warp == FA_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(kv_full, 2 * HdB<D>::RBYTES);
      tma_load_4d(sK, &tmK, kv_full, 0, h, k0, kb);
      tma_load_4d(sV, &tmV, kv_full, 0, h, k0, kb);
      const float* l2 = lse2p + ((int64_t)qb * H + h) * nq_pad;
      const float* dl = deltap + ((int64_t)qb * H + h) * nq_pad;
      for (int i = 0; i < ntiles; ++i) {
        const int s = i % FF_STAGES;
        uint8_t* st = sStage + s * FF_STAGE_BYTES;
        mbar_wait(&in_empty[s], ((i / FF_STAGES) & 1) ^ 1);
        mbar_expect_tx(&in_full[s], 2 * FB_CBYTES + 512);
        tma_load_4d(st, &tmQ, &in_full[s], 0, h, i * FB_C, qb);
        tma_load_4d(st + FB_CBYTES, &tmDO, &in_full[s], 0, h, i * FB_C, qb);
        bulk_load_1d(st + 2 * FB_CBYTES, l2 + i * FB_C, 256, &in_full[s]);
        bulk_load_1d(st + 2 * FB_CBYTES + 256, dl + i * FB_C, 256, &in_full[s]);
      }
    }
    return;
  }
  const int wg = threadIdx.x >> 7, t4 = lane & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint64_t dK0 = make_smem_desc(smem_u32(sK) + wg * G::WG, 8192, G::SBO, G::ROW);
  const uint64_t dV0 = make_smem_desc(smem_u32(sV) + wg * G::WG, 8192, G::SBO, G::ROW);
  const uint64_t dSt0 = make_smem_desc(smem_u32(sStage), 8192, G::SBO, G::ROW);
  float acc_v[G::NACC], acc_k[G::NACC];
#pragma unroll
  for (int e = 0; e < G::NACC; ++e) acc_v[e] = acc_k[e] = 0.f;
  mbar_wait(kv_full, 0);
  for (int i = 0; i < ntiles; ++i) {
    const int s = i % FF_STAGES;
    const uint64_t so = (uint64_t)((s * FF_STAGE_BYTES) >> 4), so_do = so + (FB_CBYTES >> 4);
    const float* sl = reinterpret_cast<const float*>(sStage + s * FF_STAGE_BYTES + 2 * FB_CBYTES);
    mbar_wait(&in_full[s], (i / FF_STAGES) & 1);
    float st[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64_ss<0, 0>(st, dK0 + kk * 2, dSt0 + so + kk * 2, kk != 0);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64_ss<0, 0>(dp, dV0 + kk * 2, dSt0 + so_do + kk * 2, kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(st);
    wgmma_hold(dp);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 l2 = *reinterpret_cast<const float2*>(sl + 8 * jj + 2 * t4);       // columns = queries
      const float2 dl = *reinterpret_cast<const float2*>(sl + 64 + 8 * jj + 2 * t4);  // delta * scale
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int x = 4 * jj + 2 * r;
        st[x] = fast_exp2(fmaf(st[x], scale_log2, -l2.x));
        st[x + 1] = fast_exp2(fmaf(st[x + 1], scale_log2, -l2.y));
        dp[x] = st[x] * fmaf(dp[x], scale, -dl.x);
        dp[x + 1] = st[x + 1] * fmaf(dp[x + 1], scale, -dl.y);
      }
    }
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      acc_to_afrag(st, kk, pa[kk]);
      acc_to_afrag(dp, kk, da[kk]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FB_C / 16; ++kk) wgmma_m64nD_rs<D, 1>(acc_v, pa[kk], dSt0 + so_do + kk * G::MN_KSTEP, 1);
#pragma unroll
    for (int kk = 0; kk < FB_C / 16; ++kk) wgmma_m64nD_rs<D, 1>(acc_k, da[kk], dSt0 + so + kk * G::MN_KSTEP, 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(acc_v);
    wgmma_hold(acc_k);
    if (signal) mbar_arrive(&in_empty[s]);
  }
  store_acc_rows<D>(acc_v, dv, kb, Nk, H, h, k0 + wg * 64, 1.f);
  store_acc_rows<D>(acc_k, dk, kb, Nk, H, h, k0 + wg * 64, 1.f);
}

template <int D>
__global__ void __launch_bounds__(FA_THREADS, 1)
    attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                       const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                       const float* __restrict__ lse2p, const float* __restrict__ deltap, __nv_bfloat16* __restrict__ dq,
                       int B, int Nq, int nq_pad, int Nk, int H, int kv_shift, float scale, float scale_log2) {
  using G = Hd<D>;
  constexpr int FB_CBYTES = HdB<D>::CBYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sDO = smem + HdB<D>::RBYTES;
  uint8_t* sK = smem + 2 * HdB<D>::RBYTES;       // [FQ_STAGES]
  uint8_t* sV = sK + FQ_STAGES * FB_CBYTES;       // [FQ_STAGES]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + FQ_STAGES * FB_CBYTES);
  uint64_t* qd_full = bars;
  uint64_t* in_full = bars + 1;
  uint64_t* in_empty = in_full + FQ_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * FB_R, h = blockIdx.y, b = blockIdx.z;
  const int kb = (b + kv_shift) % B;
  const int ntiles = (Nk + FB_C - 1) / FB_C;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    mbar_init(qd_full, 1);
    for (int s = 0; s < FQ_STAGES; ++s) {
      mbar_init(&in_full[s], 1);
      mbar_init(&in_empty[s], 2);
    }
    mbar_fence_init();
  }
  if (warp == FA_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();

  if (warp == FA_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(qd_full, 2 * HdB<D>::RBYTES);
      tma_load_4d(sQ, &tmQ, qd_full, 0, h, q0, b);
      tma_load_4d(sDO, &tmDO, qd_full, 0, h, q0, b);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j % FQ_STAGES;
        mbar_wait(&in_empty[s], ((j / FQ_STAGES) & 1) ^ 1);
        mbar_expect_tx(&in_full[s], 2 * FB_CBYTES);
        tma_load_4d(sK + s * FB_CBYTES, &tmK, &in_full[s], 0, h, j * FB_C, kb);
        tma_load_4d(sV + s * FB_CBYTES, &tmV, &in_full[s], 0, h, j * FB_C, kb);
      }
    }
    return;
  }
  const int wg = threadIdx.x >> 7;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint64_t dQ0 = make_smem_desc(smem_u32(sQ) + wg * G::WG, 8192, G::SBO, G::ROW);
  const uint64_t dDO0 = make_smem_desc(smem_u32(sDO) + wg * G::WG, 8192, G::SBO, G::ROW);
  const uint64_t dK0 = make_smem_desc(smem_u32(sK), 8192, G::SBO, G::ROW);
  const uint64_t dV0 = make_smem_desc(smem_u32(sV), 8192, G::SBO, G::ROW);
  float l2[2], dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    const int64_t o = ((int64_t)b * H + h) * nq_pad + row;
    l2[r] = row < Nq ? lse2p[o] : INFINITY;
    dl[r] = row < Nq ? deltap[o] : 0.f;
  }
  float acc[G::NACC];
#pragma unroll
  for (int e = 0; e < G::NACC; ++e) acc[e] = 0.f;
  mbar_wait(qd_full, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % FQ_STAGES;
    const uint64_t so = (uint64_t)((s * FB_CBYTES) >> 4);
    mbar_wait(&in_full[s], (j / FQ_STAGES) & 1);
    float sv[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64_ss<0, 0>(sv, dQ0 + kk * 2, dK0 + so + kk * 2, kk != 0);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64_ss<0, 0>(dp, dDO0 + kk * 2, dV0 + so + kk * 2, kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(sv);
    wgmma_hold(dp);
#pragma unroll
    for (int x = 0; x < 32; ++x) {
      const int r = (x >> 1) & 1;
      dp[x] = fast_exp2(fmaf(sv[x], scale_log2, -l2[r])) * fmaf(dp[x], scale, -dl[r]);
    }
    uint32_t da[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_afrag(dp, kk, da[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FB_C / 16; ++kk) wgmma_m64nD_rs<D, 1>(acc, da[kk], dK0 + so + kk * G::MN_KSTEP, 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(acc);
    if (signal) mbar_arrive(&in_empty[s]);
  }
  store_acc_rows<D>(acc, dq, b, Nq, H, h, q0 + wg * 64, 1.f);
}

// Shared-qk cross-attention (reference: lightglue.py:207-216): sequence b attends to its partner p = (b + B/2) mod B
// and p to b with the same projection qk, so both directions share one similarity S = qk_b qk_p^T.  A CTA owns 128
// rows of b (qk_b, v_b, dO_b resident in smem, lse2 / delta of its rows in registers) and streams 64-row tiles of p
// (qk_p, v_p, dO_p, lse2_p, delta_p) through the TMA ring.  Per tile and warpgroup:
//     S = qk_b qk_p^T,  dP = dO_b v_p^T,  dP' = v_b dO_p^T                    (wgmma from smem)
//     P = exp2(c S - lse2_b[row])     (b -> p: rows are the queries)
//     P' = exp2(c S - lse2_p[col])    (p -> b, transposed: columns are the queries)
//     dS = P (dP scale - delta_b scale) + P' (dP' scale - delta_p scale)
//     dV_b += P' dO_p,   dqk_b += dS qk_p                                     (register A operands)
// so dqk_b = dQ_b + dK_b comes out of one sweep: 5 contractions per tile instead of the 7 of a dQ kernel plus a
// dK / dV kernel per direction.  The summation order is fixed (no atomics).  Padding follows the generic kernels: rows
// of p past N load as zeros with lse2 = +inf, so they meet a zero qk_p / dO_p row and P' = 0; rows of b past N are not
// stored.
constexpr int FA_D = 64;                                  // the shared-qk kernel's head dim
constexpr int FB_CBYTES = HdB<FA_D>::CBYTES;              // 8 KiB
constexpr int FX_STAGES = 4;
constexpr int FX_STAGE_BYTES = 25 * 1024;                // qk_p 8 KiB | v_p 8 KiB | dO_p 8 KiB | lse2 256 B | delta 256 B
constexpr int FX_OFF_STAGE = 3 * FB_R * FA_D * 2;         // after the resident qk_b, v_b, dO_b tiles (16 KiB each)
constexpr int FX_SMEM = FX_OFF_STAGE + FX_STAGES * FX_STAGE_BYTES + 256;
// a whole producer warpgroup, so that setmaxnreg can move registers from it to the two consumer warpgroups: S, dP,
// dP', the two accumulators and the in-flight A fragments do not fit in the 168 registers a thread gets at 288 or
// 384 threads per CTA
constexpr int FX_THREADS = 3 * 128;
constexpr int FX_PRODUCER_REGS = 40, FX_CONSUMER_REGS = 232;

__global__ void __launch_bounds__(FX_THREADS, 1)
    attn_bwd_shared_qk_kernel(const __grid_constant__ CUtensorMap tmQKr, const __grid_constant__ CUtensorMap tmVr,
                              const __grid_constant__ CUtensorMap tmDOr, const __grid_constant__ CUtensorMap tmQKs,
                              const __grid_constant__ CUtensorMap tmVs, const __grid_constant__ CUtensorMap tmDOs,
                              const float* __restrict__ lse2p, const float* __restrict__ deltap,
                              __nv_bfloat16* __restrict__ dqk, __nv_bfloat16* __restrict__ dv, int B, int N, int n_pad,
                              int H, int kv_shift, float scale, float scale_log2) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQK = smem;
  uint8_t* sV = smem + FB_R * FA_D * 2;
  uint8_t* sDO = smem + 2 * FB_R * FA_D * 2;
  uint8_t* sStage = smem + FX_OFF_STAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FX_SMEM - 256);
  uint64_t* res_full = bars;
  uint64_t* in_full = bars + 1;               // [FX_STAGES]
  uint64_t* in_empty = in_full + FX_STAGES;   // [FX_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * FB_R, h = blockIdx.y, b = blockIdx.z;
  const int p = (b + kv_shift) % B;
  const int ntiles = (N + FB_C - 1) / FB_C;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    mbar_init(res_full, 1);
    for (int s = 0; s < FX_STAGES; ++s) {
      mbar_init(&in_full[s], 1);
      mbar_init(&in_empty[s], 2);
    }
    mbar_fence_init();
  }
  if (warp == FA_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmQKr);
    tma_prefetch_desc(&tmVr);
    tma_prefetch_desc(&tmDOr);
    tma_prefetch_desc(&tmQKs);
    tma_prefetch_desc(&tmVs);
    tma_prefetch_desc(&tmDOs);
  }
  __syncthreads();

  if (warp >= FA_PRODUCER) {
    setmaxnreg_dec<FX_PRODUCER_REGS>();
    if (warp == FA_PRODUCER && lane == 0) {
      mbar_expect_tx(res_full, 3 * FB_R * FA_D * 2);
      tma_load_4d(sQK, &tmQKr, res_full, 0, h, r0, b);
      tma_load_4d(sV, &tmVr, res_full, 0, h, r0, b);
      tma_load_4d(sDO, &tmDOr, res_full, 0, h, r0, b);
      const float* l2 = lse2p + ((int64_t)p * H + h) * n_pad;
      const float* dl = deltap + ((int64_t)p * H + h) * n_pad;
      for (int i = 0; i < ntiles; ++i) {
        const int s = i % FX_STAGES;
        uint8_t* st = sStage + s * FX_STAGE_BYTES;
        mbar_wait(&in_empty[s], ((i / FX_STAGES) & 1) ^ 1);
        mbar_expect_tx(&in_full[s], 3 * FB_CBYTES + 512);
        tma_load_4d(st, &tmQKs, &in_full[s], 0, h, i * FB_C, p);
        tma_load_4d(st + FB_CBYTES, &tmVs, &in_full[s], 0, h, i * FB_C, p);
        tma_load_4d(st + 2 * FB_CBYTES, &tmDOs, &in_full[s], 0, h, i * FB_C, p);
        bulk_load_1d(st + 3 * FB_CBYTES, l2 + i * FB_C, 256, &in_full[s]);
        bulk_load_1d(st + 3 * FB_CBYTES + 256, dl + i * FB_C, 256, &in_full[s]);
      }
    }
    return;
  }
  setmaxnreg_inc<FX_CONSUMER_REGS>();
  const int wg = threadIdx.x >> 7, t4 = lane & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint64_t dQK0 = make_smem_desc(smem_u32(sQK) + wg * 8192, 8192, 1024);
  const uint64_t dV0 = make_smem_desc(smem_u32(sV) + wg * 8192, 8192, 1024);
  const uint64_t dDO0 = make_smem_desc(smem_u32(sDO) + wg * 8192, 8192, 1024);
  const uint64_t dSt0 = make_smem_desc(smem_u32(sStage), 8192, 1024);
  float l2r[2], dlr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    const int64_t o = ((int64_t)b * H + h) * n_pad + row;
    l2r[r] = row < N ? lse2p[o] : INFINITY;
    dlr[r] = row < N ? deltap[o] : 0.f;
  }
  float acc_v[32], acc_q[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) acc_v[e] = acc_q[e] = 0.f;
  mbar_wait(res_full, 0);
  for (int i = 0; i < ntiles; ++i) {
    const int s = i % FX_STAGES;
    const uint64_t so = (uint64_t)((s * FX_STAGE_BYTES) >> 4);
    const uint64_t so_v = so + (FB_CBYTES >> 4), so_do = so + ((2 * FB_CBYTES) >> 4);
    const float* sl = reinterpret_cast<const float*>(sStage + s * FX_STAGE_BYTES + 3 * FB_CBYTES);
    mbar_wait(&in_full[s], (i / FX_STAGES) & 1);
    float sv[32], dp[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FA_D / 16; ++kk) wgmma_m64n64_ss<0, 0>(sv, dQK0 + kk * 2, dSt0 + so + kk * 2, kk != 0);
#pragma unroll
    for (int kk = 0; kk < FA_D / 16; ++kk) wgmma_m64n64_ss<0, 0>(dp, dDO0 + kk * 2, dSt0 + so_v + kk * 2, kk != 0);
#pragma unroll
    for (int kk = 0; kk < FA_D / 16; ++kk) wgmma_m64n64_ss<0, 0>(dpt, dV0 + kk * 2, dSt0 + so_do + kk * 2, kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(sv);
    wgmma_hold(dp);
    wgmma_hold(dpt);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 l2c = *reinterpret_cast<const float2*>(sl + 8 * jj + 2 * t4);       // columns = rows of p
      const float2 dlc = *reinterpret_cast<const float2*>(sl + 64 + 8 * jj + 2 * t4);  // delta_p * scale
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jj + 2 * r + e;
          const float pr = fast_exp2(fmaf(sv[x], scale_log2, -l2r[r]));
          const float pc = fast_exp2(fmaf(sv[x], scale_log2, -(e ? l2c.y : l2c.x)));
          dp[x] = fmaf(pr, fmaf(dp[x], scale, -dlr[r]), pc * fmaf(dpt[x], scale, -(e ? dlc.y : dlc.x)));
          sv[x] = pc;
        }
    }
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      acc_to_afrag(sv, kk, pa[kk]);
      acc_to_afrag(dp, kk, da[kk]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FB_C / 16; ++kk) wgmma_m64n64_rs<1>(acc_v, pa[kk], dSt0 + so_do + kk * 128, 1);
#pragma unroll
    for (int kk = 0; kk < FB_C / 16; ++kk) wgmma_m64n64_rs<1>(acc_q, da[kk], dSt0 + so + kk * 128, 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(acc_v);
    wgmma_hold(acc_q);
    if (signal) mbar_arrive(&in_empty[s]);
  }
  store_acc_rows<FA_D>(acc_v, dv, b, N, H, h, r0 + wg * 64, 1.f);
  store_acc_rows<FA_D>(acc_q, dqk, b, N, H, h, r0 + wg * 64, 1.f);
}

int64_t attn_bwd_ws_floats(int B, int Nq, int Nk, int H) {
  // lse2 / delta padded to whole query tiles (also covers the fp32 path's B * Nq * H delta floats)
  const int64_t nq_pad = (int64_t)((Nq + FB_C - 1) / FB_C) * FB_C;
  return 2 * (int64_t)B * H * nq_pad;
}

template <int D>
static int attn_bwd_tc_hd(const void* q, const void* k, const void* v, const void* out, const float* lse,
                          const void* dout, void* dq, void* dk, void* dv, float* ws, int B, int Nq, int Nk, int H,
                          int kv_shift, float scale, cudaStream_t stream) {
  constexpr int FQ_SMEM = HdB<D>::FQ_SMEM, FF_SMEM = HdB<D>::FF_SMEM;
  const int nq_pad = (Nq + FB_C - 1) / FB_C * FB_C;
  float* lse2p = ws;
  float* deltap = lse2p + (int64_t)B * H * nq_pad;
  int rc;
  {
    const int64_t nrows = (int64_t)B * nq_pad * H;
    attn_bwd_prep_fused_kernel<D><<<(unsigned)((nrows * 8 + 255) / 256), 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), lse, lse2p, deltap, nrows, Nq,
        nq_pad, H, scale);
  }
  const float sl2 = scale * kLog2e;
  if (D == FA_D && attn_bwd_is_shared_qk(q, k, dq, dk, B, Nq, Nk, kv_shift)) {  // dq (= dk) receives dq + dk
    CUtensorMap tqr, tvr, tdor, tqs, tvs, tdos;
    if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_shared_qk_kernel), FX_SMEM))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tqr, q, B, Nq, H, FB_R))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tvr, v, B, Nq, H, FB_R))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tdor, dout, B, Nq, H, FB_R))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tqs, q, B, Nq, H, FB_C))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tvs, v, B, Nq, H, FB_C))) return rc;
    if ((rc = make_qkv_tmap<FA_D>(&tdos, dout, B, Nq, H, FB_C))) return rc;
    attn_bwd_shared_qk_kernel<<<dim3((Nq + FB_R - 1) / FB_R, H, B), FX_THREADS, FX_SMEM, stream>>>(
        tqr, tvr, tdor, tqs, tvs, tdos, lse2p, deltap, static_cast<__nv_bfloat16*>(dq), static_cast<__nv_bfloat16*>(dv),
        B, Nq, nq_pad, H, kv_shift, scale, sl2);
    return check_launch("attn_bwd_shared_qk");
  }
  CUtensorMap tq, tdo, tk, tv;
  // dQ kernel: 128-query resident tiles, 64-key streamed tiles
  if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_dq_kernel<D>), FQ_SMEM))) return rc;
  if ((rc = make_qkv_tmap<D>(&tq, q, B, Nq, H, FB_R))) return rc;
  if ((rc = make_qkv_tmap<D>(&tdo, dout, B, Nq, H, FB_R))) return rc;
  if ((rc = make_qkv_tmap<D>(&tk, k, B, Nk, H, FB_C))) return rc;
  if ((rc = make_qkv_tmap<D>(&tv, v, B, Nk, H, FB_C))) return rc;
  attn_bwd_dq_kernel<D><<<dim3((Nq + FB_R - 1) / FB_R, H, B), FA_THREADS, FQ_SMEM, stream>>>(
      tq, tdo, tk, tv, lse2p, deltap, static_cast<__nv_bfloat16*>(dq), B, Nq, nq_pad, Nk, H, kv_shift, scale, sl2);
  if ((rc = check_launch("attn_bwd_dq"))) return rc;
  // dK / dV kernel: 128-key resident tiles, 64-query streamed tiles
  if ((rc = make_qkv_tmap<D>(&tq, q, B, Nq, H, FB_C))) return rc;
  if ((rc = make_qkv_tmap<D>(&tdo, dout, B, Nq, H, FB_C))) return rc;
  if ((rc = make_qkv_tmap<D>(&tk, k, B, Nk, H, FB_R))) return rc;
  if ((rc = make_qkv_tmap<D>(&tv, v, B, Nk, H, FB_R))) return rc;
  if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_dkv_kernel<D>), FF_SMEM))) return rc;
  attn_bwd_dkv_kernel<D><<<dim3((Nk + FB_R - 1) / FB_R, H, B), FA_THREADS, FF_SMEM, stream>>>(
      tq, tdo, tk, tv, lse2p, deltap, static_cast<__nv_bfloat16*>(dk), static_cast<__nv_bfloat16*>(dv), B, Nq, nq_pad,
      Nk, H, kv_shift, scale, sl2);
  return check_launch("attn_bwd_dkv");
}

int attn_bwd_tc(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                void* dq, void* dk, void* dv, float* ws, int B, int Nq, int Nk, int H, int kv_shift, float scale,
                int head_dim, cudaStream_t stream) {
  return head_dim == 32
             ? attn_bwd_tc_hd<32>(q, k, v, out, lse, dout, dq, dk, dv, ws, B, Nq, Nk, H, kv_shift, scale, stream)
             : attn_bwd_tc_hd<64>(q, k, v, out, lse, dout, dq, dk, dv, ws, B, Nq, Nk, H, kv_shift, scale, stream);
}

}  // namespace lgb
