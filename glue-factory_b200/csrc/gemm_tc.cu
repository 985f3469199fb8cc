// Batched bf16 GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers, operands staged by TMA
// into 128-byte-swizzled shared memory).  Used for the assignment similarity sim = mdesc0 . mdesc1^T
// (lightglue.py:283), its two backward contractions and the layer's projections, which need every combination of
// K-major / MN-major operands (wgmma reads both layouts straight from shared memory).
//
// Persistent CTAs (one per SM) walk 128x128 tiles of C, n fastest so neighbouring CTAs share the A tile in L2.
// Warp roles: warpgroups 0 and 1 each own 64 rows of the tile (m64n128k16 wgmma, 64 accumulators per thread); warp 8
// is the TMA producer (one lane).  A 4-stage smem ring of 64-wide K blocks (one 128-byte swizzle atom per operand row)
// runs ahead across tile boundaries, so the loads of tile i+1 overlap the epilogue of tile i.
//
// Epilogue: each warpgroup writes alpha * acc (+ bias) into its own 128-byte-swizzled staging buffer in shared memory,
// and one thread hands the buffer to the TMA unit: a tensor store, or for an accumulating fp32 C a tensor reduce-add
// (C += tile, done at L2: the SM never reads C).  The warpgroup goes straight on to the next tile's MMAs while the
// stores drain; it waits for the TMA unit to have read the buffer only before it fills it again.  A C that TMA cannot
// address (base or pitch not 16-byte aligned) is written straight from the accumulator registers instead.
#include <string.h>

#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

constexpr int GB_M = 128, GB_N = 128, GB_K = 64, G_STAGES = 4;
constexpr int G_TILE = GB_M * GB_K * 2;  // 16 KiB per operand per stage
constexpr int G_THREADS = 2 * 128 + 32;  // two consumer warpgroups + the producer warp
constexpr int G_PRODUCER = 8;            // warp index of the producer
constexpr int G_BOX = 64 * 128;          // one TMA box of C: 64 rows x 128 bytes (32 fp32 / 64 bf16 columns), 8 KiB
// staging per consumer warpgroup in the generic kernel: its whole 64 x 128 slice of the tile
template <typename OutT>
__host__ __device__ constexpr int g_stage_bytes() { return 64 * GB_N * (int)sizeof(OutT); }
template <typename OutT>
__host__ __device__ constexpr int g_smem() { return G_STAGES * 2 * G_TILE + 2 * g_stage_bytes<OutT>() + 256; }

__device__ __forceinline__ void st_shared_pair(uint32_t addr, float v0, float v1) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
}
__device__ __forceinline__ void st_shared_pair(uint32_t addr, uint32_t packed) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(packed) : "memory");
}

// Staged epilogue of one warpgroup's 64 x 128 accumulator: C (+)= alpha * acc (+ bias[col]) through `stage`
// (SB bytes, 1024-aligned, SB / 8 KiB boxes of 64 rows x 128 bytes in the 128-byte swizzle of tmC).  An fp32 tile
// that does not fit (SB = 16 KiB in the A-panel kernel) goes out in column passes of SB / 256 columns.  Same per-element
// arithmetic as gemm_store_tile; TMA clips the rows >= M and columns >= N of ragged tiles.  Called by all 128 threads
// of the warpgroup; `leader` (one of them) issues and tracks the bulk stores.
template <typename OutT, int SB>
__device__ __forceinline__ void gemm_store_tile_tma(const float (&d)[64], uint8_t* stage, const CUtensorMap* tmC,
                                                    int M, int N, int m_base, int n0, int bo, float alpha,
                                                    const float* __restrict__ bias, int reduce_add, int wg,
                                                    bool leader) {
  constexpr int ES = (int)sizeof(OutT);
  constexpr int PASS_COLS = SB / (64 * ES), PASSES = GB_N / PASS_COLS, BOXES = SB / G_BOX, BOX_COLS = 128 / ES;
  static_assert(SB % G_BOX == 0 && GB_N % PASS_COLS == 0, "staging holds whole boxes");
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r0 = wq * 16 + (lane >> 2);  // row within the slice; (r0 + 8i) & 7 == lane >> 2
  const uint32_t sbase = smem_u32(stage);
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    if (leader) bulk_wait_read<0>();  // the previous stores out of this buffer have read it
    named_bar(1 + wg, 128);
#pragma unroll
    for (int jj = 0; jj < PASS_COLS / 8; ++jj) {
      const int j = p * (PASS_COLS / 8) + jj;
      const int c = 8 * jj + 2 * (lane & 3);  // column within the pass
      const int col = n0 + 8 * j + 2 * (lane & 3);
      float b0 = 0.f, b1 = 0.f;
      if (bias) {
        if (col < N) b0 = bias[col];
        if (col + 1 < N) b1 = bias[col + 1];
      }
      const uint32_t cb = (uint32_t)(c * ES);  // byte offset of the pair within the pass's rows
      const uint32_t box = cb >> 7, chunk = (cb >> 4) & 7;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t row = (uint32_t)(r0 + 8 * i);
        const float v0 = fmaf(d[4 * j + 2 * i], alpha, b0), v1 = fmaf(d[4 * j + 2 * i + 1], alpha, b1);
        const uint32_t addr = sbase + box * G_BOX + row * 128 + ((chunk ^ (uint32_t)(lane >> 2)) << 4) + (cb & 15);
        if constexpr (ES == 4)
          st_shared_pair(addr, v0, v1);
        else
          st_shared_pair(addr, pack_bf16(v0, v1));
      }
    }
    fence_proxy_async_smem();  // the st.shared above -> visible to the TMA unit
    named_bar(1 + wg, 128);
    if (leader && m_base < M) {
#pragma unroll
      for (int b = 0; b < BOXES; ++b) {
        const int cx = n0 + p * PASS_COLS + b * BOX_COLS;
        if (cx >= N) break;
        if (reduce_add)
          tma_reduce_add_3d(tmC, stage + b * G_BOX, cx, m_base, bo);
        else
          tma_store_3d(tmC, stage + b * G_BOX, cx, m_base, bo);
      }
      bulk_commit();
    }
  }
}

// Register epilogue for a C that TMA cannot address: C (+)= alpha * acc (+ bias[col]) straight from the accumulators.
// Each thread owns two adjacent columns of 16 column groups in two rows; pairs are stored as one 8-byte (fp32) /
// 4-byte (bf16) word when `vec` (C and its pitches even-aligned), element by element otherwise.  reduce_add (fp32 C
// only) adds into C.
template <typename OutT>
__device__ __forceinline__ void gemm_store_tile(const float (&d)[64], OutT* __restrict__ C, int M, int N, int64_t ldc,
                                                int m_base, int n0, float alpha, const float* __restrict__ bias,
                                                int reduce_add, int vec) {
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r0 = m_base + wq * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < GB_N / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    if (col >= N) continue;
    const bool two = col + 1 < N;
    float b0 = 0.f, b1 = 0.f;
    if (bias) {
      b0 = bias[col];
      if (two) b1 = bias[col + 1];
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = r0 + 8 * i;
      if (row >= M) continue;
      float v0 = fmaf(d[4 * j + 2 * i], alpha, b0), v1 = fmaf(d[4 * j + 2 * i + 1], alpha, b1);
      OutT* dst = C + (int64_t)row * ldc + col;
      if constexpr (sizeof(OutT) == 4) {
        if (vec && two) {
          float2* p2 = reinterpret_cast<float2*>(dst);
          if (reduce_add) {
            const float2 o = *p2;
            v0 += o.x;
            v1 += o.y;
          }
          *p2 = make_float2(v0, v1);
        } else {
          dst[0] = reduce_add ? dst[0] + v0 : v0;
          if (two) dst[1] = reduce_add ? dst[1] + v1 : v1;
        }
      } else {
        if (vec && two) {
          *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
        } else {
          dst[0] = __float2bfloat16(v0);
          if (two) dst[1] = __float2bfloat16(v1);
        }
      }
    }
  }
}

template <bool A_MN, bool B_MN, typename OutT>
__global__ void __launch_bounds__(G_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmC /* {N, M, batch} over C, used when tma_out */,
                     OutT* __restrict__ C, int M, int N, int K, int64_t ldc, int64_t strideC, float alpha, int tiles_m,
                     int tiles_n, int ntiles,
                     int kps /* split-K: k-blocks per split (0 = off); the tile's batch index is then the split */,
                     const float* __restrict__ bias /* [N] added to every row, or null */,
                     int reduce_add /* fp32 C only: C += alpha A B (+ bias) */, int tma_out, int vec) {
  constexpr int SB = g_stage_bytes<OutT>();
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;
  uint8_t* sB = smem + G_STAGES * G_TILE;
  uint8_t* sC = smem + 2 * G_STAGES * G_TILE;  // [2 warpgroups][SB]
  uint64_t* full = reinterpret_cast<uint64_t*>(sC + 2 * SB);
  uint64_t* empty = full + G_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = (K + GB_K - 1) / GB_K;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    for (int s = 0; s < G_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  if (warp == G_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (tma_out) tma_prefetch_desc(&tmC);
  }
  __syncthreads();

  if (warp == G_PRODUCER) {
    if (lane == 0) {
      int it = 0;  // running k-block count across tiles (ring position)
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int n0 = (t % tiles_n) * GB_N, m0 = ((t / tiles_n) % tiles_m) * GB_M, bo = t / (tiles_n * tiles_m);
        const int k_first = kps ? bo * kps : 0, k_last = kps ? min(nk, k_first + kps) : nk;
        const int b = kps ? 0 : bo;  // split-K reads the one input batch at different k offsets
        for (int kb = k_first; kb < k_last; ++kb, ++it) {
          const int s = it % G_STAGES;
          mbar_wait(&empty[s], ((it / G_STAGES) & 1) ^ 1);
          mbar_expect_tx(&full[s], 2 * G_TILE);
          uint8_t* a = sA + s * G_TILE;
          uint8_t* bb = sB + s * G_TILE;
          if (!A_MN) {
            tma_load_3d(a, &tmA, &full[s], kb * GB_K, m0, b);
          } else {
            tma_load_3d(a, &tmA, &full[s], m0, kb * GB_K, b);
            tma_load_3d(a + 8192, &tmA, &full[s], m0 + 64, kb * GB_K, b);
          }
          if (!B_MN) {
            tma_load_3d(bb, &tmB, &full[s], kb * GB_K, n0, b);
          } else {
            tma_load_3d(bb, &tmB, &full[s], n0, kb * GB_K, b);
            tma_load_3d(bb + 8192, &tmB, &full[s], n0 + 64, kb * GB_K, b);
          }
        }
      }
    }
  } else {
    const int wg = threadIdx.x >> 7;
    const bool signal = (threadIdx.x & 127) == 0;
    // the warpgroup's 64 rows of A start 8 KiB into the block in both layouts (K-major: 64 rows of 128 B further;
    // MN-major: the second 64-wide TMA box)
    const uint64_t ad0 = make_smem_desc(smem_u32(sA) + wg * 8192, 8192, 1024);
    const uint64_t bd0 = make_smem_desc(smem_u32(sB), 8192, 1024);
    constexpr uint64_t a_step = (A_MN ? 2048 : 32) >> 4, b_step = (B_MN ? 2048 : 32) >> 4;
    int it = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int n0 = (t % tiles_n) * GB_N, m0 = ((t / tiles_n) % tiles_m) * GB_M, bo = t / (tiles_n * tiles_m);
      const int nk_item = kps ? min(nk, (bo + 1) * kps) - bo * kps : nk;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int kb = 0; kb < nk_item; ++kb, ++it) {
        const int s = it % G_STAGES;
        mbar_wait(&full[s], (it / G_STAGES) & 1);
        wgmma_fence();
        const uint64_t so = (uint64_t)((s * G_TILE) >> 4);
#pragma unroll
        for (int kk = 0; kk < GB_K / 16; ++kk)
          wgmma_m64n128_ss<A_MN, B_MN>(d, ad0 + so + kk * a_step, bd0 + so + kk * b_step, (kb | kk) != 0);
        wgmma_commit();
        wgmma_wait<1>();  // the previous block's MMAs have retired: its stage goes back to the producer
        if (kb > 0 && signal) mbar_arrive(&empty[(it - 1) % G_STAGES]);
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if (signal) mbar_arrive(&empty[(it - 1) % G_STAGES]);
      if (tma_out)
        gemm_store_tile_tma<OutT, SB>(d, sC + wg * SB, &tmC, M, N, m0 + wg * 64, n0, bo, alpha, bias, reduce_add, wg,
                                      signal);
      else
        gemm_store_tile<OutT>(d, C + (int64_t)bo * strideC, M, N, ldc, m0 + wg * 64, n0, alpha, bias,
                              reduce_add, vec);
    }
    if (tma_out && signal) bulk_wait<0>();  // the CTA's last stores have landed before it exits
  }
}

// ---------------------------------------------------------------------------------------------
// A-panel-resident variant for the layer's K <= 256 GEMMs (y = x W^T and dx = dy W with a 256-wide contraction: 6 of the
// 10 forward projections and 5 of the 9 input-gradient GEMMs of a layer).  The generic kernel above re-loads the A tile
// for every n-tile (128 KiB of operands per 128 x 128 output tile).  Here a work item is one 128-row panel of A: the
// panel (KB x 16 KiB) is loaded ONCE into one of two resident buffers (the next item's panel is prefetched while this
// one is multiplied), only the B blocks stream through a ring, and the CTA walks all n-tiles of the panel.  Operand
// bytes per panel for N = 256: 64 + 128 KiB instead of 256 KiB; for N = 768: 64 + 384 instead of 768.  A is K-major
// (rows of x / dy).  Same warpgroup split and epilogue (bias, bf16 / fp32, accumulate) as the generic kernel; its
// staging is 16 KiB per warpgroup (the panels and the B ring leave 32 KiB), which holds a bf16 slice whole and an fp32
// slice in two column halves.
// ---------------------------------------------------------------------------------------------
constexpr int GP_KB = 4;                      // K <= 256
constexpr int GP_BSTAGES = 4;                 // 16 KiB B blocks in flight
constexpr int GP_BBLK = GB_N * GB_K * 2;      // 16 KiB
constexpr int GP_STAGE = 2 * G_BOX;           // epilogue staging per consumer warpgroup
constexpr int GP_SMEM = 2 * GP_KB * G_TILE + GP_BSTAGES * GP_BBLK + 2 * GP_STAGE + 256;

template <bool B_MN, typename OutT>
__global__ void __launch_bounds__(G_THREADS, 1)
    gemm_apanel_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmC, OutT* __restrict__ C, int M, int N, int K, int64_t ldc,
                       float alpha, int tiles_m, int tiles_n, const float* __restrict__ bias, int reduce_add,
                       int tma_out, int vec) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;                                   // [2 panels][GP_KB blocks]
  uint8_t* sB = smem + 2 * GP_KB * G_TILE;              // [GP_BSTAGES]
  uint8_t* sC = sB + GP_BSTAGES * GP_BBLK;              // [2 warpgroups][GP_STAGE]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sC + 2 * GP_STAGE);
  uint64_t* a_full = bars;                 // [2]
  uint64_t* a_empty = bars + 2;            // [2]
  uint64_t* b_full = bars + 4;             // [GP_BSTAGES]
  uint64_t* b_empty = b_full + GP_BSTAGES; // [GP_BSTAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = (K + GB_K - 1) / GB_K;
  const int nitems = tiles_m;

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();
    for (int s = 0; s < 2; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 2);
    }
    for (int s = 0; s < GP_BSTAGES; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 2);
    }
    mbar_fence_init();
  }
  if (warp == G_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (tma_out) tma_prefetch_desc(&tmC);
  }
  __syncthreads();

  if (warp == G_PRODUCER) {
    if (lane == 0) {
      auto load_panel = [&](int item, int li) {  // li: this CTA's running item index -> panel buffer li & 1
        const int pa = li & 1;
        mbar_wait(&a_empty[pa], ((li >> 1) & 1) ^ 1);
        mbar_expect_tx(&a_full[pa], KB * G_TILE);
        for (int kb = 0; kb < KB; ++kb) tma_load_3d(sA + (pa * GP_KB + kb) * G_TILE, &tmA, &a_full[pa], kb * GB_K, item * GB_M, 0);
      };
      int li = 0, bi = 0;
      if ((int)blockIdx.x < nitems) load_panel(blockIdx.x, 0);
      for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++li) {
        for (int nt = 0; nt < tiles_n; ++nt) {
          // the next item's panel is requested after this item's first n-tile is on its way: its buffer is released when
          // the PREVIOUS item's MMAs retire, and by then they have (the B ring's back-pressure paces this thread)
          if (nt == (tiles_n > 1 ? 1 : 0) && item + (int)gridDim.x < nitems && tiles_n > 1)
            load_panel(item + gridDim.x, li + 1);
          for (int kb = 0; kb < KB; ++kb, ++bi) {
            const int s = bi % GP_BSTAGES;
            mbar_wait(&b_empty[s], ((bi / GP_BSTAGES) & 1) ^ 1);
            mbar_expect_tx(&b_full[s], GP_BBLK);
            uint8_t* bb = sB + s * GP_BBLK;
            if (!B_MN) {
              tma_load_3d(bb, &tmB, &b_full[s], kb * GB_K, nt * GB_N, 0);
            } else {
              tma_load_3d(bb, &tmB, &b_full[s], nt * GB_N, kb * GB_K, 0);
              tma_load_3d(bb + 8192, &tmB, &b_full[s], nt * GB_N + 64, kb * GB_K, 0);
            }
          }
        }
        if (tiles_n == 1 && item + (int)gridDim.x < nitems) load_panel(item + gridDim.x, li + 1);
      }
    }
  } else {
    const int wg = threadIdx.x >> 7;
    const bool signal = (threadIdx.x & 127) == 0;
    const uint64_t ad0 = make_smem_desc(smem_u32(sA) + wg * 8192, 8192, 1024);
    const uint64_t bd0 = make_smem_desc(smem_u32(sB), 8192, 1024);
    constexpr uint64_t a_step = 32 >> 4, b_step = (B_MN ? 2048 : 32) >> 4;
    int li = 0, bi = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++li) {
      const int pa = li & 1;
      mbar_wait(&a_full[pa], (li >> 1) & 1);
      for (int nt = 0; nt < tiles_n; ++nt) {
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        for (int kb = 0; kb < KB; ++kb, ++bi) {
          const int s = bi % GP_BSTAGES;
          mbar_wait(&b_full[s], (bi / GP_BSTAGES) & 1);
          wgmma_fence();
          const uint64_t ao = (uint64_t)(((pa * GP_KB + kb) * G_TILE) >> 4), bo = (uint64_t)((s * GP_BBLK) >> 4);
#pragma unroll
          for (int kk = 0; kk < GB_K / 16; ++kk)
            wgmma_m64n128_ss<false, B_MN>(d, ad0 + ao + kk * a_step, bd0 + bo + kk * b_step, (kb | kk) != 0);
          wgmma_commit();
          wgmma_wait<1>();
          if (kb > 0 && signal) mbar_arrive(&b_empty[(bi - 1) % GP_BSTAGES]);
        }
        wgmma_wait<0>();
        wgmma_hold(d);
        if (signal) {
          mbar_arrive(&b_empty[(bi - 1) % GP_BSTAGES]);
          if (nt == tiles_n - 1) mbar_arrive(&a_empty[pa]);  // every MMA that reads this panel has retired
        }
        if (tma_out)
          gemm_store_tile_tma<OutT, GP_STAGE>(d, sC + wg * GP_STAGE, &tmC, M, N, item * GB_M + wg * 64, nt * GB_N, 0,
                                              alpha, bias, reduce_add, wg, signal);
        else
          gemm_store_tile<OutT>(d, C, M, N, ldc, item * GB_M + wg * 64, nt * GB_N, alpha, bias, reduce_add, vec);
      }
    }
    if (tma_out && signal) bulk_wait<0>();
  }
}

// C and its pitches allow the paired (two-column) stores of the epilogue
template <typename OutT>
static int pair_aligned(const void* C, int64_t ldc, int batch, int64_t strideC) {
  constexpr int ES = (int)sizeof(OutT);
  return (reinterpret_cast<uintptr_t>(C) % (2 * ES)) == 0 && ldc % 2 == 0 && (batch == 1 || strideC % 2 == 0);
}

// Tensor map of C for the staged epilogue: dims {N, M, batch}, 64-row x 128-byte boxes in the 128-byte swizzle.
// *tma_out = 0 (and the map left zeroed) when TMA cannot address C: its base, row pitch or batch stride is not a
// multiple of 16 bytes.  The kernel then writes C from registers.
template <typename OutT>
static int make_c_map(CUtensorMap* tc, int* tma_out, const void* C, int batch, int M, int N, int64_t ldc,
                      int64_t strideC) {
  constexpr int ES = (int)sizeof(OutT);
  memset(tc, 0, sizeof(*tc));
  *tma_out = reinterpret_cast<uintptr_t>(C) % 16 == 0 && (ldc * ES) % 16 == 0 &&
             (batch == 1 || (strideC * ES) % 16 == 0);
  if (!*tma_out) return 0;
  const uint64_t dims[3] = {(uint64_t)N, (uint64_t)M, (uint64_t)batch};
  const uint64_t str[2] = {(uint64_t)ldc * ES, (uint64_t)(batch > 1 ? strideC : (int64_t)M * ldc) * ES};
  const uint32_t box[3] = {128 / ES, 64, 1};
  return make_tmap(tc, C, ES == 4, 3, dims, str, box);
}

template <bool A_MN, bool B_MN, typename OutT>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int batch, int M, int N, int K,
                       int64_t ldc, int64_t strideC, float alpha, cudaStream_t stream, int kps = 0,
                       const float* bias = nullptr, int reduce_add = 0) {
  LGB_REQUIRE(!reduce_add || sizeof(OutT) == 4, kErrInvalid, "gemm: accumulate-into-C needs an fp32 C");
  auto kern = gemm_bf16_kernel<A_MN, B_MN, OutT>;
  constexpr int smem = g_smem<OutT>();
  {
    int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem);
    if (rc) return rc;
  }
  CUtensorMap tc;
  int tma_out = 0;
  {
    int rc = make_c_map<OutT>(&tc, &tma_out, C, batch, M, N, ldc, strideC);
    if (rc) return rc;
  }
  const int num_sms = device_sm_count();
  const int tiles_m = (M + GB_M - 1) / GB_M, tiles_n = (N + GB_N - 1) / GB_N;
  const int64_t ntiles = (int64_t)tiles_m * tiles_n * batch;
  LGB_REQUIRE(ntiles < (1ll << 31), kErrUnsupported, "gemm: too many tiles");
  const unsigned grid = (unsigned)(ntiles < num_sms ? ntiles : num_sms);
  kern<<<grid, G_THREADS, smem, stream>>>(ta, tb, tc, static_cast<OutT*>(C), M, N, K, ldc, strideC, alpha, tiles_m,
                                          tiles_n, (int)ntiles, kps, bias, reduce_add, tma_out,
                                          pair_aligned<OutT>(C, ldc, batch, strideC));
  return check_launch("gemm_bf16");
}

// C[m, n] = sum over splits (in split order: deterministic) of the fp32 partial tiles
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ C, int M,
                                                           int N, int64_t ldc, int splits) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int64_t total = (int64_t)M * N;
  if (i >= total) return;
  if ((N & 3) == 0) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sidx = 0; sidx < splits; ++sidx) {
      const float4 v = *reinterpret_cast<const float4*>(ws + (int64_t)sidx * total + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float* dst = C + (i / N) * ldc + (i % N);
    dst[0] = acc.x; dst[1] = acc.y; dst[2] = acc.z; dst[3] = acc.w;
  } else {
    for (int64_t e = i; e < i + 4 && e < total; ++e) {
      float acc = 0.f;
      for (int sidx = 0; sidx < splits; ++sidx) acc += ws[(int64_t)sidx * total + e];
      C[(e / N) * ldc + (e % N)] = acc;
    }
  }
}

// split-K plan for a [M,N] = sum_K product: as many splits as idle SMs allow, at least 4 k-blocks each
static void splitk_plan(int M, int N, int K, int* splits, int* kps) {
  const int tiles = ((M + GB_M - 1) / GB_M) * ((N + GB_N - 1) / GB_N);
  const int nk = (K + GB_K - 1) / GB_K;
  int s = device_sm_count() / tiles;
  if (s > nk / 4) s = nk / 4;
  if (s < 1) s = 1;
  *kps = (nk + s - 1) / s;
  *splits = (nk + *kps - 1) / *kps;
}

}  // namespace lgb

using namespace lgb;

static int make_ab_maps(CUtensorMap* ta, CUtensorMap* tb, const void* A, const void* B, int batch, int M, int N, int K,
                        int a_mn_major, int b_mn_major, int64_t lda, int64_t ldb, int64_t strideA, int64_t strideB) {
  {
    // A: K-major -> dims {K, M, batch}; MN-major (stored [K,M]) -> dims {M, K, batch}
    const uint64_t inner = a_mn_major ? (uint64_t)M : (uint64_t)K, outer = a_mn_major ? (uint64_t)K : (uint64_t)M;
    const uint64_t dims[3] = {inner, outer, (uint64_t)batch};
    const uint64_t str[2] = {(uint64_t)lda * 2, (uint64_t)(batch > 1 ? strideA : (int64_t)outer * lda) * 2};
    const uint32_t box[3] = {64, a_mn_major ? 64u : 128u, 1};
    int rc = make_tmap_bf16(ta, A, 3, dims, str, box);
    if (rc) return rc;
  }
  {
    const uint64_t inner = b_mn_major ? (uint64_t)N : (uint64_t)K, outer = b_mn_major ? (uint64_t)K : (uint64_t)N;
    const uint64_t dims[3] = {inner, outer, (uint64_t)batch};
    const uint64_t str[2] = {(uint64_t)ldb * 2, (uint64_t)(batch > 1 ? strideB : (int64_t)outer * ldb) * 2};
    const uint32_t box[3] = {64, b_mn_major ? 64u : 128u, 1};
    int rc = make_tmap_bf16(tb, B, 3, dims, str, box);
    if (rc) return rc;
  }
  return 0;
}

extern "C" int64_t lgb200_gemm_splitk_ws_floats(int M, int N, int K) {
  int splits = 1, kps = 0;
  splitk_plan(M, N, K, &splits, &kps);
  return (int64_t)splits * M * N;
}

extern "C" int lgb200_gemm_bf16_splitk(const void* A, const void* B, float* C, int M, int N, int K, int a_mn_major,
                                       int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, float* ws,
                                       cudaStream_t stream) {
  LGB_REQUIRE(A && B && C && ws, kErrInvalid, "gemm_bf16_splitk: null pointer");
  LGB_REQUIRE(M > 0 && N > 0 && K > 0, kErrInvalid, "gemm_bf16_splitk: empty problem %dx%dx%d", M, N, K);
  LGB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, kErrInvalid, "gemm_bf16_splitk: lda/ldb must be multiples of 8 elements");
  CUtensorMap ta, tb;
  int rc = make_ab_maps(&ta, &tb, A, B, 1, M, N, K, a_mn_major, b_mn_major, lda, ldb, 0, 0);
  if (rc) return rc;
  int splits = 1, kps = 0;
  splitk_plan(M, N, K, &splits, &kps);
#define LGB_SPLITK_CASE(AM, BMJ)                                                                                  \
  if (a_mn_major == AM && b_mn_major == BMJ)                                                                      \
    rc = launch_gemm<AM, BMJ, float>(ta, tb, ws, splits, M, N, K, N, (int64_t)M * N, 1.f, stream, kps);
  LGB_SPLITK_CASE(0, 0)
  LGB_SPLITK_CASE(0, 1)
  LGB_SPLITK_CASE(1, 0)
  LGB_SPLITK_CASE(1, 1)
#undef LGB_SPLITK_CASE
  if (rc) return rc;
  const int64_t quads = ((int64_t)M * N + 3) / 4;
  splitk_reduce_kernel<<<(unsigned)((quads + 255) / 256), 256, 0, stream>>>(ws, C, M, N, ldc, splits);
  return check_launch("gemm_bf16_splitk");
}

extern "C" int lgb200_gemm_bf16(const void* A, const void* B, void* C, int batch, int M, int N, int K, int a_mn_major,
                                int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, int64_t strideA,
                                int64_t strideB, int64_t strideC, int c_dtype, float alpha, cudaStream_t stream) {
  LGB_REQUIRE(A && B && C, kErrInvalid, "gemm_bf16: null pointer");
  LGB_REQUIRE(batch > 0 && M > 0 && N > 0 && K > 0, kErrInvalid, "gemm_bf16: empty problem %dx%dx%dx%d", batch, M, N, K);
  LGB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, kErrInvalid, "gemm_bf16: lda/ldb must be multiples of 8 elements");
  LGB_REQUIRE(batch == 1 || (strideA % 8 == 0 && strideB % 8 == 0), kErrInvalid,
              "gemm_bf16: batch strides must be multiples of 8 elements");
  CUtensorMap ta, tb;
  {
    int rc = make_ab_maps(&ta, &tb, A, B, batch, M, N, K, a_mn_major, b_mn_major, lda, ldb, strideA, strideB);
    if (rc) return rc;
  }
#define LGB_GEMM_CASE(AM, BMJ)                                                                              \
  if (a_mn_major == AM && b_mn_major == BMJ) {                                                              \
    if (c_dtype == LGB200_F32) return launch_gemm<AM, BMJ, float>(ta, tb, C, batch, M, N, K, ldc, strideC, alpha, stream); \
    if (c_dtype == LGB200_BF16)                                                                             \
      return launch_gemm<AM, BMJ, __nv_bfloat16>(ta, tb, C, batch, M, N, K, ldc, strideC, alpha, stream);  \
  }
  LGB_GEMM_CASE(0, 0)
  LGB_GEMM_CASE(0, 1)
  LGB_GEMM_CASE(1, 0)
  LGB_GEMM_CASE(1, 1)
#undef LGB_GEMM_CASE
  LGB_REQUIRE(false, kErrInvalid, "gemm_bf16: bad major/dtype flags");
}

// y = alpha * op(A) op(B)^T + bias (+ C when beta != 0): the nn.Linear-shaped projections of the layer
// (lightglue.py:139-148, 156-163, 174-183, 195-221, 280) and their input-gradient GEMMs, single problem (no batch).
extern "C" int lgb200_linear(const void* A, const void* B, void* C, const float* bias, int M, int N, int K,
                             int a_mn_major, int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, int c_dtype,
                             float alpha, int accumulate, cudaStream_t stream) {
  LGB_REQUIRE(A && B && C, kErrInvalid, "linear: null pointer");
  LGB_REQUIRE(M > 0 && N > 0 && K > 0, kErrInvalid, "linear: empty problem %dx%dx%d", M, N, K);
  LGB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, kErrInvalid, "linear: lda/ldb must be multiples of 8 elements");
  LGB_REQUIRE(!accumulate || c_dtype == LGB200_F32, kErrInvalid, "linear: accumulate needs an fp32 C");
  CUtensorMap ta, tb;
  int rc = make_ab_maps(&ta, &tb, A, B, 1, M, N, K, a_mn_major, b_mn_major, lda, ldb, 0, 0);
  if (rc) return rc;
  {  // A-panel-resident kernel: K <= 256, K-major A
    if (!a_mn_major && K <= GP_KB * GB_K && (c_dtype == LGB200_F32 || c_dtype == LGB200_BF16)) {
      const int tiles_m = (M + GB_M - 1) / GB_M, tiles_n = (N + GB_N - 1) / GB_N;
      const int sms = device_sm_count();
      const unsigned grid = (unsigned)(tiles_m < sms ? tiles_m : sms);
#define LGB_AP_LAUNCH(BMJ, T)                                                                                    \
  {                                                                                                              \
    auto kern = gemm_apanel_kernel<BMJ, T>;                                                                      \
    if ((rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), GP_SMEM))) return rc;                        \
    CUtensorMap tc;                                                                                              \
    int tma_out = 0;                                                                                             \
    if ((rc = make_c_map<T>(&tc, &tma_out, C, 1, M, N, ldc, 0))) return rc;                                      \
    kern<<<grid, G_THREADS, GP_SMEM, stream>>>(ta, tb, tc, static_cast<T*>(C), M, N, K, ldc, alpha, tiles_m,     \
                                               tiles_n, bias, accumulate ? 1 : 0, tma_out,                       \
                                               pair_aligned<T>(C, ldc, 1, 0));                                   \
    return check_launch("linear(apanel)");                                                                       \
  }
      if (c_dtype == LGB200_F32) {
        if (b_mn_major) LGB_AP_LAUNCH(true, float) else LGB_AP_LAUNCH(false, float)
      } else {
        if (b_mn_major) LGB_AP_LAUNCH(true, __nv_bfloat16) else LGB_AP_LAUNCH(false, __nv_bfloat16)
      }
#undef LGB_AP_LAUNCH
    }
  }
#define LGB_LIN_CASE(AM, BMJ)                                                                                       \
  if (a_mn_major == AM && b_mn_major == BMJ) {                                                                      \
    if (c_dtype == LGB200_F32)                                                                                      \
      return launch_gemm<AM, BMJ, float>(ta, tb, C, 1, M, N, K, ldc, 0, alpha, stream, 0, bias, accumulate ? 1 : 0); \
    if (c_dtype == LGB200_BF16)                                                                                     \
      return launch_gemm<AM, BMJ, __nv_bfloat16>(ta, tb, C, 1, M, N, K, ldc, 0, alpha, stream, 0, bias, 0);       \
  }
  LGB_LIN_CASE(0, 0)
  LGB_LIN_CASE(0, 1)
  LGB_LIN_CASE(1, 0)
  LGB_LIN_CASE(1, 1)
#undef LGB_LIN_CASE
  LGB_REQUIRE(false, kErrInvalid, "linear: bad major/dtype flags");
}
