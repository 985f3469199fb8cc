// SuperPoint keypoint extraction on Hopper (inference only): the frozen extractor of the homography pre-training and
// uncached MegaDepth configurations (gluefactory_nonfree/superpoint.py, SuperPoint._forward).
//
//  conv1a      gray conversion + 1 -> 64 3x3 conv + bias + ReLU on CUDA cores, NHWC bf16 out.
//  sp_conv     implicit-GEMM convolution on wgmma (bf16 operands, fp32 accumulators).  A CTA owns an 8 x 16 pixel
//              output tile (M = 128, one 64-row warpgroup per 4 pixel rows) and BN output channels.  K runs over
//              (tap, 64-channel block); each 128 x 64 A block is gathered by cp.async straight from the NHWC input
//              (zero-filled outside the image: the conv's padding) into the 128-byte swizzle wgmma reads, three
//              stages deep.  Epilogues: bias + ReLU; bias + ReLU + 2x2 max-pool (only the pooled map is written);
//              65-way softmax, dustbin dropped, depth-to-space into the full-resolution score map; L2 normalisation
//              of each pixel's 256 channels (the tile holds whole pixel rows).
//  sp_nms      simple_nms (two suppression rounds) per tile with the 5r halo its chained max-pools need, then the
//              border removal.  Comparisons only: equal to the reference bit for bit on the same score map.
//  sp_count / sp_select   candidates above the threshold, per-image top-k by a 4 x 8-bit radix select, device
//              padding for force_num_keypoints.
//  sp_sample   bilinear grid_sample of the dense descriptors (legacy align_corners=True, or the fixed variant),
//              L2-normalised, one warp per keypoint, written as [B, K, C].
//
// SuperPoint-open (gluefactory/models/extractors/superpoint_open.py) puts a BatchNorm after every conv.  With running
// statistics (eval mode) its affine y = scale x + shift is folded into the conv epilogues above (AFF): after the ReLU
// and before the pool in the encoder, before the softmax / L2 normalisation in the heads.  With batch statistics
// (training mode) the convs write the pre-BatchNorm activations (ReLU, or RAW fp32 for the heads), lgb200_bn_stats
// sums them, and spo_bn_apply normalises: plain, + 2x2 max-pool, + softmax / depth-to-space, + L2 normalisation.
#include <algorithm>

#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

__device__ __forceinline__ void sp_cp16(void* dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void sp_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void sp_cp_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------------------------
// conv1a
// ---------------------------------------------------------------------------------------------
// one thread per (pixel, 8 output channels); gray = (r * .299 + g * .587) + b * .114 rounded per op like torch's
// (image * scale).sum(1)
// AFF: ReLU then the per-channel affine scale * x + shift (an eval-mode BatchNorm)
template <bool AFF>
__global__ void __launch_bounds__(256) sp_conv1a_kernel(const float* __restrict__ img, int C,
                                                        const float* __restrict__ w, const float* __restrict__ bias,
                                                        __nv_bfloat16* __restrict__ out, int B, int H, int W,
                                                        const float* __restrict__ scale,
                                                        const float* __restrict__ shift) {
  __shared__ float sw[64 * 9], sb[64];
  __shared__ float ss[AFF ? 64 : 1], sh[AFF ? 64 : 1];
  for (int i = threadIdx.x; i < 64 * 9; i += blockDim.x) sw[i] = w[i];
  for (int i = threadIdx.x; i < 64; i += blockDim.x) sb[i] = bias[i];
  if constexpr (AFF)
    for (int i = threadIdx.x; i < 64; i += blockDim.x) {
      ss[i] = scale[i];
      sh[i] = shift[i];
    }
  __syncthreads();
  const int64_t n = (int64_t)B * H * W * 8;
  const int64_t HW = (int64_t)H * W;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(t & 7);
    const int64_t p = t >> 3;
    const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / HW);
    const float* im = img + (int64_t)b * C * HW;
    float v[9];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int yy = y + dy - 1, xx = x + dx - 1;
        float s = 0.f;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          const int64_t o = (int64_t)yy * W + xx;
          if (C == 3)
            s = __fadd_rn(__fadd_rn(__fmul_rn(im[o], 0.299f), __fmul_rn(im[HW + o], 0.587f)),
                          __fmul_rn(im[2 * HW + o], 0.114f));
          else
            s = im[o];
        }
        v[dy * 3 + dx] = s;
      }
    uint32_t packed[4];
#pragma unroll
    for (int c2 = 0; c2 < 4; ++c2) {
      float r[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = g * 8 + c2 * 2 + h;
        float a = sb[c];
#pragma unroll
        for (int k = 0; k < 9; ++k) a = fmaf(sw[c * 9 + k], v[k], a);
        r[h] = fmaxf(a, 0.f);
        if constexpr (AFF) r[h] = fmaf(r[h], ss[c], sh[c]);
      }
      packed[c2] = pack_bf16(r[0], r[1]);
    }
    *reinterpret_cast<uint4*>(out + p * 64 + g * 8) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  }
}

// ---------------------------------------------------------------------------------------------
// implicit-GEMM convolution
// ---------------------------------------------------------------------------------------------
constexpr int SP_TY = 8, SP_TX = 16, SP_TM = SP_TY * SP_TX;  // output tile: 8 pixel rows x 16 columns
constexpr int SP_STAGES = 3;
constexpr int SP_THREADS = 256;
enum { SP_EP_RELU = 0, SP_EP_POOL = 1, SP_EP_SOFTMAX = 2, SP_EP_L2N = 3, SP_EP_RAW = 4 };

template <int BN>
__host__ __device__ constexpr int sp_stage_bytes() { return (SP_TM + BN) * 128; }
template <int BN>
__host__ __device__ constexpr int sp_smem_bytes() {
  constexpr int pipe = SP_STAGES * sp_stage_bytes<BN>();
  constexpr int stage = SP_TM * (BN + 1) * 4;
  return (pipe > stage ? pipe : stage) + 1024;  // + alignment slack
}

// row r, 16-byte chunk c of a 128-byte-swizzled K-major block
__device__ __forceinline__ int sw128(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }

// AFF: the staged values (after the ReLU of the encoder epilogues) become scale * v + shift before the epilogue
// proper.  SP_EP_RAW: conv + bias as fp32 [B, H, W, BN * tiles_n].
template <int BN, int EP, bool AFF = false>
__global__ void __launch_bounds__(SP_THREADS)
    sp_conv_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const __nv_bfloat16* __restrict__ w,
                   const float* __restrict__ bias, void* __restrict__ out, int H, int W, int Cin, int Cout, int ks,
                   int tiles_n, const float* __restrict__ scale, const float* __restrict__ shift) {
  extern __shared__ uint8_t sp_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sp_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int tn = blockIdx.y % tiles_n, n0 = tn * BN;
  const int y0 = (blockIdx.y / tiles_n) * SP_TY, x0 = blockIdx.x * SP_TX, b = blockIdx.z;
  const int cb_n = Cin / 64, nk = ks * ks * cb_n, Ktot = ks * ks * Cin, pad = ks / 2;
  const __nv_bfloat16* xb = x + (int64_t)b * H * W * ldx;

  auto load = [&](int kb, int s) {
    uint8_t* sa = smem + s * sp_stage_bytes<BN>();
    uint8_t* sb = sa + SP_TM * 128;
    const int tap = kb / cb_n, cb = kb % cb_n;
    const int dy = tap / ks - pad, dx = tap % ks - pad;
#pragma unroll
    for (int i = 0; i < SP_TM * 8 / SP_THREADS; ++i) {
      const int q = tid + i * SP_THREADS, r = q >> 3, c = q & 7;
      const int yy = y0 + (r >> 4) + dy, xx = x0 + (r & 15) + dx;
      const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
      const __nv_bfloat16* src = ok ? xb + ((int64_t)yy * W + xx) * ldx + cb * 64 + c * 8 : x;
      sp_cp16(sa + sw128(r, c), src, ok);
    }
#pragma unroll
    for (int i = 0; i < BN * 8 / SP_THREADS; ++i) {
      const int q = tid + i * SP_THREADS, r = q >> 3, c = q & 7;
      sp_cp16(sb + sw128(r, c), w + (int64_t)(n0 + r) * Ktot + kb * 64 + c * 8, true);
    }
  };

  constexpr int NSUB = BN >= 128 ? BN / 128 : 1;  // n128 wgmma per k-step (n64 for BN = 64)
  constexpr int NACC = BN >= 128 ? 64 : 32;
  float d[NSUB][NACC];
#pragma unroll
  for (int s = 0; s < NSUB; ++s)
#pragma unroll
    for (int i = 0; i < NACC; ++i) d[s][i] = 0.f;

#pragma unroll
  for (int s = 0; s < SP_STAGES - 1; ++s) {
    if (s < nk) load(s, s);
    sp_cp_commit();
  }
  for (int kb = 0; kb < nk; ++kb) {
    sp_cp_wait<SP_STAGES - 2>();
    fence_proxy_async_smem();
    __syncthreads();  // block kb has landed for every thread; the MMAs of kb - 1 have retired in every warpgroup
    const int nxt = kb + SP_STAGES - 1;
    if (nxt < nk) load(nxt, nxt % SP_STAGES);
    sp_cp_commit();
    const int s = kb % SP_STAGES;
    const uint32_t sa = smem_u32(smem + s * sp_stage_bytes<BN>());
    const uint64_t ad = make_smem_desc(sa + wg * 8192, 8192, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int sub = 0; sub < NSUB; ++sub) {
        const uint64_t bd = make_smem_desc(sa + SP_TM * 128 + sub * 16384, 8192, 1024);
        if constexpr (BN >= 128)
          wgmma_m64n128_ss<0, 0>(d[sub], ad + kk * 2, bd + kk * 2, (kb | kk) != 0);
        else
          wgmma_m64n64_ss<0, 0>(d[sub], ad + kk * 2, bd + kk * 2, (kb | kk) != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int sub = 0; sub < NSUB; ++sub) wgmma_hold(d[sub]);
  }
  sp_cp_wait<0>();
  __syncthreads();  // the pipeline buffers become the epilogue's staging tile

  // staging: st[m][c] = acc + bias (ReLU'd for the encoder convs), m = 16 * row + column of the pixel tile
  constexpr int LD = BN + 1;
  float* st = reinterpret_cast<float*>(smem);
  {
    const int rbase = wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int sub = 0; sub < NSUB; ++sub)
#pragma unroll
      for (int j = 0; j < NACC / 4; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int col = sub * 128 + 8 * j + 2 * (lane & 3) + c;
            float v = d[sub][4 * j + 2 * i + c] + bias[n0 + col];
            if (EP == SP_EP_RELU || EP == SP_EP_POOL) v = fmaxf(v, 0.f);
            if constexpr (AFF) v = fmaf(v, scale[n0 + col], shift[n0 + col]);
            st[(rbase + 8 * i) * LD + col] = v;
          }
  }
  __syncthreads();

  if constexpr (EP == SP_EP_RELU) {
    __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out) + (int64_t)b * H * W * Cout;
    for (int q = tid; q < SP_TM * BN / 2; q += SP_THREADS) {
      const int m = q / (BN / 2), c = 2 * (q % (BN / 2));
      const int yy = y0 + (m >> 4), xx = x0 + (m & 15);
      if (yy < H && xx < W)
        *reinterpret_cast<uint32_t*>(o + ((int64_t)yy * W + xx) * Cout + n0 + c) =
            pack_bf16(st[m * LD + c], st[m * LD + c + 1]);
    }
  } else if constexpr (EP == SP_EP_POOL) {
    const int Hp = H / 2, Wp = W / 2;
    __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out) + (int64_t)b * Hp * Wp * Cout;
    for (int q = tid; q < (SP_TM / 4) * BN / 2; q += SP_THREADS) {
      const int p = q / (BN / 2), c = 2 * (q % (BN / 2));
      const int py = p >> 3, px = p & 7;
      const int yy = y0 / 2 + py, xx = x0 / 2 + px;
      if (yy < Hp && xx < Wp) {
        const int m = (2 * py) * 16 + 2 * px;
        float v0 = fmaxf(fmaxf(st[m * LD + c], st[(m + 1) * LD + c]),
                         fmaxf(st[(m + 16) * LD + c], st[(m + 17) * LD + c]));
        float v1 = fmaxf(fmaxf(st[m * LD + c + 1], st[(m + 1) * LD + c + 1]),
                         fmaxf(st[(m + 16) * LD + c + 1], st[(m + 17) * LD + c + 1]));
        *reinterpret_cast<uint32_t*>(o + ((int64_t)yy * Wp + xx) * Cout + n0 + c) = pack_bf16(v0, v1);
      }
    }
  } else if constexpr (EP == SP_EP_SOFTMAX) {
    // 65 logits per pixel; channel c < 64 goes to score pixel (8 y + c / 8, 8 x + c % 8)
    __shared__ float mx[SP_TM], inv[SP_TM];
    if (tid < SP_TM) {
      const float* l = st + tid * LD;
      float m = l[0];
      for (int c = 1; c < 65; ++c) m = fmaxf(m, l[c]);
      float s = 0.f;
      for (int c = 0; c < 65; ++c) s += expf(l[c] - m);
      mx[tid] = m;
      inv[tid] = s;
    }
    __syncthreads();
    float* o = static_cast<float*>(out) + (int64_t)b * (8 * H) * (8 * W);
    for (int q = tid; q < SP_TM * 64; q += SP_THREADS) {
      // output order (tile row, sub-row, tile column, sub-column): each 128-float run is one score row
      const int cx = q & 7, tx = (q >> 3) & 15, cy = (q >> 7) & 7, ty = q >> 10;
      const int yy = y0 + ty, xx = x0 + tx;
      if (yy < H && xx < W) {
        const int m = ty * 16 + tx;
        o[(int64_t)(8 * yy + cy) * (8 * W) + 8 * xx + cx] = expf(st[m * LD + cy * 8 + cx] - mx[m]) / inv[m];
      }
    }
  } else if constexpr (EP == SP_EP_RAW) {
    const int ld = BN * tiles_n;
    float* o = static_cast<float*>(out) + (int64_t)b * H * W * ld;
    for (int q = tid; q < SP_TM * BN / 4; q += SP_THREADS) {
      const int m = q / (BN / 4), c = 4 * (q % (BN / 4));
      const int yy = y0 + (m >> 4), xx = x0 + (m & 15);
      if (yy < H && xx < W)
        *reinterpret_cast<float4*>(o + ((int64_t)yy * W + xx) * ld + n0 + c) =
            make_float4(st[m * LD + c], st[m * LD + c + 1], st[m * LD + c + 2], st[m * LD + c + 3]);
    }
  } else {
    // L2 normalisation over the BN (= Cout) channels of a pixel: one warp per pixel, fp32 NHWC out
    float* o = static_cast<float*>(out) + (int64_t)b * H * W * Cout;
    for (int m = warp; m < SP_TM; m += SP_THREADS / 32) {
      const int yy = y0 + (m >> 4), xx = x0 + (m & 15);
      if (yy >= H || xx >= W) continue;
      float ss = 0.f;
      for (int c = lane; c < BN; c += 32) ss += st[m * LD + c] * st[m * LD + c];
      ss = warp_sum(ss);
      const float r = 1.f / fmaxf(sqrtf(ss), 1e-12f);
      for (int c = lane; c < BN; c += 32) o[((int64_t)yy * W + xx) * Cout + c] = st[m * LD + c] * r;
    }
  }
}

template <int BN, int EP, bool AFF>
static int launch_sp_conv(const __nv_bfloat16* x, int ldx, const __nv_bfloat16* w, const float* bias,
                          const float* scale, const float* shift, void* out, int B, int H, int W, int Cin, int Cout,
                          int ks, int tiles_n, cudaStream_t st) {
  auto k = sp_conv_kernel<BN, EP, AFF>;
  constexpr int smem = sp_smem_bytes<BN>();
  if (ensure_dyn_smem(reinterpret_cast<const void*>(k), smem)) return kErrCuda;
  dim3 grid((W + SP_TX - 1) / SP_TX, ((H + SP_TY - 1) / SP_TY) * tiles_n, B);
  k<<<grid, SP_THREADS, smem, st>>>(x, ldx, w, bias, out, H, W, Cin, Cout, ks, tiles_n, scale, shift);
  return check_launch("sp_conv");
}

// the shape checks and instantiation choice of lgb200_sp_conv (AFF false) and lgb200_spo_conv (AFF true, or RAW)
template <bool AFF>
static int sp_conv_dispatch(const void* x, int ldx, const void* weight, const float* bias, const float* scale,
                            const float* shift, void* out, int B, int H, int W, int Cin, int Cout, int ksize,
                            int epilogue, cudaStream_t stream) {
  LGB_REQUIRE(x && weight && bias && out, kErrInvalid, "sp_conv: null pointer");
  LGB_REQUIRE(!AFF || epilogue == SP_EP_RAW || (scale && shift), kErrInvalid, "sp_conv: null scale / shift");
  LGB_REQUIRE(B > 0 && H > 0 && W > 0 && B <= 65535, kErrInvalid, "sp_conv: bad extents B=%d H=%d W=%d", B, H, W);
  LGB_REQUIRE(ksize == 1 || ksize == 3, kErrInvalid, "sp_conv: ksize %d (1 or 3)", ksize);
  LGB_REQUIRE(Cin % 64 == 0 && Cin > 0 && ldx >= Cin && ldx % 8 == 0, kErrInvalid,
              "sp_conv: Cin %d must be a multiple of 64 and ldx %d >= Cin a multiple of 8", Cin, ldx);
  LGB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(weight)) & 15) == 0, kErrInvalid,
              "sp_conv: x and weight must be 16-byte aligned");
  const int ty = (H + SP_TY - 1) / SP_TY;
  auto grid_ok = [&](int tiles_n) { return (int64_t)ty * tiles_n <= 65535; };
  const __nv_bfloat16 *xb = (const __nv_bfloat16*)x, *wb = (const __nv_bfloat16*)weight;
  switch (epilogue) {
    case SP_EP_RELU:
    case SP_EP_POOL: {
      LGB_REQUIRE(Cout % 64 == 0, kErrInvalid, "sp_conv: Cout %d must be a multiple of 64", Cout);
      if (Cout == 64) {
        LGB_REQUIRE(grid_ok(1), kErrInvalid, "sp_conv: image too tall");
        return epilogue == SP_EP_RELU
                   ? launch_sp_conv<64, SP_EP_RELU, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout,
                                                         ksize, 1, stream)
                   : launch_sp_conv<64, SP_EP_POOL, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout,
                                                         ksize, 1, stream);
      }
      LGB_REQUIRE(Cout % 128 == 0 && grid_ok(Cout / 128), kErrInvalid, "sp_conv: Cout %d (64 or a multiple of 128)",
                  Cout);
      return epilogue == SP_EP_RELU
                 ? launch_sp_conv<128, SP_EP_RELU, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout,
                                                        ksize, Cout / 128, stream)
                 : launch_sp_conv<128, SP_EP_POOL, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout,
                                                        ksize, Cout / 128, stream);
    }
    case SP_EP_SOFTMAX:
      LGB_REQUIRE(Cout == 65 && grid_ok(1), kErrInvalid, "sp_conv: the softmax epilogue takes Cout 65 (got %d)", Cout);
      return launch_sp_conv<128, SP_EP_SOFTMAX, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout, ksize,
                                                     1, stream);
    case SP_EP_L2N:
      LGB_REQUIRE(Cout == 256 && grid_ok(1), kErrInvalid, "sp_conv: the normalising epilogue takes Cout 256 (got %d)",
                  Cout);
      LGB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, kErrInvalid, "sp_conv: out must be 16-byte aligned");
      return launch_sp_conv<256, SP_EP_L2N, AFF>(xb, ldx, wb, bias, scale, shift, out, B, H, W, Cin, Cout, ksize, 1,
                                                 stream);
    case SP_EP_RAW:
      LGB_REQUIRE(Cout > 0 && grid_ok((Cout + 127) / 128), kErrInvalid, "sp_conv: raw epilogue, Cout %d", Cout);
      LGB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, kErrInvalid, "sp_conv: out must be 16-byte aligned");
      return launch_sp_conv<128, SP_EP_RAW, false>(xb, ldx, wb, bias, nullptr, nullptr, out, B, H, W, Cin, Cout, ksize,
                                                   (Cout + 127) / 128, stream);
    default:
      LGB_REQUIRE(false, kErrInvalid, "sp_conv: unknown epilogue %d", epilogue);
  }
}

// ---------------------------------------------------------------------------------------------
// NMS (simple_nms) + border removal
// ---------------------------------------------------------------------------------------------
constexpr int SP_NMS_E = 96;  // extended tile edge (output tile + 2 * 5r halo)
constexpr int SP_NMS_THREADS = 512;
constexpr int SP_NMS_CELLS = SP_NMS_E * SP_NMS_E;
constexpr int SP_NMS_SMEM = SP_NMS_CELLS * (4 * 4 + 3);

// dst = max over the (2r+1)^2 window clipped to the extended tile (cells outside the image hold -inf / 0)
template <typename T>
__device__ void sp_boxmax(const T* src, T* tmp, T* dst, int r) {
  for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
    const int y = i / SP_NMS_E, x = i % SP_NMS_E;
    T m = src[i];
    for (int k = max(0, x - r); k <= min(SP_NMS_E - 1, x + r); ++k) m = src[y * SP_NMS_E + k] > m ? src[y * SP_NMS_E + k] : m;
    tmp[i] = m;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
    const int y = i / SP_NMS_E, x = i % SP_NMS_E;
    T m = tmp[i];
    for (int k = max(0, y - r); k <= min(SP_NMS_E - 1, y + r); ++k) m = tmp[k * SP_NMS_E + x] > m ? tmp[k * SP_NMS_E + x] : m;
    dst[i] = m;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(SP_NMS_THREADS)
    sp_nms_kernel(const float* __restrict__ scores, const float* __restrict__ image_size, float* __restrict__ out,
                  int H, int W, int r, int rb) {
  extern __shared__ __align__(16) uint8_t nms_smem[];
  float* S = reinterpret_cast<float*>(nms_smem);
  float* X = S + SP_NMS_CELLS;
  float* Tf = X + SP_NMS_CELLS;
  float* Y = Tf + SP_NMS_CELLS;
  uint8_t* M = reinterpret_cast<uint8_t*>(Y + SP_NMS_CELLS);
  uint8_t* Tu = M + SP_NMS_CELLS;
  uint8_t* U = Tu + SP_NMS_CELLS;
  const int halo = 5 * r, T = SP_NMS_E - 2 * halo;
  const int b = blockIdx.z, oy = blockIdx.y * T - halo, ox = blockIdx.x * T - halo;
  const float* sb = scores + (int64_t)b * H * W;
  const float ninf = -INFINITY;
  for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
    const int y = oy + i / SP_NMS_E, x = ox + i % SP_NMS_E;
    S[i] = (y >= 0 && y < H && x >= 0 && x < W) ? sb[(int64_t)y * W + x] : ninf;
  }
  __syncthreads();
  sp_boxmax(S, Tf, Y, r);
  for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
    const int y = oy + i / SP_NMS_E, x = ox + i % SP_NMS_E;
    M[i] = (y >= 0 && y < H && x >= 0 && x < W) && S[i] == Y[i];
  }
  __syncthreads();
  for (int round = 0; round < 2; ++round) {
    sp_boxmax(M, Tu, U, r);  // U: suppression mask
    for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
      const int y = oy + i / SP_NMS_E, x = ox + i % SP_NMS_E;
      X[i] = (y >= 0 && y < H && x >= 0 && x < W) ? (U[i] ? 0.f : S[i]) : ninf;
    }
    __syncthreads();
    sp_boxmax(X, Tf, Y, r);
    for (int i = threadIdx.x; i < SP_NMS_CELLS; i += blockDim.x) {
      const int y = oy + i / SP_NMS_E, x = ox + i % SP_NMS_E;
      if ((y >= 0 && y < H && x >= 0 && x < W) && X[i] == Y[i] && !U[i]) M[i] = 1;
    }
    __syncthreads();
  }
  // border removal (scores[:, :rb] = -1 etc.); with image_size the far borders start at int(h) - rb, int(w) - rb,
  // resolved like a Python slice start
  int ylim = H - rb, xlim = W - rb;
  if (image_size != nullptr) {
    ylim = (int)image_size[2 * b + 1] - rb;
    xlim = (int)image_size[2 * b] - rb;
    ylim = ylim < 0 ? max(ylim + H, 0) : ylim;
    xlim = xlim < 0 ? max(xlim + W, 0) : xlim;
  }
  for (int i = threadIdx.x; i < T * T; i += blockDim.x) {
    const int ly = halo + i / T, lx = halo + i % T;
    const int y = oy + ly, x = ox + lx;
    if (y >= H || x >= W) continue;
    const int c = ly * SP_NMS_E + lx;
    float v = M[c] ? S[c] : 0.f;
    if (rb > 0 && (y < rb || x < rb || y >= ylim || x >= xlim)) v = -1.f;
    out[(int64_t)b * H * W + (int64_t)y * W + x] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// selection
// ---------------------------------------------------------------------------------------------
constexpr int SP_SEL_THREADS = 1024;

__device__ __forceinline__ uint32_t sp_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// block-wide exclusive scan of one flag per thread; returns the prefix, *total the block sum
__device__ __forceinline__ int sp_block_scan(int f, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  const int pre = __popc(bal & ((1u << lane) - 1));
  if (lane == 0) warp_tot[warp] = __popc(bal);
  __syncthreads();
  if (warp == 0) {
    int v = warp_tot[lane];
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    warp_tot[32 + lane] = inc - v;
    if (lane == 31) warp_tot[64] = inc;
  }
  __syncthreads();
  const int r = warp_tot[32 + warp] + pre;
  *total = warp_tot[64];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(SP_SEL_THREADS)
    sp_count_kernel(const float* __restrict__ nms, float thr, int* __restrict__ counts, int HW) {
  __shared__ int acc;
  if (threadIdx.x == 0) acc = 0;
  __syncthreads();
  const float* v = nms + (int64_t)blockIdx.x * HW;
  int c = 0;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) c += v[i] > thr;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) atomicAdd(&acc, c);
  __syncthreads();
  if (threadIdx.x == 0) counts[blockIdx.x] = acc;
}

// One CTA per image.  k <= 0 or count <= k: every candidate in row-major order (the reference's torch.where order,
// which top_k_keypoints keeps when it has no more than k).  Otherwise the k largest in descending score order, exact
// ties broken towards the lower row-major index.  Slots [kept, cap) are padding: with `uniform` ([B, cap, 2] in
// [0, 1)), coordinate i is drawn in [min, max] of the kept keypoints' coordinate i, or [0, *pad_hi] when none is
// kept (pad_to_length's random_c); scores 0.
__global__ void __launch_bounds__(SP_SEL_THREADS)
    sp_select_kernel(const float* __restrict__ nms, float thr, int k, int cap, const float* __restrict__ uniform,
                     const float* __restrict__ pad_hi, float* __restrict__ kpts, float* __restrict__ scores,
                     int* __restrict__ counts, int H, int W) {
  extern __shared__ __align__(16) unsigned long long sel[];
  __shared__ int warp_tot[65];
  __shared__ unsigned hist[256];
  __shared__ int s_digit, s_rem;
  __shared__ float s_red[4][32];
  const int b = blockIdx.x, tid = threadIdx.x, HW = H * W;
  const float* v = nms + (int64_t)b * HW;
  float* kp = kpts + (int64_t)b * cap * 2;
  float* sc = scores + (int64_t)b * cap;

  int cnt = 0;
  {
    int c = 0;
    for (int i = tid; i < HW; i += blockDim.x) c += v[i] > thr;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((tid & 31) == 0) warp_tot[tid >> 5] = c;
    __syncthreads();
    for (int w = 0; w < SP_SEL_THREADS / 32; ++w) cnt += warp_tot[w];
    __syncthreads();
  }
  int kept;
  if (k <= 0 || cnt <= k) {
    kept = min(cnt, cap);
    int base = 0;
    for (int i0 = 0; i0 < HW; i0 += blockDim.x) {
      const int i = i0 + tid;
      const float s = i < HW ? v[i] : 0.f;
      const int f = i < HW && s > thr;
      int tot;
      const int pos = base + sp_block_scan(f, warp_tot, &tot);
      if (f && pos < cap) {
        kp[2 * pos] = (float)(i % W);
        kp[2 * pos + 1] = (float)(i / W);
        sc[pos] = s;
      }
      base += tot;
    }
  } else {
    kept = min(k, cap);
    // radix select of the k-th largest key, 8 bits at a time from the top
    uint32_t prefix = 0, pmask = 0;
    int rem = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = tid; i < HW; i += blockDim.x) {
        const float s = v[i];
        if (!(s > thr)) continue;
        const uint32_t key = sp_key(s);
        if ((key & pmask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        int acc = 0, d = 255;
        for (; d > 0; --d) {
          if (acc + (int)hist[d] >= rem) break;
          acc += hist[d];
        }
        s_digit = d;
        s_rem = rem - acc;
      }
      __syncthreads();
      prefix |= (uint32_t)s_digit << shift;
      pmask |= 255u << shift;
      rem = s_rem;
      __syncthreads();
    }
    // gather: every key above the k-th, and the first `rem` equal to it in row-major order
    int base = 0, eq_base = 0;
    for (int i0 = 0; i0 < HW; i0 += blockDim.x) {
      const int i = i0 + tid;
      const float s = i < HW ? v[i] : 0.f;
      const bool cand = i < HW && s > thr;
      const uint32_t key = cand ? sp_key(s) : 0u;
      const int eq = cand && key == prefix;
      int eq_tot;
      const int eq_rank = eq_base + sp_block_scan(eq, warp_tot, &eq_tot);
      const int f = (cand && key > prefix) || (eq && eq_rank < rem);
      int tot;
      const int pos = base + sp_block_scan(f, warp_tot, &tot);
      if (f) sel[pos] = ((unsigned long long)key << 32) | (0xFFFFFFFFu - (uint32_t)i);
      base += tot;
      eq_base += eq_tot;
    }
    // bitonic sort, descending, of the k entries padded with zeros to a power of two
    int P = 1;
    while (P < k) P <<= 1;
    for (int i = k + tid; i < P; i += blockDim.x) sel[i] = 0ull;
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = tid; i < P / 2; i += blockDim.x) {
          const int lo = 2 * i - (i & (stride - 1));
          const int hi = lo + stride;
          const bool desc = (lo & size) == 0;
          const unsigned long long a = sel[lo], c = sel[hi];
          if ((a < c) == desc) {
            sel[lo] = c;
            sel[hi] = a;
          }
        }
        __syncthreads();
      }
    }
    for (int j = tid; j < kept; j += blockDim.x) {
      const uint32_t idx = 0xFFFFFFFFu - (uint32_t)(sel[j] & 0xFFFFFFFFull);
      kp[2 * j] = (float)(idx % W);
      kp[2 * j + 1] = (float)(idx / W);
      sc[j] = v[idx];
    }
  }
  if (tid == 0 && counts) counts[b] = kept;
  if (cap <= kept) return;
  __syncthreads();
  // padding
  float lo[2] = {0.f, 0.f}, hi[2] = {pad_hi ? *pad_hi : 0.f, pad_hi ? *pad_hi : 0.f};
  if (kept > 0) {
    float mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
    for (int j = tid; j < kept; j += blockDim.x) {
      mn0 = fminf(mn0, kp[2 * j]);
      mx0 = fmaxf(mx0, kp[2 * j]);
      mn1 = fminf(mn1, kp[2 * j + 1]);
      mx1 = fmaxf(mx1, kp[2 * j + 1]);
    }
    for (int o = 16; o > 0; o >>= 1) {
      mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
      mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
    }
    if ((tid & 31) == 0) {
      s_red[0][tid >> 5] = mn0;
      s_red[1][tid >> 5] = mx0;
      s_red[2][tid >> 5] = mn1;
      s_red[3][tid >> 5] = mx1;
    }
    __syncthreads();
    lo[0] = lo[1] = INFINITY;
    hi[0] = hi[1] = -INFINITY;
    for (int w = 0; w < SP_SEL_THREADS / 32; ++w) {
      lo[0] = fminf(lo[0], s_red[0][w]);
      hi[0] = fmaxf(hi[0], s_red[1][w]);
      lo[1] = fminf(lo[1], s_red[2][w]);
      hi[1] = fmaxf(hi[1], s_red[3][w]);
    }
  }
  const float* u = uniform ? uniform + (int64_t)b * cap * 2 : nullptr;
  for (int j = kept + tid; j < cap; j += blockDim.x) {
    kp[2 * j] = u ? lo[0] + u[2 * j] * (hi[0] - lo[0]) : 0.f;
    kp[2 * j + 1] = u ? lo[1] + u[2 * j + 1] * (hi[1] - lo[1]) : 0.f;
    sc[j] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// descriptor sampling
// ---------------------------------------------------------------------------------------------
// one warp per keypoint, C = 32 * CPL channels (lane: CPL consecutive channels)
template <int CPL>
__global__ void __launch_bounds__(256) sp_sample_kernel(const float* __restrict__ desc, const float* __restrict__ kpts,
                                                        float* __restrict__ out, int B, int K, int h, int w,
                                                        int legacy) {
  constexpr int C = 32 * CPL;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= B * K) return;
  const int b = gw / K;
  float kx = kpts[2 * (int64_t)gw], ky = kpts[2 * (int64_t)gw + 1];
  float ix, iy;
  if (legacy) {  // sample_descriptors: align_corners=True
    kx = (kx - 8.f / 2 + 0.5f) / ((float)w * 8 - 8.f / 2 - 0.5f);
    ky = (ky - 8.f / 2 + 0.5f) / ((float)h * 8 - 8.f / 2 - 0.5f);
    kx = kx * 2 - 1;
    ky = ky * 2 - 1;
    ix = ((kx + 1) / 2) * (w - 1);
    iy = ((ky + 1) / 2) * (h - 1);
  } else {  // sample_descriptors_fix_sampling: align_corners=False
    kx = kx / ((float)w * 8) * 2 - 1;
    ky = ky / ((float)h * 8) * 2 - 1;
    ix = ((kx + 1) * w - 1) / 2;
    iy = ((ky + 1) * h - 1) / 2;
  }
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy;
  const float wx1 = ix - fx, wx0 = (fx + 1) - ix, wy1 = iy - fy, wy0 = (fy + 1) - iy;
  const float wt[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};
  const int tx[4] = {x0, x0 + 1, x0, x0 + 1}, ty[4] = {y0, y0, y0 + 1, y0 + 1};
  float acc[CPL];
#pragma unroll
  for (int c = 0; c < CPL; ++c) acc[c] = 0.f;
  const float* db = desc + (int64_t)b * h * w * C;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    if (tx[t] < 0 || tx[t] >= w || ty[t] < 0 || ty[t] >= h) continue;
    const float* p = db + ((int64_t)ty[t] * w + tx[t]) * C + lane * CPL;
#pragma unroll
    for (int c = 0; c < CPL; c += 4) {
      const float4 q = *reinterpret_cast<const float4*>(p + c);
      acc[c] += wt[t] * q.x;
      acc[c + 1] += wt[t] * q.y;
      acc[c + 2] += wt[t] * q.z;
      acc[c + 3] += wt[t] * q.w;
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c) ss += acc[c] * acc[c];
  ss = warp_sum(ss);
  const float r = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  float* o = out + (int64_t)gw * C + lane * CPL;
#pragma unroll
  for (int c = 0; c < CPL; c += 4)
    *reinterpret_cast<float4*>(o + c) = make_float4(acc[c] * r, acc[c + 1] * r, acc[c + 2] * r, acc[c + 3] * r);
}

// ---------------------------------------------------------------------------------------------
// training-mode BatchNorm of SuperPoint-open from batch statistics
// ---------------------------------------------------------------------------------------------
// sums = [sum x (C) | sum x^2 (C) | count] in fp64 (lgb200_bn_stats, possibly summed across ranks): mean and biased
// variance as bn_relu_fwd_kernel forms them, y = (x - mean) rstd gamma + beta.  Every CTA fills its own copy.
enum { SPO_BN_PLAIN = 0, SPO_BN_POOL = 1, SPO_BN_SOFTMAX = 2, SPO_BN_L2N = 3 };
constexpr int SPO_BN_MAXC = 512;
constexpr int SPO_BN_THREADS = 256;

struct SpoBnSmem {
  float mu[SPO_BN_MAXC], rs[SPO_BN_MAXC], g[SPO_BN_MAXC], b[SPO_BN_MAXC];
};

__device__ __forceinline__ void spo_bn_setup(SpoBnSmem& sm, const double* __restrict__ sums,
                                             const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                             int C) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const double n = sums[2 * C];
    const double m = sums[c] / n;
    const double var = fmax(sums[C + c] / n - m * m, 0.0);
    sm.mu[c] = (float)m;
    sm.rs[c] = 1.f / sqrtf((float)var + eps);
    sm.g[c] = gamma[c];
    sm.b[c] = beta[c];
  }
  __syncthreads();
}

__device__ __forceinline__ float spo_bn(const SpoBnSmem& sm, int c, float v) {
  return fmaf((v - sm.mu[c]) * sm.rs[c], sm.g[c], sm.b[c]);
}

__device__ __forceinline__ void spo_unpack8(const uint4& u, float* v) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __uint_as_float(w[i] << 16);
    v[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
}

// PLAIN: bf16 [B, H, W, C] -> bf16 [B, H, W, C].  POOL: -> bf16 [B, H/2, W/2, C], the 2x2 max of the normalised
// values (floor sizes).  One thread per 8 channels of an output pixel, 16-byte loads and stores.
template <int OP>
__global__ void __launch_bounds__(SPO_BN_THREADS)
    spo_bn_nhwc_kernel(const __nv_bfloat16* __restrict__ x, const double* __restrict__ sums,
                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                       __nv_bfloat16* __restrict__ out, int B, int H, int W, int C) {
  __shared__ SpoBnSmem sm;
  spo_bn_setup(sm, sums, gamma, beta, eps, C);
  // C / 8 divides the grid stride (C a power of two <= 512), so a thread keeps its 8 channels
  const int cv = C / 8;
  const int Ho = OP == SPO_BN_POOL ? H / 2 : H, Wo = OP == SPO_BN_POOL ? W / 2 : W;
  const int64_t np = (int64_t)B * Ho * Wo;
  const int start = blockIdx.x * blockDim.x + threadIdx.x, c0 = (start % cv) * 8;
  const int pstride = gridDim.x * blockDim.x / cv;
  for (int64_t p = start / cv; p < np; p += pstride) {
    float r[8];
    if constexpr (OP == SPO_BN_PLAIN) {
      float v[8];
      spo_unpack8(*reinterpret_cast<const uint4*>(x + p * C + c0), v);
#pragma unroll
      for (int e = 0; e < 8; ++e) r[e] = spo_bn(sm, c0 + e, v[e]);
    } else {
      const int px = (int)(p % Wo), py = (int)((p / Wo) % Ho), b = (int)(p / ((int64_t)Wo * Ho));
      const __nv_bfloat16* xb = x + (((int64_t)b * H + 2 * py) * W + 2 * px) * C + c0;
#pragma unroll
      for (int e = 0; e < 8; ++e) r[e] = -INFINITY;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[8];
        spo_unpack8(*reinterpret_cast<const uint4*>(xb + ((int64_t)(q >> 1) * W + (q & 1)) * C), v);
#pragma unroll
        for (int e = 0; e < 8; ++e) r[e] = fmaxf(r[e], spo_bn(sm, c0 + e, v[e]));
      }
    }
    *reinterpret_cast<uint4*>(out + p * C + c0) =
        make_uint4(pack_bf16(r[0], r[1]), pack_bf16(r[2], r[3]), pack_bf16(r[4], r[5]), pack_bf16(r[6], r[7]));
  }
}

// SOFTMAX: logits fp32 [B, h, w, 128] (channels 65.. ignored) -> normalise the 65 -> softmax -> depth-to-space score
// map fp32 [B, 8h, 8w].  16 lanes per pixel: lane j holds channels 4j .. 4j + 3 (score row j / 2, columns
// 4 (j & 1) .. + 3 of the pixel's 8x8 cell) and every lane the dustbin, channel 64.
__global__ void __launch_bounds__(SPO_BN_THREADS)
    spo_bn_softmax_kernel(const float* __restrict__ x, const double* __restrict__ sums,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          float* __restrict__ out, int B, int h, int w) {
  __shared__ SpoBnSmem sm;
  spo_bn_setup(sm, sums, gamma, beta, eps, 65);
  const int lane = threadIdx.x & 31, j = lane & 15;
  const unsigned mask = 0xFFFFu << (lane & 16);
  const int64_t np = (int64_t)B * h * w;
  for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4; p < np;
       p += ((int64_t)gridDim.x * blockDim.x) >> 4) {
    const float4 q = *reinterpret_cast<const float4*>(x + p * 128 + 4 * j);
    float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) v[t] = spo_bn(sm, 4 * j + t, v[t]);
    const float dust = spo_bn(sm, 64, x[p * 128 + 64]);
    float m = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(mask, m, o));
    m = fmaxf(m, dust);
    float e[4], s;
#pragma unroll
    for (int t = 0; t < 4; ++t) e[t] = expf(v[t] - m);
    s = (e[0] + e[1]) + (e[2] + e[3]);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(mask, s, o);
    s += expf(dust - m);
    const int xx = (int)(p % w), yy = (int)((p / w) % h), b = (int)(p / ((int64_t)w * h));
    float* o = out + ((int64_t)b * 8 * h + 8 * yy + (j >> 1)) * (8 * (int64_t)w) + 8 * xx + 4 * (j & 1);
    *reinterpret_cast<float4*>(o) = make_float4(e[0] / s, e[1] / s, e[2] / s, e[3] / s);
  }
}

// L2N: fp32 [T, 256] -> normalise -> divide by max(||.||, 1e-12) per pixel, fp32 [T, 256].  One warp per pixel.
__global__ void __launch_bounds__(SPO_BN_THREADS)
    spo_bn_l2n_kernel(const float* __restrict__ x, const double* __restrict__ sums, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float eps, float* __restrict__ out, int64_t T) {
  __shared__ SpoBnSmem sm;
  spo_bn_setup(sm, sums, gamma, beta, eps, 256);
  const int lane = threadIdx.x & 31;
  for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < T;
       p += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const float* xp = x + p * 256 + 8 * lane;
    const float4 a = *reinterpret_cast<const float4*>(xp), c = *reinterpret_cast<const float4*>(xp + 4);
    float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] = spo_bn(sm, 8 * lane + e, v[e]);
      ss += v[e] * v[e];
    }
    ss = warp_sum(ss);
    const float r = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    float* op = out + p * 256 + 8 * lane;
    *reinterpret_cast<float4*>(op) = make_float4(v[0] * r, v[1] * r, v[2] * r, v[3] * r);
    *reinterpret_cast<float4*>(op + 4) = make_float4(v[4] * r, v[5] * r, v[6] * r, v[7] * r);
  }
}

static int sp_conv1a_launch(bool aff, const float* image, int C, const float* weight, const float* bias,
                            const float* scale, const float* shift, void* out, int B, int H, int W,
                            cudaStream_t stream) {
  LGB_REQUIRE(image && weight && bias && out, kErrInvalid, "sp_conv1a: null pointer");
  LGB_REQUIRE(!aff || (scale && shift), kErrInvalid, "sp_conv1a: null scale / shift");
  LGB_REQUIRE(C == 1 || C == 3, kErrInvalid, "sp_conv1a: image has %d channels (1 or 3)", C);
  LGB_REQUIRE(B > 0 && H > 0 && W > 0, kErrInvalid, "sp_conv1a: empty image");
  LGB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, kErrInvalid, "sp_conv1a: out must be 16-byte aligned");
  const int64_t n = (int64_t)B * H * W * 8;
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, 65535LL * 16);
  if (aff)
    sp_conv1a_kernel<true><<<blocks, 256, 0, stream>>>(image, C, weight, bias, static_cast<__nv_bfloat16*>(out), B,
                                                        H, W, scale, shift);
  else
    sp_conv1a_kernel<false><<<blocks, 256, 0, stream>>>(image, C, weight, bias, static_cast<__nv_bfloat16*>(out), B,
                                                         H, W, nullptr, nullptr);
  return check_launch("sp_conv1a");
}

}  // namespace lgb

using namespace lgb;

extern "C" {

int lgb200_sp_conv1a(const float* image, int C, const float* weight, const float* bias, void* out, int B, int H,
                     int W, cudaStream_t stream) {
  return sp_conv1a_launch(false, image, C, weight, bias, nullptr, nullptr, out, B, H, W, stream);
}

int lgb200_sp_conv(const void* x, int ldx, const void* weight, const float* bias, void* out, int B, int H, int W,
                   int Cin, int Cout, int ksize, int epilogue, cudaStream_t stream) {
  LGB_REQUIRE(epilogue != SP_EP_RAW, kErrInvalid, "sp_conv: unknown epilogue %d", epilogue);
  return sp_conv_dispatch<false>(x, ldx, weight, bias, nullptr, nullptr, out, B, H, W, Cin, Cout, ksize, epilogue,
                                 stream);
}

int lgb200_sp_nms(const float* scores, const float* image_size, float* out, int B, int H, int W, int radius,
                  int remove_borders, cudaStream_t stream) {
  LGB_REQUIRE(scores && out && scores != out, kErrInvalid, "sp_nms: null or aliased pointer");
  LGB_REQUIRE(B > 0 && H > 0 && W > 0 && B <= 65535, kErrInvalid, "sp_nms: bad extents");
  LGB_REQUIRE(radius >= 0 && 10 * radius < SP_NMS_E, kErrUnsupported, "sp_nms: radius %d (at most %d)", radius,
              (SP_NMS_E - 1) / 10);
  LGB_REQUIRE(remove_borders >= 0, kErrInvalid, "sp_nms: remove_borders %d", remove_borders);
  const int T = SP_NMS_E - 10 * radius;
  if (ensure_dyn_smem(reinterpret_cast<const void*>(sp_nms_kernel), SP_NMS_SMEM)) return kErrCuda;
  dim3 grid((W + T - 1) / T, (H + T - 1) / T, B);
  LGB_REQUIRE(grid.y <= 65535, kErrInvalid, "sp_nms: image too tall");
  sp_nms_kernel<<<grid, SP_NMS_THREADS, SP_NMS_SMEM, stream>>>(scores, image_size, out, H, W, radius,
                                                               remove_borders);
  return check_launch("sp_nms");
}

int lgb200_sp_count(const float* nms, float threshold, int* counts, int B, int H, int W, cudaStream_t stream) {
  LGB_REQUIRE(nms && counts && B > 0 && H > 0 && W > 0, kErrInvalid, "sp_count: bad arguments");
  LGB_REQUIRE((int64_t)H * W < (1LL << 31), kErrInvalid, "sp_count: image too large");
  sp_count_kernel<<<B, SP_SEL_THREADS, 0, stream>>>(nms, threshold, counts, H * W);
  return check_launch("sp_count");
}

int lgb200_sp_select(const float* nms, float threshold, int k, int cap, const float* uniform, const float* pad_hi,
                     float* keypoints, float* scores, int* counts, int B, int H, int W, cudaStream_t stream) {
  LGB_REQUIRE(nms && keypoints && scores && B > 0 && H > 0 && W > 0 && cap > 0, kErrInvalid,
              "sp_select: bad arguments");
  LGB_REQUIRE((int64_t)H * W < (1LL << 31), kErrInvalid, "sp_select: image too large");
  LGB_REQUIRE(k <= LGB200_SP_MAX_K, kErrUnsupported, "sp_select: k %d (at most %d)", k, LGB200_SP_MAX_K);
  int P = 1;
  while (k > 0 && P < k) P <<= 1;
  const int smem = k > 0 ? P * 8 : 0;
  if (ensure_dyn_smem(reinterpret_cast<const void*>(sp_select_kernel), smem > 0 ? smem : 8)) return kErrCuda;
  sp_select_kernel<<<B, SP_SEL_THREADS, smem, stream>>>(nms, threshold, k, cap, uniform, pad_hi, keypoints, scores,
                                                        counts, H, W);
  return check_launch("sp_select");
}

int lgb200_sp_sample(const float* desc, const float* keypoints, float* out, int B, int K, int h, int w, int C,
                     int legacy, cudaStream_t stream) {
  LGB_REQUIRE(desc && keypoints && out, kErrInvalid, "sp_sample: null pointer");
  LGB_REQUIRE(B > 0 && K >= 0 && h > 0 && w > 0, kErrInvalid, "sp_sample: bad extents");
  LGB_REQUIRE(C == 256 || C == 128, kErrUnsupported, "sp_sample: C %d (128 or 256)", C);
  LGB_REQUIRE(((reinterpret_cast<uintptr_t>(desc) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, kErrInvalid,
              "sp_sample: desc and out must be 16-byte aligned");
  if (K == 0) return 0;
  const int64_t warps = (int64_t)B * K;
  const int blocks = (int)((warps * 32 + 255) / 256);
  if (C == 256)
    sp_sample_kernel<8><<<blocks, 256, 0, stream>>>(desc, keypoints, out, B, K, h, w, legacy);
  else
    sp_sample_kernel<4><<<blocks, 256, 0, stream>>>(desc, keypoints, out, B, K, h, w, legacy);
  return check_launch("sp_sample");
}

int lgb200_spo_conv1a(const float* image, int C, const float* weight, const float* bias, const float* scale,
                      const float* shift, void* out, int B, int H, int W, cudaStream_t stream) {
  return sp_conv1a_launch(true, image, C, weight, bias, scale, shift, out, B, H, W, stream);
}

int lgb200_spo_conv(const void* x, int ldx, const void* weight, const float* bias, const float* scale,
                    const float* shift, void* out, int B, int H, int W, int Cin, int Cout, int ksize, int epilogue,
                    cudaStream_t stream) {
  return sp_conv_dispatch<true>(x, ldx, weight, bias, scale, shift, out, B, H, W, Cin, Cout, ksize, epilogue, stream);
}

int lgb200_spo_bn_apply(const void* x, const double* sums, const float* gamma, const float* beta, float eps,
                        void* out, int B, int H, int W, int C, int op, cudaStream_t stream) {
  LGB_REQUIRE(x && sums && gamma && beta && out && x != out, kErrInvalid, "spo_bn_apply: null or aliased pointer");
  LGB_REQUIRE(B > 0 && H > 0 && W > 0, kErrInvalid, "spo_bn_apply: bad extents B=%d H=%d W=%d", B, H, W);
  LGB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, kErrInvalid,
              "spo_bn_apply: x and out must be 16-byte aligned");
  const int64_t T = (int64_t)B * H * W;
  auto grid = [&](int64_t threads) {
    return (unsigned)std::min<int64_t>((threads + SPO_BN_THREADS - 1) / SPO_BN_THREADS, 8LL * device_sm_count());
  };
  switch (op) {
    case SPO_BN_PLAIN:
    case SPO_BN_POOL: {
      LGB_REQUIRE(C >= 8 && C <= SPO_BN_MAXC && (C & (C - 1)) == 0, kErrUnsupported,
                  "spo_bn_apply: C %d is not a power of two in [8, %d]", C, SPO_BN_MAXC);
      LGB_REQUIRE(op == SPO_BN_PLAIN || (H >= 2 && W >= 2), kErrInvalid, "spo_bn_apply: %dx%d map too small to pool",
                  H, W);
      const int64_t n = op == SPO_BN_PLAIN ? T * (C / 8) : (int64_t)B * (H / 2) * (W / 2) * (C / 8);
      if (op == SPO_BN_PLAIN)
        spo_bn_nhwc_kernel<SPO_BN_PLAIN><<<grid(n), SPO_BN_THREADS, 0, stream>>>(
            (const __nv_bfloat16*)x, sums, gamma, beta, eps, (__nv_bfloat16*)out, B, H, W, C);
      else
        spo_bn_nhwc_kernel<SPO_BN_POOL><<<grid(n), SPO_BN_THREADS, 0, stream>>>(
            (const __nv_bfloat16*)x, sums, gamma, beta, eps, (__nv_bfloat16*)out, B, H, W, C);
      break;
    }
    case SPO_BN_SOFTMAX:
      LGB_REQUIRE(C == 65, kErrInvalid, "spo_bn_apply: the softmax op takes C 65 (got %d)", C);
      spo_bn_softmax_kernel<<<grid(T * 16), SPO_BN_THREADS, 0, stream>>>((const float*)x, sums, gamma, beta, eps,
                                                                        (float*)out, B, H, W);
      break;
    case SPO_BN_L2N:
      LGB_REQUIRE(C == 256, kErrInvalid, "spo_bn_apply: the normalising op takes C 256 (got %d)", C);
      spo_bn_l2n_kernel<<<grid(T * 32), SPO_BN_THREADS, 0, stream>>>((const float*)x, sums, gamma, beta, eps,
                                                                    (float*)out, T);
      break;
    default:
      LGB_REQUIRE(false, kErrInvalid, "spo_bn_apply: unknown op %d", op);
  }
  return check_launch("spo_bn_apply");
}

}  // extern "C"
