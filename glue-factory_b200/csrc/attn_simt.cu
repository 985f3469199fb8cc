// fp32 CUDA-core attention (forward + backward) -- the full-precision parity path (`precision="fp32"`).  The bf16
// wgmma kernels (attn_tc.cu) are tested against fp64 torch, not against this file.
//
//   out = softmax(scale * q k^T) v       per (batch, head), head_dim kD = 64 or 32
// (reference: gluefactory/models/matchers/lightglue.py:118-121 self-attention,
//  :207-216 cross-attention evaluated as two one-directional passes).
//
// Tensors are token-major [B, N, H, kD].  The key/value batch of query batch b is
// (b + kv_shift) % B, which expresses the two directions of cross-attention on the
// concatenated [image0; image1] batch as ONE launch.  The forward also takes packed sequences of
// different lengths in one token-major [T, H, kD] buffer (attn_fwd_varlen_simt_kernel).
//
// Work split: two threads per row ("row" = query in fwd/dq, key in dkv), each owning half of the kD
// channels; dot products are completed with one shuffle.  The opposite operand is staged through
// shared memory in 64-row tiles and read as warp-wide broadcasts.
#include <math.h>

#include "common.cuh"
#include "lgb200.h"

namespace lgb {

constexpr int kTile = 64;  // rows per smem tile == rows per CTA

// cooperative load of `rows` x kD (row stride ld elements) into smem [kTile][kD], zero-filled past nvalid
template <int kD>
__device__ __forceinline__ void load_tile(float (*dst)[kD], const float* src, int64_t ld, int nvalid) {
  for (int idx = threadIdx.x; idx < kTile * kD; idx += blockDim.x) {
    const int r = idx >> (kD == 64 ? 6 : 5), c = idx & (kD - 1);
    dst[r][c] = r < nvalid ? src[(int64_t)r * ld + c] : 0.f;
  }
}

// One CTA of the forward: 64 query rows r0.. of head h.  Uniform batches (VARLEN false): query batch b, key batch kb,
// lse [B, H, Nq].  Packed sequences (VARLEN true): b / kb are the token rows of the sequence's first query / key,
// Nq / Nk its lengths, lse [H, Tq].
template <int kD, bool VARLEN>
__device__ __forceinline__ void attn_fwd_simt_cta(const float* __restrict__ q, const float* __restrict__ k,
                                                  const float* __restrict__ v, float* __restrict__ out,
                                                  float* __restrict__ lse, int b, int kb, int r0, int Nq, int Nk,
                                                  int H, int h, int Tq, float scale) {
  constexpr int kHalf = kD / 2;
  __shared__ float sk[kTile][kD];
  __shared__ float sv[kTile][kD];
  const int row = r0 + (threadIdx.x >> 1);
  const int half = threadIdx.x & 1;
  const int64_t ld = (int64_t)H * kD;
  const bool rvalid = row < Nq;
  const int64_t qrow = VARLEN ? (int64_t)b + row : (int64_t)b * Nq + row;
  const int64_t krow = VARLEN ? (int64_t)kb : (int64_t)kb * Nk;
  float qr[kHalf], o[kHalf];
#pragma unroll
  for (int d = 0; d < kHalf; ++d) {
    qr[d] = rvalid ? q[qrow * ld + h * kD + half * kHalf + d] * scale : 0.f;
    o[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < Nk; j0 += kTile) {
    const int nv = min(kTile, Nk - j0);
    __syncthreads();
    load_tile(sk, k + (krow + j0) * ld + h * kD, ld, nv);
    load_tile(sv, v + (krow + j0) * ld + h * kD, ld, nv);
    __syncthreads();
    for (int j = 0; j < nv; ++j) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) s = fmaf(qr[d], sk[j][half * kHalf + d], s);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if (s > m) {
        const float a = expf(m - s);
        l *= a;
#pragma unroll
        for (int d = 0; d < kHalf; ++d) o[d] *= a;
        m = s;
      }
      const float p = expf(s - m);
      l += p;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) o[d] = fmaf(p, sv[j][half * kHalf + d], o[d]);
    }
  }
  if (rvalid) {
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < kHalf; ++d) out[qrow * ld + h * kD + half * kHalf + d] = o[d] * inv;
    if (half == 0) {
      if constexpr (VARLEN)
        lse[(int64_t)h * Tq + b + row] = m + logf(l);
      else
        lse[((int64_t)b * H + h) * Nq + row] = m + logf(l);
    }
  }
}

template <int kD>
__global__ void __launch_bounds__(128) attn_fwd_simt_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                            const float* __restrict__ v, float* __restrict__ out,
                                                            float* __restrict__ lse, int B, int Nq, int Nk, int H,
                                                            int kv_shift, float scale) {
  const int b = blockIdx.z;
  attn_fwd_simt_cta<kD, false>(q, k, v, out, lse, b, (b + kv_shift) % B, blockIdx.x * kTile, Nq, Nk, H, blockIdx.y, 0,
                               scale);
}

// Packed sequences (see attn_fwd_varlen_tc_kernel): sequence s = blockIdx.z
template <int kD>
__global__ void __launch_bounds__(128)
    attn_fwd_varlen_simt_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                float* __restrict__ out, float* __restrict__ lse, const int* __restrict__ q_off,
                                const int* __restrict__ q_len, const int* __restrict__ k_off,
                                const int* __restrict__ k_len, int Tq, int H, float scale) {
  const int s = blockIdx.z, r0 = blockIdx.x * kTile;
  const int nq = q_len[s], nk = k_len[s];
  if (r0 >= nq || nk <= 0) return;
  attn_fwd_simt_cta<kD, true>(q, k, v, out, lse, q_off[s], k_off[s], r0, nq, nk, H, blockIdx.y, Tq, scale);
}

// delta[b,h,i] = sum_d dout[b,i,h,d] * out[b,i,h,d]   (8 lanes per row, kD / 8 channels each)
template <int kD>
__global__ void __launch_bounds__(256) attn_delta_kernel(const float* __restrict__ out, const float* __restrict__ dout,
                                                         float* __restrict__ delta, int64_t nrows /*B*N*H*/, int N,
                                                         int H) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = gid >> 3;  // (b, n, h) flattened token-major
  const int sub = (int)(gid & 7);
  float acc = 0.f;
  if (r < nrows) {
#pragma unroll
    for (int e = 0; e < kD / 8; ++e) acc += out[r * kD + sub * (kD / 8) + e] * dout[r * kD + sub * (kD / 8) + e];
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (r < nrows && sub == 0) {
    const int h = (int)(r % H);
    const int64_t bn = r / H;
    const int n = (int)(bn % N);
    const int64_t b = bn / N;
    delta[(b * H + h) * N + n] = acc;
  }
}

// dq_i = scale * sum_j p_ij (dp_ij - delta_i) k_j
template <int kD>
__global__ void __launch_bounds__(128)
    attn_bwd_dq_simt_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                            const float* __restrict__ dout, const float* __restrict__ lse,
                            const float* __restrict__ delta, float* __restrict__ dq, int B, int Nq, int Nk, int H,
                            int kv_shift, float scale) {
  constexpr int kHalf = kD / 2;
  __shared__ float sk[kTile][kD];
  __shared__ float sv[kTile][kD];
  const int b = blockIdx.z, h = blockIdx.y;
  const int kb = (b + kv_shift) % B;
  const int row = blockIdx.x * kTile + (threadIdx.x >> 1);
  const int half = threadIdx.x & 1;
  const int64_t ld = (int64_t)H * kD;
  const bool rvalid = row < Nq;
  float qr[kHalf], go[kHalf], acc[kHalf];
#pragma unroll
  for (int d = 0; d < kHalf; ++d) {
    const int64_t off = ((int64_t)b * Nq + row) * ld + h * kD + half * kHalf + d;
    qr[d] = rvalid ? q[off] * scale : 0.f;
    go[d] = rvalid ? dout[off] : 0.f;
    acc[d] = 0.f;
  }
  const float L = rvalid ? lse[((int64_t)b * H + h) * Nq + row] : 0.f;
  const float Dl = rvalid ? delta[((int64_t)b * H + h) * Nq + row] : 0.f;
  for (int j0 = 0; j0 < Nk; j0 += kTile) {
    const int nv = min(kTile, Nk - j0);
    __syncthreads();
    load_tile(sk, k + ((int64_t)kb * Nk + j0) * ld + h * kD, ld, nv);
    load_tile(sv, v + ((int64_t)kb * Nk + j0) * ld + h * kD, ld, nv);
    __syncthreads();
    for (int j = 0; j < nv; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) {
        s = fmaf(qr[d], sk[j][half * kHalf + d], s);
        dp = fmaf(go[d], sv[j][half * kHalf + d], dp);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      dp += __shfl_xor_sync(0xffffffffu, dp, 1);
      const float ds = expf(s - L) * (dp - Dl) * scale;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) acc[d] = fmaf(ds, sk[j][half * kHalf + d], acc[d]);
    }
  }
  if (rvalid) {
#pragma unroll
    for (int d = 0; d < kHalf; ++d)
      dq[((int64_t)b * Nq + row) * ld + h * kD + half * kHalf + d] = acc[d];
  }
}

// dv_j = sum_i p_ij do_i ;  dk_j = scale * sum_i p_ij (dp_ij - delta_i) q_i
// launched over KEY batches kb; the query batch is qb = (kb - kv_shift) mod B.
template <int kD>
__global__ void __launch_bounds__(128)
    attn_bwd_dkv_simt_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                             const float* __restrict__ dout, const float* __restrict__ lse,
                             const float* __restrict__ delta, float* __restrict__ dk, float* __restrict__ dv, int B,
                             int Nq, int Nk, int H, int kv_shift, float scale) {
  constexpr int kHalf = kD / 2;
  __shared__ float sq[kTile][kD];
  __shared__ float sdo[kTile][kD];
  __shared__ float sl[kTile], sd[kTile];
  const int kb = blockIdx.z, h = blockIdx.y;
  const int qb = ((kb - kv_shift) % B + B) % B;
  const int row = blockIdx.x * kTile + (threadIdx.x >> 1);
  const int half = threadIdx.x & 1;
  const int64_t ld = (int64_t)H * kD;
  const bool rvalid = row < Nk;
  float kr[kHalf], vr[kHalf], gk[kHalf], gv[kHalf];
#pragma unroll
  for (int d = 0; d < kHalf; ++d) {
    const int64_t off = ((int64_t)kb * Nk + row) * ld + h * kD + half * kHalf + d;
    kr[d] = rvalid ? k[off] * scale : 0.f;
    vr[d] = rvalid ? v[off] : 0.f;
    gk[d] = gv[d] = 0.f;
  }
  for (int i0 = 0; i0 < Nq; i0 += kTile) {
    const int nv = min(kTile, Nq - i0);
    __syncthreads();
    load_tile(sq, q + ((int64_t)qb * Nq + i0) * ld + h * kD, ld, nv);
    load_tile(sdo, dout + ((int64_t)qb * Nq + i0) * ld + h * kD, ld, nv);
    if (threadIdx.x < kTile) {
      const bool ok = (int)threadIdx.x < nv;
      sl[threadIdx.x] = ok ? lse[((int64_t)qb * H + h) * Nq + i0 + threadIdx.x] : 0.f;
      sd[threadIdx.x] = ok ? delta[((int64_t)qb * H + h) * Nq + i0 + threadIdx.x] : 0.f;
    }
    __syncthreads();
    for (int i = 0; i < nv; ++i) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) {
        s = fmaf(kr[d], sq[i][half * kHalf + d], s);
        dp = fmaf(vr[d], sdo[i][half * kHalf + d], dp);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      dp += __shfl_xor_sync(0xffffffffu, dp, 1);
      const float p = expf(s - sl[i]);
      const float ds = p * (dp - sd[i]) * scale;
#pragma unroll
      for (int d = 0; d < kHalf; ++d) {
        gv[d] = fmaf(p, sdo[i][half * kHalf + d], gv[d]);
        gk[d] = fmaf(ds, sq[i][half * kHalf + d], gk[d]);
      }
    }
  }
  if (rvalid) {
#pragma unroll
    for (int d = 0; d < kHalf; ++d) {
      const int64_t off = ((int64_t)kb * Nk + row) * ld + h * kD + half * kHalf + d;
      dk[off] = gk[d];
      dv[off] = gv[d];
    }
  }
}

template <int kD>
static int attn_fwd_simt_hd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk,
                            int H, int kv_shift, float scale, cudaStream_t stream) {
  dim3 grid((Nq + kTile - 1) / kTile, H, B);
  attn_fwd_simt_kernel<kD><<<grid, 128, 0, stream>>>((const float*)q, (const float*)k, (const float*)v, (float*)out,
                                                     lse, B, Nq, Nk, H, kv_shift, scale);
  return check_launch("attn_fwd_simt");
}

int attn_fwd_simt(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                  int kv_shift, float scale, int head_dim, cudaStream_t stream) {
  return head_dim == 32 ? attn_fwd_simt_hd<32>(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, stream)
                        : attn_fwd_simt_hd<64>(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, stream);
}

int attn_fwd_varlen_simt(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                         const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int H,
                         float scale, int head_dim, cudaStream_t stream) {
  dim3 grid((max_q_len + kTile - 1) / kTile, H, S);
  if (head_dim == 32)
    attn_fwd_varlen_simt_kernel<32><<<grid, 128, 0, stream>>>((const float*)q, (const float*)k, (const float*)v,
                                                              (float*)out, lse, q_off, q_len, k_off, k_len, Tq, H, scale);
  else
    attn_fwd_varlen_simt_kernel<64><<<grid, 128, 0, stream>>>((const float*)q, (const float*)k, (const float*)v,
                                                              (float*)out, lse, q_off, q_len, k_off, k_len, Tq, H, scale);
  return check_launch("attn_fwd_varlen_simt");
}

int attn_delta(const void* out, const void* dout, float* delta, int B, int N, int H, int head_dim,
               cudaStream_t stream) {
  const int64_t nrows = (int64_t)B * N * H;
  const unsigned grid = (unsigned)((nrows * 8 + 255) / 256);
  if (head_dim == 32)
    attn_delta_kernel<32><<<grid, 256, 0, stream>>>((const float*)out, (const float*)dout, delta, nrows, N, H);
  else
    attn_delta_kernel<64><<<grid, 256, 0, stream>>>((const float*)out, (const float*)dout, delta, nrows, N, H);
  return check_launch("attn_delta");
}

template <int kD>
static int attn_bwd_simt_hd(const void* q, const void* k, const void* v, const void* out, const float* lse,
                            const void* dout, void* dq, void* dk, void* dv, float* delta, int B, int Nq, int Nk, int H,
                            int kv_shift, float scale, cudaStream_t stream) {
  int rc = attn_delta(out, dout, delta, B, Nq, H, kD, stream);
  if (rc) return rc;
  dim3 gq((Nq + kTile - 1) / kTile, H, B);
  attn_bwd_dq_simt_kernel<kD><<<gq, 128, 0, stream>>>((const float*)q, (const float*)k, (const float*)v,
                                                      (const float*)dout, lse, delta, (float*)dq, B, Nq, Nk, H,
                                                      kv_shift, scale);
  dim3 gk((Nk + kTile - 1) / kTile, H, B);
  attn_bwd_dkv_simt_kernel<kD><<<gk, 128, 0, stream>>>((const float*)q, (const float*)k, (const float*)v,
                                                       (const float*)dout, lse, delta, (float*)dk, (float*)dv, B, Nq,
                                                       Nk, H, kv_shift, scale);
  return check_launch("attn_bwd_simt");
}

int attn_bwd_simt(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                  void* dq, void* dk, void* dv, float* delta, int B, int Nq, int Nk, int H, int kv_shift, float scale,
                  int head_dim, cudaStream_t stream) {
  return head_dim == 32
             ? attn_bwd_simt_hd<32>(q, k, v, out, lse, dout, dq, dk, dv, delta, B, Nq, Nk, H, kv_shift, scale, stream)
             : attn_bwd_simt_hd<64>(q, k, v, out, lse, dout, dq, dk, dv, delta, B, Nq, Nk, H, kv_shift, scale, stream);
}

}  // namespace lgb
