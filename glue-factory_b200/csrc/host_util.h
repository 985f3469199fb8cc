// Internal host-side declarations shared between translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace lgb {

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes = 128);
// same for fp32 (fp32 = true) or bf16 elements
int make_tmap(CUtensorMap* out, const void* base, bool fp32, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: set it once per (kernel, device), not once
// per process.  Returns 0 or kErrCuda.
int ensure_dyn_smem(const void* func, int bytes);
// SM count of the CURRENT device (cached per device ordinal)
int device_sm_count();

// fp32 CUDA-core attention (attn_simt.cu); head_dim 32 or 64, checked by the api.cu entry points
int attn_fwd_simt(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                  int kv_shift, float scale, int head_dim, cudaStream_t stream);
int attn_bwd_simt(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                  void* dq, void* dk, void* dv, float* delta, int B, int Nq, int Nk, int H, int kv_shift, float scale,
                  int head_dim, cudaStream_t stream);
int attn_delta(const void* out, const void* dout, float* delta, int B, int N, int H, int head_dim,
               cudaStream_t stream);
int attn_fwd_varlen_simt(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                         const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int H,
                         float scale, int head_dim, cudaStream_t stream);

// wgmma attention (attn_tc.cu); head_dim as above, the shared-qk backward at 64 only
int attn_fwd_tc(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                int kv_shift, float scale, int head_dim, cudaStream_t stream);
int attn_bwd_tc(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                void* dq, void* dk, void* dv, float* delta, int B, int Nq, int Nk, int H, int kv_shift, float scale,
                int head_dim, cudaStream_t stream);
int attn_fwd_varlen_tc(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                       const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int Tk,
                       int H, float scale, int head_dim, cudaStream_t stream);

// lgb200_attn_bwd's shared-qk cross-attention case (q == k, dq == dk, both directions in one batch)
inline bool attn_bwd_is_shared_qk(const void* q, const void* k, const void* dq, const void* dk, int B, int Nq, int Nk,
                                  int kv_shift) {
  return q == k && dq == dk && Nq == Nk && 2 * kv_shift == B;
}

// scratch (floats) lgb200_attn_bwd needs for the bf16 path (padded softmax statistics)
int64_t attn_bwd_ws_floats(int B, int Nq, int Nk, int H);

}  // namespace lgb
