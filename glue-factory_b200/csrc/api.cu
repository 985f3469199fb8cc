// Host-side plumbing shared by all entry points: error reporting, device check, TMA descriptor
// construction (driver entry point fetched through the runtime, no link-time libcuda dependency).
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"
#include "host_util.h"
#include "lgb200.h"

namespace lgb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA error: %s", what, cudaGetErrorString(e));
    return kErrCuda;
  }
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
    set_error("cuTensorMapEncodeTiled not available: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// bf16 tensor map with 128-byte swizzle. dims/strides fastest-first; strides in BYTES for dims 1..rank-1.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes) {
  return make_tmap(out, base, /*fp32=*/false, rank, dims, strides_bytes, box, swizzle_bytes);
}

int make_tmap(CUtensorMap* out, const void* base, bool fp32, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return kErrCuda;
  LGB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, kErrInvalid, "TMA base pointer not 16-byte aligned");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      LGB_REQUIRE((strides_bytes[i - 1] & 15) == 0, kErrInvalid, "TMA stride %llu not a multiple of 16 bytes",
                  (unsigned long long)strides_bytes[i - 1]);
      gstr[i - 1] = strides_bytes[i - 1];
    }
  }
  auto encode = [&]() {
    return fn(out, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
              const_cast<void*>(base), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              swizzle_bytes == 32   ? CU_TENSOR_MAP_SWIZZLE_32B
              : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                    : CU_TENSOR_MAP_SWIZZLE_128B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = encode();
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // a thread that has not issued a CUDA runtime call yet (e.g. a fresh autograd worker whose first CUDA work is this
    // entry point) has no current context for the driver API: bind the primary context and retry
    cudaFree(nullptr);
    r = encode();
  }
  LGB_REQUIRE(r == CUDA_SUCCESS, kErrCuda, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int ensure_dyn_smem(const void* func, int bytes) {
  // remembers the largest size configured per (kernel, device); a kernel whose dynamic size varies from launch to
  // launch (the Sinkhorn strip cache) raises the limit when a larger request comes along
  constexpr int kMaxFuncs = 64, kMaxDevs = 16;
  static const void* funcs[kMaxFuncs];
  static int done[kMaxFuncs][kMaxDevs];  // bytes configured on device d (0: never)
  static int nfuncs = 0;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "cudaGetDevice: %s", cudaGetErrorString(e));
  int slot = -1;
  for (int i = 0; i < nfuncs; ++i)
    if (funcs[i] == func) slot = i;
  if (slot >= 0 && dev < kMaxDevs && done[slot][dev] >= bytes && done[slot][dev] > 0) return 0;
  e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "cudaFuncSetAttribute(%d bytes): %s", bytes, cudaGetErrorString(e));
  if (slot < 0 && nfuncs < kMaxFuncs) {
    slot = nfuncs++;
    funcs[slot] = func;
    for (int d = 0; d < kMaxDevs; ++d) done[slot][d] = 0;
  }
  if (slot >= 0 && dev < kMaxDevs) done[slot][dev] = bytes > 0 ? bytes : 1;
  return 0;
}

int device_sm_count() {
  static int counts[16];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 16 && counts[dev]) return counts[dev];
  int n = 0;
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  if (n <= 0) n = 132;  // H100 SXM
  if (dev >= 0 && dev < 16) counts[dev] = n;
  return n;
}

}  // namespace lgb

using namespace lgb;

extern "C" {

int lgb200_abi_version(void) { return LGB200_ABI_VERSION; }
const char* lgb200_last_error(void) { return g_err; }

int lgb200_check_device(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  LGB_REQUIRE(e == cudaSuccess, kErrCuda, "cudaGetDevice: %s", cudaGetErrorString(e));
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  LGB_REQUIRE(major == 9 && minor == 0, kErrUnsupported, "device %d is sm_%d%d; this library is built for sm_90a only", dev,
              major, minor);
  return 0;
}

int lgb200_attn_fwd_hd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk,
                       int H, int kv_shift, float scale, int dtype, int head_dim, cudaStream_t stream) {
  LGB_REQUIRE(q && k && v && out && lse, kErrInvalid, "attn_fwd: null pointer");
  LGB_REQUIRE(B > 0 && Nq > 0 && Nk > 0 && H > 0, kErrInvalid, "attn_fwd: empty input B=%d Nq=%d Nk=%d H=%d", B, Nq,
              Nk, H);
  LGB_REQUIRE(kv_shift >= 0 && kv_shift < B, kErrInvalid, "attn_fwd: kv_shift %d out of range", kv_shift);
  LGB_REQUIRE(head_dim == 32 || head_dim == 64, kErrUnsupported, "attn_fwd: head_dim %d (built for 32 and 64)",
              head_dim);
  if (dtype == LGB200_F32) return attn_fwd_simt(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, head_dim, stream);
  LGB_REQUIRE(dtype == LGB200_BF16, kErrInvalid, "attn_fwd: bad dtype %d", dtype);
  return attn_fwd_tc(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, head_dim, stream);
}

int lgb200_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                    int kv_shift, float scale, int dtype, cudaStream_t stream) {
  return lgb200_attn_fwd_hd(q, k, v, out, lse, B, Nq, Nk, H, kv_shift, scale, dtype, 64, stream);
}

int lgb200_attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                           const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int Tk,
                           int H, float scale, int dtype, int head_dim, cudaStream_t stream) {
  LGB_REQUIRE(q && k && v && out && lse && q_off && q_len && k_off && k_len, kErrInvalid,
              "attn_fwd_varlen: null pointer");
  LGB_REQUIRE(S >= 0 && max_q_len >= 0 && Tq >= 0 && Tk >= 0 && H > 0, kErrInvalid,
              "attn_fwd_varlen: bad extents S=%d max_q_len=%d Tq=%d Tk=%d H=%d", S, max_q_len, Tq, Tk, H);
  LGB_REQUIRE(head_dim == 32 || head_dim == 64, kErrUnsupported, "attn_fwd_varlen: head_dim %d (built for 32 and 64)",
              head_dim);
  LGB_REQUIRE(dtype == LGB200_F32 || dtype == LGB200_BF16, kErrInvalid, "attn_fwd_varlen: bad dtype %d", dtype);
  if (S == 0 || max_q_len == 0 || Tq == 0 || Tk == 0) return 0;  // no sequence has both queries and keys
  if (dtype == LGB200_F32)
    return attn_fwd_varlen_simt(q, k, v, out, lse, q_off, q_len, k_off, k_len, S, max_q_len, Tq, H, scale, head_dim,
                                stream);
  return attn_fwd_varlen_tc(q, k, v, out, lse, q_off, q_len, k_off, k_len, S, max_q_len, Tq, Tk, H, scale, head_dim,
                            stream);
}

int64_t lgb200_attn_bwd_ws_floats(int B, int Nq, int Nk, int H) { return attn_bwd_ws_floats(B, Nq, Nk, H); }

int lgb200_attn_bwd_hd(const void* q, const void* k, const void* v, const void* out, const float* lse,
                       const void* dout, void* dq, void* dk, void* dv, float* delta_ws, int B, int Nq, int Nk, int H,
                       int kv_shift, float scale, int dtype, int head_dim, cudaStream_t stream) {
  LGB_REQUIRE(q && k && v && out && lse && dout && dq && dk && dv && delta_ws, kErrInvalid, "attn_bwd: null pointer");
  LGB_REQUIRE(B > 0 && Nq > 0 && Nk > 0 && H > 0, kErrInvalid, "attn_bwd: empty input");
  LGB_REQUIRE(kv_shift >= 0 && kv_shift < B, kErrInvalid, "attn_bwd: kv_shift %d out of range", kv_shift);
  LGB_REQUIRE(head_dim == 32 || head_dim == 64, kErrUnsupported, "attn_bwd: head_dim %d (built for 32 and 64)",
              head_dim);
  const bool shared_qk = attn_bwd_is_shared_qk(q, k, dq, dk, B, Nq, Nk, kv_shift);
  LGB_REQUIRE(!shared_qk || dtype == LGB200_BF16, kErrUnsupported,
              "attn_bwd: dq == dk (shared-qk cross-attention) runs on the bf16 tensor-core path only");
  LGB_REQUIRE(!shared_qk || head_dim == 64, kErrUnsupported,
              "attn_bwd: dq == dk (shared-qk cross-attention) is built for head_dim 64 only");
  if (dtype == LGB200_F32)
    return attn_bwd_simt(q, k, v, out, lse, dout, dq, dk, dv, delta_ws, B, Nq, Nk, H, kv_shift, scale, head_dim,
                         stream);
  LGB_REQUIRE(dtype == LGB200_BF16, kErrInvalid, "attn_bwd: bad dtype %d", dtype);
  return attn_bwd_tc(q, k, v, out, lse, dout, dq, dk, dv, delta_ws, B, Nq, Nk, H, kv_shift, scale, head_dim, stream);
}

int lgb200_attn_bwd(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                    void* dq, void* dk, void* dv, float* delta_ws, int B, int Nq, int Nk, int H, int kv_shift,
                    float scale, int dtype, cudaStream_t stream) {
  return lgb200_attn_bwd_hd(q, k, v, out, lse, dout, dq, dk, dv, delta_ws, B, Nq, Nk, H, kv_shift, scale, dtype, 64,
                            stream);
}

}  // extern "C"
