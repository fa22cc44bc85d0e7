// Shared device helpers for libnar_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include "../../include/nar_b200.h"

#define NAR_CHECK_CUDA(expr)                                   \
  do {                                                         \
    cudaError_t _e = (expr);                                   \
    if (_e != cudaSuccess) return (int)_e;                     \
  } while (0)

#define NAR_LAUNCH_CHECK()                                     \
  do {                                                         \
    cudaError_t _e = cudaGetLastError();                       \
    if (_e != cudaSuccess) return (int)_e;                     \
  } while (0)

struct nar_ctx {
  int device;
  int sm_count;
  void* encode_tiled;   // cuTensorMapEncodeTiled entry point
  // feature gather: device table of per-column descriptors, rebuilt only when the static part of the plan changes
  void* gather_desc;            // device, NAR_GATHER_DESC_BYTES
  void* gather_key;             // host copy of the static plan fields the table was built from (nar_feature_plan*)
  int gather_key_valid;
};
#define NAR_GATHER_DESC_BYTES (2 * 512 * 16 + 64)
// grid-stride kernels launched without a nar_ctx cap their grid at a few blocks per SM of an H100 SXM (132 SMs)
#define NAR_GRID_SMS 132

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

namespace nar {

__device__ __forceinline__ float leaky_relu(float x) { return x > 0.f ? x : 0.2f * x; }

// tanh with ~1e-7 absolute error in ~8 instructions (tanhf costs ~30 and the GEMM epilogue is not overlapped with
// its main loop): odd polynomial near 0 (no cancellation), 1 - 2/(e^{2x}+1) elsewhere (MUFU.EX2 + fast divide).
__device__ __forceinline__ float tanh_fast(float x) {
  const float ax = fabsf(x);
  if (ax < 0.1f) {
    const float x2 = x * x;
    return x * (1.0f + x2 * (-0.33333334f + x2 * (0.13333334f + x2 * -0.05396825f)));
  }
  const float t = __expf(2.0f * ax);
  const float r = 1.0f - __fdividef(2.0f, t + 1.0f);
  return copysignf(r, x);
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == NAR_ACT_LEAKY_RELU) return leaky_relu(x);
  if (act == NAR_ACT_TANH) return tanhf(x);     // tanh_fast measured slower inside the GEMM epilogue (divergent branch)
  return x;
}

// derivative of the activation expressed through the forward OUTPUT y
__device__ __forceinline__ float act_grad_from_output(float y, int act) {
  if (act == NAR_ACT_LEAKY_RELU) return y > 0.f ? 1.f : 0.2f;
  if (act == NAR_ACT_TANH) return 1.f - y * y;
  return 1.f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- Philox4x32-10 (spec: oracle/sampler_ref.py) ------------------------------------
struct Philox4 { uint32_t x, y, z, w; };
__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
__device__ __forceinline__ uint32_t philox_word(const Philox4& p, uint32_t i) {
  return i == 0 ? p.x : (i == 1 ? p.y : (i == 2 ? p.z : p.w));
}
// 64-bit shuffle key of element idx: (rand32 << 32) | idx
__device__ __forceinline__ uint64_t shuffle_key(uint64_t seed, uint32_t step, uint32_t stream, uint32_t ctx,
                                                uint32_t idx) {
  Philox4 p = philox4x32_10(idx >> 2, ctx, stream, step, (uint32_t)seed, (uint32_t)(seed >> 32));
  return ((uint64_t)philox_word(p, idx & 3u) << 32) | (uint64_t)idx;
}

// bit of an id in the 4096-bit Bloom filters in front of the session-row exclusion lists (top n, label ranks)
__device__ __forceinline__ uint32_t bloom_slot(int64_t id) { return ((uint32_t)id * 2654435761u) >> 20; }

}  // namespace nar
