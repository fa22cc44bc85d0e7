// Per-unique-id CAR layer 1 (nar_model.py:343-370 feature rows, :374-405 CAR block).
//
// A candidate row of the reference is concat(user context of position l, item features of article id) * gamma + beta
// (nar_model.py:343-364).  For the negatives the item half depends on the article id only (reference timestamp = the
// batch maximum, :356) and every negative is drawn from the step's candidate pool of at most K*20 ids (:1300), so the
// first Dense layer splits exactly into
//     pre(l, k) = ctx(l) * W1[ctx rows] + b1  +  item(u(l,k)) * W1[item rows]  =  PC[l] + PI[u]
// with PC computed once per position and PI once per distinct id (two small GEMMs instead of one over all L*(1+K)
// rows).  This file holds the HBM-bound kernel after those GEMMs:
//   car_combine_kernel  H1[l, j] = leaky( j == 0 ? PP[l] : PC[l] + PI[u(l, j-1)] )        (forward)
// The backward (dPP, dPC = sum over a position's negatives, dPI = sum over the rows that drew u) is formed in the epilogue
// of the layer-2 dgrad (gemm_wgmma.cu, EXT_CAR_BWD), which recomputes pre from the same operands: dH1 never reaches HBM.
#include "common.cuh"

namespace nar {
namespace car {

constexpr int NT = 256;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void add4(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ float4 act4(float4 v, int act) {
  return make_float4(apply_act(v.x, act), apply_act(v.y, act), apply_act(v.z, act), apply_act(v.w, act));
}

// one CTA per position l: its 1+K candidate rows of H1
__global__ void __launch_bounds__(NT)
car_combine_kernel(const float* __restrict__ PP, const float* __restrict__ PC, const float* __restrict__ PI,
                   const int32_t* __restrict__ pos_idx, const int32_t* __restrict__ neg_uidx, int K, int C, int act,
                   float* __restrict__ H1c) {
  extern __shared__ int32_t s_u[];                  // [K]
  const int64_t l = blockIdx.x;
  const int64_t pos = pos_idx[l];
  for (int k = threadIdx.x; k < K; k += NT) s_u[k] = neg_uidx[pos * K + k];
  __syncthreads();
  const int n_cand = K + 1;
  float* out = H1c + l * n_cand * (int64_t)C;
  for (int c = threadIdx.x * 4; c < C; c += NT * 4) {
    *reinterpret_cast<float4*>(out + c) = act4(ld4(PP + l * C + c), act);
    const float4 pc = ld4(PC + l * C + c);
    int k = 0;
    for (; k + 4 <= K; k += 4) {                    // 4 independent PI rows in flight
      float4 v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q] = ld4(PI + (int64_t)s_u[k + q] * C + c);
#pragma unroll
      for (int q = 0; q < 4; ++q) { add4(v[q], pc); *reinterpret_cast<float4*>(out + (int64_t)(k + q + 1) * C + c) = act4(v[q], act); }
    }
    for (; k < K; ++k) {
      float4 v = ld4(PI + (int64_t)s_u[k] * C + c);
      add4(v, pc);
      *reinterpret_cast<float4*>(out + (int64_t)(k + 1) * C + c) = act4(v, act);
    }
  }
}

}  // namespace car
}  // namespace nar

extern "C" int nar_car_combine(const float* PP, const float* PC, const float* PI, const int32_t* pos_idx, const int32_t* neg_uidx,
                               int64_t L, int64_t K, int64_t C, int act, float* H1c, void* stream) {
  if (!PP || !PC || !PI || !pos_idx || !neg_uidx || !H1c) return NAR_ERR_INVALID;
  if ((C & 3) || K <= 0 || K > 8192) return NAR_ERR_INVALID;
  if (L <= 0) return NAR_OK;
  nar::car::car_combine_kernel<<<(unsigned)L, nar::car::NT, (size_t)K * sizeof(int32_t), as_stream(stream)>>>(
      PP, PC, PI, pos_idx, neg_uidx, (int)K, (int)C, act, H1c);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
