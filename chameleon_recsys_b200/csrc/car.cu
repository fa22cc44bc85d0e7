// Per-unique-id CAR layer 1 (nar_model.py:343-370 feature rows, :374-405 CAR block).
//
// A candidate row of the reference is concat(user context of position l, item features of article id) * gamma + beta
// (nar_model.py:343-364).  For the negatives the item half depends on the article id only (reference timestamp = the
// batch maximum, :356) and every negative is drawn from the step's candidate pool of at most K*20 ids (:1300), so the
// first Dense layer splits exactly into
//     pre(l, k) = ctx(l) * W1[ctx rows] + b1  +  item(u(l,k)) * W1[item rows]  =  PC[l] + PI[u]
// with PC computed once per position and PI once per distinct id (two small GEMMs instead of one over all L*(1+K)
// rows).  This file holds the HBM-bound kernel after those GEMMs:
//   car_combine_kernel    H1[l, j] = leaky( j == 0 ? PP[l] : PC[l] + PI[u(l, j-1)] )      (forward)
//   car_combine_t_kernel  the same rows stored transposed, [C, ldr] (what the training step uses)
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

// The same rows stored transposed, H1cT[c, r] (row stride ldr), so that the layer-2 weight gradient reads H1c K-major.
// CTA = 32 consecutive candidate rows x 128 columns, staged in shared memory: loaded row-wise (512 contiguous bytes per
// warp), stored column-wise (each warp writes four 128-byte column segments).  The tile's 16-byte chunk q of row r sits at
// chunk q ^ ((r >> 2) & 7): a warp's row-wise float4 stores permute the 32 chunks of one row, and its column-wise reads
// (rows 4 rq + i, rq = 0..7, four consecutive columns) hit 8 distinct chunk groups x 4 words = 32 banks.  The 32 rows'
// operand rows are looked up once per CTA (the pos_idx -> neg_uidx chain), so that each thread's loads are all in flight
// together.
constexpr int CT_ROWS = 32, CT_COLS = 128;
__global__ void __launch_bounds__(NT)
car_combine_t_kernel(const float* __restrict__ PP, const float* __restrict__ PC, const float* __restrict__ PI,
                     const int32_t* __restrict__ pos_idx, const int32_t* __restrict__ neg_uidx, int K, int C, int Rc, int act,
                     float* __restrict__ H1cT, int64_t ldr) {
  __shared__ __align__(16) float tile[CT_ROWS * CT_COLS];
  __shared__ const float* s_a[CT_ROWS];             // PP[l] (positive) or PI[u] (negative); nullptr past Rc
  __shared__ const float* s_b[CT_ROWS];             // PC[l] (negative) or nullptr
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * CT_ROWS, c0 = blockIdx.y * CT_COLS;
  if (threadIdx.x < CT_ROWS) {
    const int r = r0 + threadIdx.x, n_cand = K + 1;
    const float *a = nullptr, *b = nullptr;
    if (r < Rc) {
      const int64_t l = r / n_cand;
      const int j = r - (int)l * n_cand;
      if (j == 0) { a = PP + l * C; }
      else { a = PI + (int64_t)neg_uidx[(int64_t)pos_idx[l] * K + j - 1] * C; b = PC + l * C; }
    }
    s_a[threadIdx.x] = a; s_b[threadIdx.x] = b;
  }
  __syncthreads();
  const int c = c0 + lane * 4;
  float4 v[CT_ROWS / 8], w[CT_ROWS / 8];
#pragma unroll
  for (int i = 0; i < CT_ROWS / 8; ++i) {
    const int rl = i * 8 + warp;
    const float *a = s_a[rl], *b = s_b[rl];
    if (a && c < C) { v[i] = ld4(a + c); if (b) w[i] = ld4(b + c); }
  }
#pragma unroll
  for (int i = 0; i < CT_ROWS / 8; ++i) {
    const int rl = i * 8 + warp;
    const float *a = s_a[rl], *b = s_b[rl];
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a && c < C) {
      x = v[i];
      if (b) add4(x, w[i]);                          // PI + PC: the same single fp32 add as car_combine_kernel
      x = act4(x, act);
    }
    *reinterpret_cast<float4*>(tile + rl * CT_COLS + ((lane ^ ((rl >> 2) & 7)) << 2)) = x;
  }
  __syncthreads();
  const int rq = lane & 7, rr = r0 + 4 * rq;
#pragma unroll
  for (int i = 0; i < CT_COLS / 32; ++i) {
    const int cl = i * 32 + warp * 4 + (lane >> 3), cc = c0 + cl;
    if (cc >= C || rr >= Rc) continue;
    float e[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) e[q] = tile[(4 * rq + q) * CT_COLS + ((((cl >> 2) ^ rq) & 31) << 2) + (cl & 3)];
    float* o = H1cT + (int64_t)cc * ldr + rr;
    if (rr + 4 <= Rc) {
      *reinterpret_cast<float4*>(o) = make_float4(e[0], e[1], e[2], e[3]);
    } else {
#pragma unroll
      for (int q = 0; q < 3; ++q)
        if (rr + q < Rc) o[q] = e[q];
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

extern "C" int nar_car_combine_t(const float* PP, const float* PC, const float* PI, const int32_t* pos_idx, const int32_t* neg_uidx,
                                 int64_t L, int64_t K, int64_t C, int act, float* H1cT, int64_t ldr, void* stream) {
  using namespace nar::car;
  if (!PP || !PC || !PI || !pos_idx || !neg_uidx || !H1cT) return NAR_ERR_INVALID;
  if ((C & 3) || K <= 0 || K > 8192 || L < 0 || (reinterpret_cast<uintptr_t>(H1cT) & 15u)) return NAR_ERR_INVALID;
  const int64_t Rc = L * (K + 1);
  if ((ldr & 3) || ldr < Rc || Rc > 0x7fffffffLL - CT_ROWS || C > 0x7fffffffLL) return NAR_ERR_INVALID;
  if (L == 0) return NAR_OK;
  const dim3 grid((unsigned)((Rc + CT_ROWS - 1) / CT_ROWS), (unsigned)((C + CT_COLS - 1) / CT_COLS));
  car_combine_t_kernel<<<grid, NT, 0, as_stream(stream)>>>(PP, PC, PI, pos_idx, neg_uidx, (int)K, (int)C, (int)Rc, act, H1cT, ldr);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
