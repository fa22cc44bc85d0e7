// UGRNN recurrence of the session RNN (tf.contrib.rnn.UGRNNCell inside dynamic_rnn,
// nar_model.py:1308-1342).  The input projection x*Wx + b of ALL time steps is one wgmma GEMM
// (nar_gemm_tf32); what is left is the sequential part, independent per session:
//     act = gx[t] + h * Wh ;  g = sigmoid(act_g + 1) ; c = tanh(act_c) ; h' = g*h + (1-g)*c
// Rows are the valid positions only (session b owns rows [sess_off[b], sess_off[b+1])), so
// "zero output / state pass-through past sequence_length" needs no work at all.
//
// One CTA owns SB = 8 sessions and walks their time steps.  Per step the [Hp, 2Hp] recurrent matrix
// streams from L2 exactly once per CTA: thread (kq, jc) owns 4 gate + 4 candidate columns (float4
// loads, coalesced rows) for a 1/NSPLIT slice of k, 8-deep unrolled so 16 independent 128-bit loads are
// in flight per thread; partial sums meet in shared memory.  (Wh is 512 KB at H=256: it does not fit in
// one SM's shared memory in fp32; a cluster-resident variant is queued in DESIGN.md.)
#include "common.cuh"

namespace nar {
namespace rnn {

constexpr int SB = 4;             // sessions per CTA (8 -> 4: 64 CTAs at batch 256, and the early all-active steps cost half)
constexpr int THREADS = 256;
constexpr int MAX_HP = 1024;

__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ void fma4(float4& a, float s, const float4& w) {
  a.x = fmaf(s, w.x, a.x); a.y = fmaf(s, w.y, a.y); a.z = fmaf(s, w.z, a.z); a.w = fmaf(s, w.w, a.w);
}

struct Sess { int off[SB]; int len[SB]; int maxlen; };

__device__ __forceinline__ Sess load_sessions(const int32_t* __restrict__ sess_off, int64_t B) {
  Sess s; s.maxlen = 0;
  const int64_t b0 = (int64_t)blockIdx.x * SB;
#pragma unroll
  for (int i = 0; i < SB; ++i) {
    const int64_t b = b0 + i;
    s.off[i] = b < B ? sess_off[b] : 0;
    s.len[i] = b < B ? sess_off[b + 1] - sess_off[b] : 0;
    s.maxlen = max(s.maxlen, s.len[i]);
  }
  // longest first: at step t the sessions still running are slots [0, na) - the recurrent product skips the rest.
  // (The step count of a CTA is set by its longest session; with G1's geometric session lengths most slots are idle
  // after a few steps, and doing all SB products anyway made the whole kernel 19 x full-cost steps long.)
#pragma unroll
  for (int a = 0; a < SB - 1; ++a)
#pragma unroll
    for (int b = 0; b < SB - 1 - a; ++b)
      if (s.len[b] < s.len[b + 1]) {
        const int tl = s.len[b], to = s.off[b];
        s.len[b] = s.len[b + 1]; s.off[b] = s.off[b + 1];
        s.len[b + 1] = tl; s.off[b + 1] = to;
      }
  return s;
}
__device__ __forceinline__ int active_sessions(const Sess& s, int t) {
  int na = 0;
#pragma unroll
  for (int i = 0; i < SB; ++i) na += (s.len[i] > t) ? 1 : 0;
  return na;
}

// h[0..NA) * Wh slice of this thread -> partial sums in shared memory
template <int NA>
__device__ __forceinline__ void fwd_product(const float* __restrict__ Wh, const float* h, float* part, int Hp, int k0, int kspan,
                                            int jc, int kq) {
  const int W2 = 2 * Hp;
  float4 ag[NA], ac[NA];
#pragma unroll
  for (int s = 0; s < NA; ++s) { ag[s] = make_float4(0.f, 0.f, 0.f, 0.f); ac[s] = ag[s]; }
  const float4* wg = reinterpret_cast<const float4*>(Wh + (int64_t)k0 * W2) + jc;
  const float4* wc = reinterpret_cast<const float4*>(Wh + (int64_t)k0 * W2 + Hp) + jc;
  const int stride4 = W2 >> 2;
#pragma unroll 8
  for (int k = 0; k < kspan; ++k) {
    const float4 a = __ldg(wg + (int64_t)k * stride4), c = __ldg(wc + (int64_t)k * stride4);
#pragma unroll
    for (int s = 0; s < NA; ++s) { const float hv = h[s * Hp + k0 + k]; fma4(ag[s], hv, a); fma4(ac[s], hv, c); }
  }
#pragma unroll
  for (int s = 0; s < NA; ++s) {
    float4* pg = reinterpret_cast<float4*>(part + ((kq * SB + s) * 2 + 0) * Hp) + jc;
    float4* pc = reinterpret_cast<float4*>(part + ((kq * SB + s) * 2 + 1) * Hp) + jc;
    *pg = ag[s]; *pc = ac[s];
  }
}

template <int NA>
__device__ __forceinline__ void bwd_product(const float* __restrict__ WhT, const float* dact, float* part, int Hp, int j0, int jspan,
                                            int kc, int jq) {
  const int W2 = 2 * Hp;
  float4 acc[NA];
#pragma unroll
  for (int s = 0; s < NA; ++s) acc[s] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* w = reinterpret_cast<const float4*>(WhT + (int64_t)j0 * Hp) + kc;
  const int stride4 = Hp >> 2;
#pragma unroll 8
  for (int j = 0; j < jspan; ++j) {
    const float4 a = __ldg(w + (int64_t)j * stride4);
#pragma unroll
    for (int s = 0; s < NA; ++s) fma4(acc[s], dact[s * W2 + j0 + j], a);
  }
#pragma unroll
  for (int s = 0; s < NA; ++s) *(reinterpret_cast<float4*>(part + (jq * SB + s) * Hp) + kc) = acc[s];
}

// shared: h[SB][Hp] | part[NSPLIT][SB][2][Hp]
__global__ void __launch_bounds__(THREADS)
ugrnn_fwd_kernel(const float* __restrict__ gx, const float* __restrict__ Wh, const int32_t* __restrict__ sess_off,
                 int64_t B, int Hp, float* __restrict__ h_out, float* __restrict__ gate, float* __restrict__ cand) {
  extern __shared__ float sh[];
  float* h = sh;
  float* part = sh + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int NG = Hp >> 2;                 // column groups of 4
  const int NSPLIT = THREADS / NG;        // k slices (host guarantees THREADS % NG == 0, NSPLIT >= 1)
  const int jc = threadIdx.x % NG, kq = threadIdx.x / NG;
  const int kspan = Hp / NSPLIT, k0 = kq * kspan;
  const int W2 = 2 * Hp;
  for (int i = threadIdx.x; i < SB * Hp; i += THREADS) h[i] = 0.f;
  __syncthreads();
  for (int t = 0; t < ss.maxlen; ++t) {
    if (t > 0) {
      // sessions that reach step t also had step t-1, so slots [0, na) are exactly the ones with a live state
      const int na = active_sessions(ss, t);
      if (na <= 1) fwd_product<1>(Wh, h, part, Hp, k0, kspan, jc, kq);
      else if (na <= 2) fwd_product<2>(Wh, h, part, Hp, k0, kspan, jc, kq);
      else fwd_product<SB>(Wh, h, part, Hp, k0, kspan, jc, kq);
    }
    __syncthreads();
    // finalise: thread j owns column j of every session
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (t < ss.len[s]) {
          const float* g = gx + (int64_t)(ss.off[s] + t) * W2;
          float a = g[j], c = g[Hp + j];
          if (t > 0) {
            for (int q = 0; q < NSPLIT; ++q) {
              a += part[((q * SB + s) * 2 + 0) * Hp + j];
              c += part[((q * SB + s) * 2 + 1) * Hp + j];
            }
          }
          const float gt = sigmoidf(a + 1.0f), cd = tanhf(c);
          const float hn = gt * h[s * Hp + j] + (1.0f - gt) * cd;
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          h_out[row] = hn; gate[row] = gt; cand[row] = cd;
          h[s * Hp + j] = hn;                 // column j of h is read in this phase by this thread only
        }
      }
    }
    __syncthreads();
  }
}

// backward through time.  d_gx = dL/d(act) (feeds the Wx / bias / Wh wgrads and the dgrad GEMM);
// h_prev[row] = state entering the step (for dWh = h_prev^T * d_gx).
// shared: dact[SB][2Hp] | dh[SB][Hp] | keep[SB][Hp] | part[NSPLIT][SB][Hp]
__global__ void __launch_bounds__(THREADS)
ugrnn_bwd_kernel(const float* __restrict__ d_hout, const float* __restrict__ h_out, const float* __restrict__ gate,
                 const float* __restrict__ cand, const float* __restrict__ WhT, const int32_t* __restrict__ sess_off,
                 int64_t B, int Hp, float* __restrict__ d_gx, float* __restrict__ h_prev) {
  extern __shared__ float sh[];
  const int W2 = 2 * Hp;
  float* dact = sh;
  float* dh = dact + SB * W2;
  float* keep = dh + SB * Hp;
  float* part = keep + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int NG = Hp >> 2;
  const int NSPLIT = THREADS / NG;
  const int kc = threadIdx.x % NG, jq = threadIdx.x / NG;
  const int jspan = W2 / NSPLIT, j0 = jq * jspan;
  for (int i = threadIdx.x; i < SB * Hp; i += THREADS) dh[i] = 0.f;
  __syncthreads();
  for (int t = ss.maxlen - 1; t >= 0; --t) {
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        float dg_act = 0.f, dc_act = 0.f, kp = 0.f;
        if (t < ss.len[s]) {
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          const float dht = d_hout[row] + dh[s * Hp + j];
          const float hp = t > 0 ? h_out[row - Hp] : 0.f;
          const float g = gate[row], c = cand[row];
          dg_act = dht * (hp - c) * g * (1.0f - g);
          dc_act = dht * (1.0f - g) * (1.0f - c * c);
          kp = dht * g;
          d_gx[(int64_t)(ss.off[s] + t) * W2 + j] = dg_act;
          d_gx[(int64_t)(ss.off[s] + t) * W2 + Hp + j] = dc_act;
          h_prev[row] = hp;
        }
        dact[s * W2 + j] = dg_act;
        dact[s * W2 + Hp + j] = dc_act;
        keep[s * Hp + j] = kp;
      }
    }
    __syncthreads();
    if (t > 0) {
      const int na = active_sessions(ss, t);          // d_act of the slots past na is zero at this step
      if (na <= 1) bwd_product<1>(WhT, dact, part, Hp, j0, jspan, kc, jq);
      else if (na <= 2) bwd_product<2>(WhT, dact, part, Hp, j0, jspan, kc, jq);
      else bwd_product<SB>(WhT, dact, part, Hp, j0, jspan, kc, jq);
      __syncthreads();
      for (int k = threadIdx.x; k < Hp; k += THREADS) {
#pragma unroll
        for (int s = 0; s < SB; ++s) {
          if (t < ss.len[s]) {
            float v = keep[s * Hp + k];
            for (int q = 0; q < NSPLIT; ++q) v += part[(q * SB + s) * Hp + k];
            dh[s * Hp + k] = v;
          }
        }
      }
    }
    __syncthreads();
  }
}

static inline bool shape_ok(int64_t Hp) {
  if (Hp <= 0 || Hp > MAX_HP || (Hp & 3)) return false;
  const int64_t NG = Hp / 4;
  if (NG > THREADS || THREADS % NG != 0) return false;
  const int64_t ns = THREADS / NG;
  return (Hp % ns) == 0 && ((2 * Hp) % ns) == 0;
}

}  // namespace rnn
}  // namespace nar

extern "C" int nar_ugrnn_fwd(nar_ctx* ctx, const float* gx, const float* Wh, const int32_t* sess_off, int64_t B, int64_t Hp,
                             float* h_out, float* gate, float* cand, void* stream) {
  using namespace nar::rnn;
  if (!ctx || !gx || !Wh || !sess_off || !h_out || !gate || !cand) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;     // Hp/4 must divide 256 (64, 128, 256, 512, 1024)
  if (B <= 0) return NAR_OK;
  const int nsplit = THREADS / (int)(Hp / 4);
  const size_t smem = (size_t)(SB * Hp + nsplit * SB * 2 * Hp) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(ugrnn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  ugrnn_fwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(gx, Wh, sess_off, B, (int)Hp, h_out, gate, cand);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_ugrnn_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* gate, const float* cand,
                             const float* WhT, const int32_t* sess_off, int64_t B, int64_t Hp, float* d_gx, float* h_prev,
                             void* stream) {
  using namespace nar::rnn;
  if (!ctx || !d_hout || !h_out || !gate || !cand || !WhT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const int nsplit = THREADS / (int)(Hp / 4);
  const size_t smem = (size_t)(SB * 2 * Hp + 2 * SB * Hp + nsplit * SB * Hp) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(ugrnn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  ugrnn_bwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(d_hout, h_out, gate, cand, WhT, sess_off, B, (int)Hp, d_gx, h_prev);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
