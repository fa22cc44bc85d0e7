// GRU recurrence of the session RNN: the cell north_star names ("session GRU") and the reference keeps one comment away
// (nar_model.py:1315 `#cell = tf.nn.rnn_cell.GRUCell(rnn_units)`); selected with rnn_cell='gru'.
//
// tf.nn.rnn_cell.GRUCell (TF 1.12 rnn_cell_impl.py):
//     [r, u] = sigmoid([x, h] * Wg + bg)          gates/kernel [in+H, 2H], gates/bias (initialised to 1.0)
//     c      = tanh([x, r*h] * Wc + bc)           candidate/kernel [in+H, H], candidate/bias
//     h'     = u * h + (1 - u) * c
// The input projections x*Wg[:in] + bg | x*Wc[:in] + bc of ALL time steps are wgmma GEMMs (nar_gemm_tf32) into
// gx [L, 3Hp] = (r | u | c); what is left is the sequential part, independent per session, with TWO dependent
// matrix-vector products per step (h * Whg, then (r*h) * Whc).  Same work split as csrc/rnn.cu: one CTA owns SB
// sessions, slots sorted longest first so that finished sessions cost nothing; rows are the valid positions only.
#include "common.cuh"

namespace nar {
namespace gru {

constexpr int SB = 4;
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

// part[kq][s][0..NW) += v[s][k0 .. k0+kspan) * W[k, :NW] for this thread's 4 columns (jc) ; W row stride = NW floats.
// One k-slice per thread group kq; the slices meet in shared memory (summed by the finalise phase).
template <int NA>
__device__ __forceinline__ void matvec(const float* __restrict__ W, int NW, const float* v, int ldv, float* part, int k0, int kspan,
                                       int jc, int kq) {
  float4 acc[NA];
#pragma unroll
  for (int s = 0; s < NA; ++s) acc[s] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* w = reinterpret_cast<const float4*>(W + (int64_t)k0 * NW) + jc;
  const int stride4 = NW >> 2;
#pragma unroll 8
  for (int k = 0; k < kspan; ++k) {
    const float4 a = __ldg(w + (int64_t)k * stride4);
#pragma unroll
    for (int s = 0; s < NA; ++s) fma4(acc[s], v[s * ldv + k0 + k], a);
  }
#pragma unroll
  for (int s = 0; s < NA; ++s) *(reinterpret_cast<float4*>(part + (int64_t)(kq * SB + s) * NW) + jc) = acc[s];
}

__device__ __forceinline__ void matvec_dyn(int na, const float* __restrict__ W, int NW, const float* v, int ldv, float* part, int k0,
                                           int kspan, int jc, int kq) {
  if (na <= 1) matvec<1>(W, NW, v, ldv, part, k0, kspan, jc, kq);
  else if (na <= 2) matvec<2>(W, NW, v, ldv, part, k0, kspan, jc, kq);
  else matvec<SB>(W, NW, v, ldv, part, k0, kspan, jc, kq);
}

// thread layout for an [K, NW] matrix: NG = NW/4 column groups, NSPLIT = THREADS/NG k-slices (NG may exceed THREADS:
// then each thread walks several column groups with NSPLIT = 1)
struct Split { int ng, nsplit, kspan; };
__device__ __forceinline__ Split make_split(int K, int NW) {
  Split s; s.ng = NW >> 2;
  s.nsplit = s.ng >= THREADS ? 1 : THREADS / s.ng;
  s.kspan = K / s.nsplit;
  return s;
}
// all threads: part[q][s][:] for q < nsplit
__device__ __forceinline__ void product(int na, const float* __restrict__ W, int K, int NW, const float* v, int ldv, float* part) {
  const Split sp = make_split(K, NW);
  if (sp.ng >= THREADS) {
    for (int jc = threadIdx.x; jc < sp.ng; jc += THREADS) matvec_dyn(na, W, NW, v, ldv, part, 0, K, jc, 0);
  } else {
    const int jc = threadIdx.x % sp.ng, kq = threadIdx.x / sp.ng;
    if (kq < sp.nsplit) matvec_dyn(na, W, NW, v, ldv, part, kq * sp.kspan, sp.kspan, jc, kq);
  }
}

// shared: h[SB][Hp] | rh[SB][Hp] | part[NSPLIT][SB][2Hp]
__global__ void __launch_bounds__(THREADS)
gru_fwd_kernel(const float* __restrict__ gx, const float* __restrict__ Whg, const float* __restrict__ Whc,
               const int32_t* __restrict__ sess_off, int64_t B, int Hp, float* __restrict__ h_out, float* __restrict__ r_out,
               float* __restrict__ u_out, float* __restrict__ c_out, float* __restrict__ rh_out) {
  extern __shared__ float sh[];
  float* h = sh;
  float* rh = sh + SB * Hp;
  float* part = rh + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int W2 = 2 * Hp, W3 = 3 * Hp;
  const int ns_g = make_split(Hp, W2).nsplit, ns_c = make_split(Hp, Hp).nsplit;
  for (int i = threadIdx.x; i < SB * Hp; i += THREADS) h[i] = 0.f;
  __syncthreads();
  for (int t = 0; t < ss.maxlen; ++t) {
    const int na = active_sessions(ss, t);
    if (t > 0) product(na, Whg, Hp, W2, h, Hp, part);
    __syncthreads();
    // gates: thread j owns unit j of every session
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (t < ss.len[s]) {
          const float* g = gx + (int64_t)(ss.off[s] + t) * W3;
          float ar = g[j], au = g[Hp + j];
          if (t > 0)
            for (int q = 0; q < ns_g; ++q) { ar += part[(int64_t)(q * SB + s) * W2 + j]; au += part[(int64_t)(q * SB + s) * W2 + Hp + j]; }
          const float r = sigmoidf(ar), u = sigmoidf(au);
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          r_out[row] = r; u_out[row] = u;
          const float x = r * h[s * Hp + j];
          rh[s * Hp + j] = x; rh_out[row] = x;
        }
      }
    }
    __syncthreads();
    if (t > 0) product(na, Whc, Hp, Hp, rh, Hp, part);
    __syncthreads();
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (t < ss.len[s]) {
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          float ac = gx[(int64_t)(ss.off[s] + t) * W3 + W2 + j];
          if (t > 0)
            for (int q = 0; q < ns_c; ++q) ac += part[(int64_t)(q * SB + s) * Hp + j];
          const float c = tanhf(ac), u = u_out[row];
          const float hn = u * h[s * Hp + j] + (1.0f - u) * c;
          c_out[row] = c; h_out[row] = hn;
          h[s * Hp + j] = hn;
        }
      }
    }
    __syncthreads();
  }
}

// backward through time.  d_gx [L,3Hp] = dL/d(pre-activations r | u | c); h_prev [L,Hp] = state entering the step
// (dWhg = h_prev^T d_gx[:, :2Hp]; dWhc = rh^T d_gx[:, 2Hp:] with rh from the forward pass).
// shared: dgate[SB][2Hp] | dcand[SB][Hp] | dh[SB][Hp] | keep[SB][Hp] | part[NSPLIT][SB][Hp]
__global__ void __launch_bounds__(THREADS)
gru_bwd_kernel(const float* __restrict__ d_hout, const float* __restrict__ h_out, const float* __restrict__ r_out,
               const float* __restrict__ u_out, const float* __restrict__ c_out, const float* __restrict__ WhgT /*[2Hp,Hp]*/,
               const float* __restrict__ WhcT /*[Hp,Hp]*/, const int32_t* __restrict__ sess_off, int64_t B, int Hp,
               float* __restrict__ d_gx, float* __restrict__ h_prev) {
  extern __shared__ float sh[];
  const int W2 = 2 * Hp, W3 = 3 * Hp;
  float* dgate = sh;
  float* dcand = dgate + SB * W2;
  float* dh = dcand + SB * Hp;
  float* keep = dh + SB * Hp;
  float* part = keep + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int ns_c = make_split(Hp, Hp).nsplit, ns_g = make_split(W2, Hp).nsplit;
  for (int i = threadIdx.x; i < SB * Hp; i += THREADS) dh[i] = 0.f;
  __syncthreads();
  for (int t = ss.maxlen - 1; t >= 0; --t) {
    const int na = active_sessions(ss, t);
    // ---- through h' = u*h + (1-u)*c and c = tanh(.)
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        float dca = 0.f, kp = 0.f;
        if (t < ss.len[s]) {
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          const float dht = d_hout[row] + dh[s * Hp + j];
          const float u = u_out[row], c = c_out[row];
          dca = dht * (1.0f - u) * (1.0f - c * c);
          kp = dht * u;
          d_gx[(int64_t)(ss.off[s] + t) * W3 + W2 + j] = dca;
        }
        dcand[s * Hp + j] = dca;
        keep[s * Hp + j] = kp;
      }
    }
    __syncthreads();
    // ---- d(r*h) = dcand * Whc^T   (only needed when a previous state exists: at t = 0 h = 0, so dr_act = 0 and nothing flows on)
    if (t > 0) product(na, WhcT, Hp, Hp, dcand, Hp, part);
    __syncthreads();
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        float dra = 0.f, dua = 0.f;
        if (t < ss.len[s]) {
          const int64_t row = (int64_t)(ss.off[s] + t) * Hp + j;
          const float hp = t > 0 ? h_out[row - Hp] : 0.f;
          const float dht = d_hout[row] + dh[s * Hp + j];
          const float r = r_out[row], u = u_out[row], c = c_out[row];
          float drh = 0.f;
          if (t > 0)
            for (int q = 0; q < ns_c; ++q) drh += part[(int64_t)(q * SB + s) * Hp + j];
          dra = drh * hp * r * (1.0f - r);
          dua = dht * (hp - c) * u * (1.0f - u);
          keep[s * Hp + j] += drh * r;
          d_gx[(int64_t)(ss.off[s] + t) * W3 + j] = dra;
          d_gx[(int64_t)(ss.off[s] + t) * W3 + Hp + j] = dua;
          h_prev[row] = hp;
        }
        dgate[s * W2 + j] = dra;
        dgate[s * W2 + Hp + j] = dua;
      }
    }
    __syncthreads();
    if (t > 0) {
      product(na, WhgT, W2, Hp, dgate, W2, part);
      __syncthreads();
      for (int k = threadIdx.x; k < Hp; k += THREADS) {
#pragma unroll
        for (int s = 0; s < SB; ++s) {
          if (t < ss.len[s]) {
            float v = keep[s * Hp + k];
            for (int q = 0; q < ns_g; ++q) v += part[(int64_t)(q * SB + s) * Hp + k];
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
  // every matrix-vector product splits K evenly: K in {Hp, 2Hp}, NW in {Hp, 2Hp}
  const int64_t ng1 = Hp / 4, ng2 = 2 * Hp / 4;
  auto ok = [](int64_t K, int64_t ng) {
    if (ng >= THREADS) return true;
    if (THREADS % ng) return false;
    return (K % (THREADS / ng)) == 0;
  };
  return ok(Hp, ng2) && ok(Hp, ng1) && ok(2 * Hp, ng1);
}
static inline int nsplit_of(int64_t NW) { const int64_t ng = NW / 4; return ng >= THREADS ? 1 : (int)(THREADS / ng); }

}  // namespace gru
}  // namespace nar

extern "C" int nar_gru_fwd(nar_ctx* ctx, const float* gx, const float* Whg, const float* Whc, const int32_t* sess_off, int64_t B,
                           int64_t Hp, float* h_out, float* r_out, float* u_out, float* c_out, float* rh_out, void* stream) {
  using namespace nar::gru;
  if (!ctx || !gx || !Whg || !Whc || !sess_off || !h_out || !r_out || !u_out || !c_out || !rh_out) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const int ns = nsplit_of(2 * Hp) > nsplit_of(Hp) ? nsplit_of(2 * Hp) : nsplit_of(Hp);
  const size_t part = (size_t)(nsplit_of(2 * Hp) * SB * 2 * Hp > nsplit_of(Hp) * SB * Hp ? nsplit_of(2 * Hp) * SB * 2 * Hp : nsplit_of(Hp) * SB * Hp);
  const size_t smem = ((size_t)2 * SB * Hp + part) * sizeof(float);
  (void)ns;
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  gru_fwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(gx, Whg, Whc, sess_off, B, (int)Hp, h_out, r_out,
                                                                                      u_out, c_out, rh_out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_gru_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* r_out, const float* u_out,
                           const float* c_out, const float* WhgT, const float* WhcT, const int32_t* sess_off, int64_t B, int64_t Hp,
                           float* d_gx, float* h_prev, void* stream) {
  using namespace nar::gru;
  if (!ctx || !d_hout || !h_out || !r_out || !u_out || !c_out || !WhgT || !WhcT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const size_t part = (size_t)nsplit_of(Hp) * SB * Hp;       // both backward products write [nsplit][SB][Hp]
  const size_t smem = ((size_t)SB * 2 * Hp + 3 * SB * Hp + part) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  gru_bwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(d_hout, h_out, r_out, u_out, c_out, WhgT, WhcT,
                                                                                      sess_off, B, (int)Hp, d_gx, h_prev);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
