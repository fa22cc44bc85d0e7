// LSTM recurrence of the session RNN: the cell the reference keeps one comment away
// (nar_model.py:1316 `#cell = tf.nn.rnn_cell.LSTMCell(rnn_units, state_is_tuple=True)`); selected with rnn_cell='lstm'.
//
// tf.nn.rnn_cell.LSTMCell (TF 1.12 rnn_cell_impl.py; no peepholes, no cell clip, no projection, forget_bias 1.0):
//     z  = [x, h] * kernel + bias                 kernel [in+H, 4H], bias [4H], columns i | j | f | o
//     c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j)
//     h' = sigmoid(o) * tanh(c')                  output = h', state = (c', h')
// The input projection x*Wx + b of ALL time steps is one wgmma GEMM into gx [L, 4Hp] (column blocks i | j | f | o, each Hp
// wide); what is left is the sequential part, independent per session, with ONE matrix-vector product per step
// (h * Wh, Wh [Hp, 4Hp]).  Same work split as csrc/gru.cu: one CTA owns SB sessions, slots sorted longest first so that
// finished sessions cost nothing; rows are the valid positions only; the k-slices of a product meet in shared memory.
//
// Saved for the backward pass: the forward overwrites gx in place with the ACTIVATED gates
// (sigmoid(i) | tanh(j) | sigmoid(f + 1) | sigmoid(o)), and writes the cell state c' of every row to c_out [L, Hp] and
// the output h' to h_out [L, Hp].  The backward reads the previous row of c_out / h_out for c and h entering a step.
#include "common.cuh"

namespace nar {
namespace lstm {

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
  // longest first: at step t the sessions still running are slots [0, na)
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

// part[kq][s][0..NW) = v[s][k0 .. k0+kspan) * W[k, :NW] for this thread's 4 columns (jc) ; W row stride = NW floats
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

// thread layout for a [K, NW] matrix: NG = NW/4 column groups, NSPLIT = THREADS/NG k-slices (NG may exceed THREADS:
// then each thread walks several column groups with NSPLIT = 1)
struct Split { int ng, nsplit, kspan; };
__device__ __host__ __forceinline__ Split make_split(int K, int NW) {
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

// shared: h[SB][Hp] | c[SB][Hp] | part[NSPLIT][SB][4Hp]
// (min blocks 1: with the default bound ptxas settles on 64 registers and spills 8 bytes; at 94 registers 2 CTAs fit an SM)
__global__ void __launch_bounds__(THREADS, 1)
lstm_fwd_kernel(float* __restrict__ gx, const float* __restrict__ Wh, const int32_t* __restrict__ sess_off, int64_t B, int Hp,
                float* __restrict__ h_out, float* __restrict__ c_out) {
  extern __shared__ float sh[];
  float* h = sh;
  float* cs = h + SB * Hp;
  float* part = cs + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int W4 = 4 * Hp;
  const int ns = make_split(Hp, W4).nsplit;
  for (int i = threadIdx.x; i < 2 * SB * Hp; i += THREADS) sh[i] = 0.f;
  __syncthreads();
  for (int t = 0; t < ss.maxlen; ++t) {
    if (t > 0) product(active_sessions(ss, t), Wh, Hp, W4, h, Hp, part);
    __syncthreads();
    // thread j owns unit j of every session (reads and writes only its own h / c entries in this phase)
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (t < ss.len[s]) {
          const int64_t r = ss.off[s] + t;
          float* g = gx + r * W4;
          float ai = g[j], aj = g[Hp + j], af = g[2 * Hp + j], ao = g[3 * Hp + j];
          if (t > 0)
            for (int q = 0; q < ns; ++q) {
              const float* p = part + (int64_t)(q * SB + s) * W4;
              ai += p[j]; aj += p[Hp + j]; af += p[2 * Hp + j]; ao += p[3 * Hp + j];
            }
          const float i = sigmoidf(ai), gg = tanhf(aj), f = sigmoidf(af + 1.0f), o = sigmoidf(ao);
          const float c = f * cs[s * Hp + j] + i * gg;
          const float hn = o * tanhf(c);
          g[j] = i; g[Hp + j] = gg; g[2 * Hp + j] = f; g[3 * Hp + j] = o;
          c_out[r * Hp + j] = c; h_out[r * Hp + j] = hn;
          cs[s * Hp + j] = c; h[s * Hp + j] = hn;
        }
      }
    }
    __syncthreads();
  }
}

// backward through time.  act [L,4Hp] = activated gates of the forward; d_gx [L,4Hp] = dL/d(pre-activations i | j | f | o);
// h_prev [L,Hp] = h entering the step (dWh = h_prev^T d_gx).  dc and dh are carried from step t to t-1:
//     dc_t = dc + dh * o * (1 - tanh^2 c) ;  d_i = dc_t * g * i(1-i) ; d_j = dc_t * i * (1-g^2) ; d_f = dc_t * c_prev * f(1-f)
//     d_o = dh * tanh(c) * o(1-o) ;  dc <- dc_t * f ;  dh <- [d_i | d_j | d_f | d_o] * Wh^T
// shared: dgate[SB][4Hp] | dh[SB][Hp] | dc[SB][Hp] | part[NSPLIT][SB][Hp]
__global__ void __launch_bounds__(THREADS)
lstm_bwd_kernel(const float* __restrict__ d_hout, const float* __restrict__ h_out, const float* __restrict__ c_out,
                const float* __restrict__ act, const float* __restrict__ WhT /*[4Hp,Hp]*/, const int32_t* __restrict__ sess_off,
                int64_t B, int Hp, float* __restrict__ d_gx, float* __restrict__ h_prev) {
  extern __shared__ float sh[];
  const int W4 = 4 * Hp;
  float* dgate = sh;
  float* dh = dgate + SB * W4;
  float* dc = dh + SB * Hp;
  float* part = dc + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int ns = make_split(W4, Hp).nsplit;
  for (int i = threadIdx.x; i < 2 * SB * Hp; i += THREADS) dh[i] = 0.f;       // dh | dc
  __syncthreads();
  for (int t = ss.maxlen - 1; t >= 0; --t) {
    for (int j = threadIdx.x; j < Hp; j += THREADS) {
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        float di = 0.f, dj = 0.f, df = 0.f, dO = 0.f;
        if (t < ss.len[s]) {
          const int64_t r = ss.off[s] + t;
          const float* a = act + r * W4;
          const float i = a[j], g = a[Hp + j], f = a[2 * Hp + j], o = a[3 * Hp + j];
          const float c = c_out[r * Hp + j];
          const float cp = t > 0 ? c_out[(r - 1) * Hp + j] : 0.f;
          const float hp = t > 0 ? h_out[(r - 1) * Hp + j] : 0.f;
          const float dht = d_hout[r * Hp + j] + dh[s * Hp + j];
          const float tc = tanhf(c);
          dO = dht * tc * o * (1.0f - o);
          const float dct = dc[s * Hp + j] + dht * o * (1.0f - tc * tc);
          di = dct * g * i * (1.0f - i);
          dj = dct * i * (1.0f - g * g);
          df = dct * cp * f * (1.0f - f);
          dc[s * Hp + j] = dct * f;
          float* d = d_gx + r * W4;
          d[j] = di; d[Hp + j] = dj; d[2 * Hp + j] = df; d[3 * Hp + j] = dO;
          h_prev[r * Hp + j] = hp;
        }
        float* dg = dgate + s * W4;
        dg[j] = di; dg[Hp + j] = dj; dg[2 * Hp + j] = df; dg[3 * Hp + j] = dO;
      }
    }
    __syncthreads();
    if (t > 0) {
      // d(state entering step t) of the slots still running at t (slots past na carry zero gradients)
      product(active_sessions(ss, t), WhT, W4, Hp, dgate, W4, part);
      __syncthreads();
      for (int k = threadIdx.x; k < Hp; k += THREADS) {
#pragma unroll
        for (int s = 0; s < SB; ++s) {
          if (t < ss.len[s]) {
            float v = 0.f;
            for (int q = 0; q < ns; ++q) v += part[(int64_t)(q * SB + s) * Hp + k];
            dh[s * Hp + k] = v;
          }
        }
      }
    }
    __syncthreads();
  }
}

// The rnn_units the other cells accept (Hp/4 divides THREADS, the UGRNN split divides Hp), and even k-slices in both
// products here: K = Hp over NW = 4Hp (forward), K = 4Hp over NW = Hp (backward)
static inline bool shape_ok(int64_t Hp) {
  if (Hp <= 0 || Hp > MAX_HP || (Hp & 3)) return false;
  const int64_t ng = Hp / 4;
  if (ng > THREADS || THREADS % ng != 0 || Hp % (THREADS / ng) != 0) return false;
  auto ok = [](int64_t K, int64_t NW) {
    const int64_t g = NW / 4;
    if (g >= THREADS) return true;
    if (THREADS % g) return false;
    return (K % (THREADS / g)) == 0;
  };
  return ok(Hp, 4 * Hp) && ok(4 * Hp, Hp);
}
static inline int64_t nsplit_of(int64_t NW) { const int64_t ng = NW / 4; return ng >= THREADS ? 1 : THREADS / ng; }
static inline size_t fwd_smem(int64_t Hp) { return (size_t)(2 * SB * Hp + nsplit_of(4 * Hp) * SB * 4 * Hp) * sizeof(float); }
static inline size_t bwd_smem(int64_t Hp) { return (size_t)(SB * 4 * Hp + 2 * SB * Hp + nsplit_of(Hp) * SB * Hp) * sizeof(float); }

}  // namespace lstm
}  // namespace nar

extern "C" int nar_lstm_fwd(nar_ctx* ctx, float* gx, const float* Wh, const int32_t* sess_off, int64_t B, int64_t Hp, float* h_out,
                            float* c_out, void* stream) {
  using namespace nar::lstm;
  if (!ctx || !gx || !Wh || !sess_off || !h_out || !c_out) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const size_t smem = fwd_smem(Hp);
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(lstm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  lstm_fwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(gx, Wh, sess_off, B, (int)Hp, h_out, c_out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_lstm_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* c_out, const float* act,
                            const float* WhT, const int32_t* sess_off, int64_t B, int64_t Hp, float* d_gx, float* h_prev,
                            void* stream) {
  using namespace nar::lstm;
  if (!ctx || !d_hout || !h_out || !c_out || !act || !WhT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const size_t smem = bwd_smem(Hp);
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(lstm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  lstm_bwd_kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(d_hout, h_out, c_out, act, WhT, sess_off, B,
                                                                                       (int)Hp, d_gx, h_prev);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
