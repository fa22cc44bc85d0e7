// Recurrences of the session RNN's three cells inside dynamic_rnn (nar_model.py:1308-1342), selected with rnn_cell:
// UGRNN (tf.contrib.rnn.UGRNNCell, :1318, the reference's cell), GRU (tf.nn.rnn_cell.GRUCell, :1315) and LSTM
// (tf.nn.rnn_cell.LSTMCell, :1316).  The input projection x*Wx + b of ALL time steps is done by wgmma GEMMs (nar_gemm_tf32)
// into gx; what is left is the sequential part, independent per session.  Rows are the valid positions only (session b owns
// rows [sess_off[b], sess_off[b+1])), so "zero output / state pass-through past sequence_length" needs no work at all.
//
// The six kernels share one work split.  One CTA owns SB sessions and walks their time steps.  Per step every recurrent
// matrix streams from L2 exactly once per CTA: thread (kq, jc) of a product owns CB column groups of 4 (float4 loads,
// coalesced rows) for a 1/nsplit slice of k, 8-deep unrolled; the k-slices' partial sums meet in shared memory, where the
// cell's finalise phase adds them.  (Wh is 512 KB at H=256: it does not fit in one SM's shared memory in fp32; a
// cluster-resident variant is queued in DESIGN.md.)
#include "common.cuh"
#include <algorithm>

namespace nar {
namespace rnn {

constexpr int SB = 4;             // sessions per CTA (8 -> 4: 64 CTAs at batch 256, and the early all-active steps cost half)
constexpr int THREADS = 256;
constexpr int MAX_HP = 1024;
constexpr int MAX_SMEM = 200 * 1024;

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

// part[kq][s][b*NW/CB + 4jc ..+4) = v[s][k0 .. k0+kspan) * W[k, b*NW/CB + 4jc ..+4) for b < CB: this thread's CB column
// groups, NW/CB columns apart; W row stride = NW floats
template <int NA, int CB>
__device__ __forceinline__ void matvec(const float* __restrict__ W, int NW, const float* v, int ldv, float* part, int k0, int kspan,
                                       int jc, int kq) {
  float4 acc[NA][CB];
#pragma unroll
  for (int s = 0; s < NA; ++s)
#pragma unroll
    for (int b = 0; b < CB; ++b) acc[s][b] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* w[CB];
#pragma unroll
  for (int b = 0; b < CB; ++b) w[b] = reinterpret_cast<const float4*>(W + (int64_t)k0 * NW + b * (NW / CB)) + jc;
  const int stride4 = NW >> 2, block4 = stride4 / CB;
#pragma unroll 8
  for (int k = 0; k < kspan; ++k) {
    float4 a[CB];
#pragma unroll
    for (int b = 0; b < CB; ++b) a[b] = __ldg(w[b] + (int64_t)k * stride4);
#pragma unroll
    for (int s = 0; s < NA; ++s) {
      const float hv = v[s * ldv + k0 + k];
#pragma unroll
      for (int b = 0; b < CB; ++b) fma4(acc[s][b], hv, a[b]);
    }
  }
#pragma unroll
  for (int s = 0; s < NA; ++s)
#pragma unroll
    for (int b = 0; b < CB; ++b) *(reinterpret_cast<float4*>(part + (int64_t)(kq * SB + s) * NW) + b * block4 + jc) = acc[s][b];
}

template <int CB>
__device__ __forceinline__ void matvec_dyn(int na, const float* __restrict__ W, int NW, const float* v, int ldv, float* part, int k0,
                                           int kspan, int jc, int kq) {
  if (na <= 1) matvec<1, CB>(W, NW, v, ldv, part, k0, kspan, jc, kq);
  else if (na <= 2) matvec<2, CB>(W, NW, v, ldv, part, k0, kspan, jc, kq);
  else matvec<SB, CB>(W, NW, v, ldv, part, k0, kspan, jc, kq);
}

// thread layout of a product over an [K, NW] matrix: ng = NW/(4 CB) thread columns, nsplit = THREADS/ng k-slices (ng may
// reach THREADS: then each thread walks several column groups with nsplit = 1)
struct Split { int ng, nsplit, kspan; };
template <int CB = 1>
__host__ __device__ __forceinline__ Split make_split(int K, int NW) {
  Split s; s.ng = (NW >> 2) / CB;
  s.nsplit = s.ng >= THREADS ? 1 : THREADS / s.ng;
  s.kspan = K / s.nsplit;
  return s;
}
// all threads: part[q][s][:NW) = v[s][:K) * W for q < nsplit and the na sessions still running.  (The UGRNN kernels, whose
// ng never exceeds THREADS, call matvec_dyn with (jc, kq) worked out once per kernel.)
__device__ __forceinline__ void product(int na, const float* __restrict__ W, int K, int NW, const float* v, int ldv, float* part) {
  const Split sp = make_split(K, NW);
  if (sp.ng >= THREADS) {
    for (int jc = threadIdx.x; jc < sp.ng; jc += THREADS) matvec_dyn<1>(na, W, NW, v, ldv, part, 0, K, jc, 0);
  } else {
    const int jc = threadIdx.x % sp.ng, kq = threadIdx.x / sp.ng;
    if (kq < sp.nsplit) matvec_dyn<1>(na, W, NW, v, ldv, part, kq * sp.kspan, sp.kspan, jc, kq);
  }
}

// ================================================================================================ UGRNN
//     act = gx[t] + h * Wh ;  g = sigmoid(act_g + 1) ; c = tanh(act_c) ; h' = g*h + (1-g)*c
// gx [L, 2Hp] (gate | candidate), Wh [Hp, 2Hp].  The forward product gives each thread one gate and one candidate column
// group (CB = 2), so 16 independent 128-bit loads are in flight per thread, and splits k by Hp/4 thread columns.
// shape_ok makes ng divide THREADS in both UGRNN products, so every thread owns one (jc, kq).
// shared: h[SB][Hp] | part[NSPLIT][SB][2][Hp]
__global__ void __launch_bounds__(THREADS)
ugrnn_fwd_kernel(const float* __restrict__ gx, const float* __restrict__ Wh, const int32_t* __restrict__ sess_off,
                 int64_t B, int Hp, float* __restrict__ h_out, float* __restrict__ gate, float* __restrict__ cand) {
  extern __shared__ float sh[];
  float* h = sh;
  float* part = sh + SB * Hp;
  const Sess ss = load_sessions(sess_off, B);
  const int W2 = 2 * Hp;
  const Split sp = make_split<2>(Hp, W2);
  const int NSPLIT = sp.nsplit, jc = threadIdx.x % sp.ng, kq = threadIdx.x / sp.ng, k0 = kq * sp.kspan;
  for (int i = threadIdx.x; i < SB * Hp; i += THREADS) h[i] = 0.f;
  __syncthreads();
  for (int t = 0; t < ss.maxlen; ++t) {
    // sessions that reach step t also had step t-1, so slots [0, na) are exactly the ones with a live state
    if (t > 0) matvec_dyn<2>(active_sessions(ss, t), Wh, W2, h, Hp, part, k0, sp.kspan, jc, kq);
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
  const Split sp = make_split(W2, Hp);
  const int NSPLIT = sp.nsplit, jc = threadIdx.x % sp.ng, kq = threadIdx.x / sp.ng, k0 = kq * sp.kspan;
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
      matvec_dyn<1>(active_sessions(ss, t), WhT, Hp, dact, W2, part, k0, sp.kspan, jc, kq);   // d_act of the slots past na is zero at this step
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

// ================================================================================================ GRU
// tf.nn.rnn_cell.GRUCell (TF 1.12 rnn_cell_impl.py):
//     [r, u] = sigmoid([x, h] * Wg + bg)          gates/kernel [in+H, 2H], gates/bias (initialised to 1.0)
//     c      = tanh([x, r*h] * Wc + bc)           candidate/kernel [in+H, H], candidate/bias
//     h'     = u * h + (1 - u) * c
// gx [L, 3Hp] = (r | u | c) input projections; TWO dependent products per step (h * Whg, then (r*h) * Whc).
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

// ================================================================================================ LSTM
// tf.nn.rnn_cell.LSTMCell (TF 1.12 rnn_cell_impl.py; no peepholes, no cell clip, no projection, forget_bias 1.0):
//     z  = [x, h] * kernel + bias                 kernel [in+H, 4H], bias [4H], columns i | j | f | o
//     c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j)
//     h' = sigmoid(o) * tanh(c')                  output = h', state = (c', h')
// gx [L, 4Hp] (column blocks i | j | f | o, each Hp wide); ONE product per step (h * Wh, Wh [Hp, 4Hp]).
// Saved for the backward pass: the forward overwrites gx in place with the ACTIVATED gates
// (sigmoid(i) | tanh(j) | sigmoid(f + 1) | sigmoid(o)), and writes the cell state c' of every row to c_out [L, Hp] and
// the output h' to h_out [L, Hp].  The backward reads the previous row of c_out / h_out for c and h entering a step.
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

// ================================================================================================ host
// Every product a cell runs splits K evenly over its k-slices.  (K, NW, CB): UGRNN (Hp, 2Hp, 2), (2Hp, Hp, 1);
// GRU (Hp, 2Hp, 1), (Hp, Hp, 1), (2Hp, Hp, 1); LSTM (Hp, 4Hp, 1), (4Hp, Hp, 1).  Accepts Hp = 32, 64, ..., 1024.
template <int CB = 1>
static bool splits_evenly(int K, int NW) {
  const Split sp = make_split<CB>(K, NW);
  return sp.ng >= THREADS || (THREADS % sp.ng == 0 && K % sp.nsplit == 0);
}
static bool shape_ok(int64_t Hp) {
  if (Hp <= 0 || Hp > MAX_HP || (Hp & 3)) return false;
  const int H = (int)Hp;
  return splits_evenly<2>(H, 2 * H) && splits_evenly(2 * H, H) && splits_evenly(H, 2 * H) && splits_evenly(H, H) &&
         splits_evenly(H, 4 * H) && splits_evenly(4 * H, H);
}
// floats of a product's partial sums part[nsplit][SB][NW]
template <int CB = 1>
static size_t part_floats(int64_t K, int64_t NW) { return (size_t)make_split<CB>((int)K, (int)NW).nsplit * SB * NW; }

// The shared memory attribute is set once per kernel, keyed on the kernel itself: ugrnn_bwd_kernel and lstm_bwd_kernel
// have the same function type, and each needs the attribute (80 and 112 KB at Hp 1024).
template <auto Kernel> bool smem_attr_set = false;

template <auto Kernel, typename... Args>
static int launch(int64_t B, size_t smem_floats, void* stream, Args... args) {
  const size_t smem = smem_floats * sizeof(float);
  if (smem > MAX_SMEM) return NAR_ERR_UNSUPPORTED;
  if (!smem_attr_set<Kernel>) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM));
    smem_attr_set<Kernel> = true;
  }
  Kernel<<<(unsigned)((B + SB - 1) / SB), THREADS, smem, as_stream(stream)>>>(args...);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

}  // namespace rnn
}  // namespace nar

using namespace nar::rnn;

extern "C" int nar_ugrnn_fwd(nar_ctx* ctx, const float* gx, const float* Wh, const int32_t* sess_off, int64_t B, int64_t Hp,
                             float* h_out, float* gate, float* cand, void* stream) {
  if (!ctx || !gx || !Wh || !sess_off || !h_out || !gate || !cand) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  return launch<ugrnn_fwd_kernel>(B, SB * Hp + part_floats<2>(Hp, 2 * Hp), stream, gx, Wh, sess_off, B, (int)Hp, h_out, gate, cand);
}

extern "C" int nar_ugrnn_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* gate, const float* cand,
                             const float* WhT, const int32_t* sess_off, int64_t B, int64_t Hp, float* d_gx, float* h_prev,
                             void* stream) {
  if (!ctx || !d_hout || !h_out || !gate || !cand || !WhT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  return launch<ugrnn_bwd_kernel>(B, 4 * SB * Hp + part_floats(2 * Hp, Hp), stream, d_hout, h_out, gate, cand, WhT, sess_off, B,
                                  (int)Hp, d_gx, h_prev);
}

extern "C" int nar_gru_fwd(nar_ctx* ctx, const float* gx, const float* Whg, const float* Whc, const int32_t* sess_off, int64_t B,
                           int64_t Hp, float* h_out, float* r_out, float* u_out, float* c_out, float* rh_out, void* stream) {
  if (!ctx || !gx || !Whg || !Whc || !sess_off || !h_out || !r_out || !u_out || !c_out || !rh_out) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  const size_t part = std::max(part_floats(Hp, 2 * Hp), part_floats(Hp, Hp));     // the two products share part
  return launch<gru_fwd_kernel>(B, 2 * SB * Hp + part, stream, gx, Whg, Whc, sess_off, B, (int)Hp, h_out, r_out, u_out, c_out,
                                rh_out);
}

extern "C" int nar_gru_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* r_out, const float* u_out,
                           const float* c_out, const float* WhgT, const float* WhcT, const int32_t* sess_off, int64_t B, int64_t Hp,
                           float* d_gx, float* h_prev, void* stream) {
  if (!ctx || !d_hout || !h_out || !r_out || !u_out || !c_out || !WhgT || !WhcT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  // both backward products write [nsplit][SB][Hp], with the same nsplit
  return launch<gru_bwd_kernel>(B, 5 * SB * Hp + part_floats(Hp, Hp), stream, d_hout, h_out, r_out, u_out, c_out, WhgT, WhcT,
                                sess_off, B, (int)Hp, d_gx, h_prev);
}

extern "C" int nar_lstm_fwd(nar_ctx* ctx, float* gx, const float* Wh, const int32_t* sess_off, int64_t B, int64_t Hp, float* h_out,
                            float* c_out, void* stream) {
  if (!ctx || !gx || !Wh || !sess_off || !h_out || !c_out) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  return launch<lstm_fwd_kernel>(B, 2 * SB * Hp + part_floats(Hp, 4 * Hp), stream, gx, Wh, sess_off, B, (int)Hp, h_out, c_out);
}

extern "C" int nar_lstm_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* c_out, const float* act,
                            const float* WhT, const int32_t* sess_off, int64_t B, int64_t Hp, float* d_gx, float* h_prev,
                            void* stream) {
  if (!ctx || !d_hout || !h_out || !c_out || !act || !WhT || !sess_off || !d_gx || !h_prev) return NAR_ERR_INVALID;
  if (!shape_ok(Hp)) return NAR_ERR_UNSUPPORTED;
  if (B <= 0) return NAR_OK;
  return launch<lstm_bwd_kernel>(B, 6 * SB * Hp + part_floats(4 * Hp, Hp), stream, d_hout, h_out, c_out, act, WhT, sess_off, B,
                                 (int)Hp, d_gx, h_prev);
}
