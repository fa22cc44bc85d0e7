// Scorer tail + loss of the NAR hot path.
//   mul_pred / mul_pred_bwd : tf.multiply(candidate_embedding, predicted_embedding) nar_model.py:478,:493
//   score_softmax_ce        : matching_dense_layer_4 (32 -> 1, :468-473,:485,:499), / temperature (:514),
//                             softmax (:515), -log p0 * mask / sum(mask) (:660-664) and its gradient
//   cosine_softmax_ce       : north_star wording (l2-normalise + dot, nar_model.py:437 commented out)
// Candidate rows of position l are contiguous: row l*n_cand + j, j = 0 positive, 1..K negatives.
#include "common.cuh"

namespace nar {
namespace loss {

__global__ void __launch_bounds__(256)
mul_pred_kernel(const float4* __restrict__ cand, const float4* __restrict__ pred, int64_t n_rows, int64_t n_cand, int C4,
                float4* __restrict__ prod) {
  const int64_t total = n_rows * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C4; const int c = (int)(i - r * C4);
    const float4 a = cand[i]; const float4 b = __ldg(pred + (r / n_cand) * C4 + c);
    prod[i] = make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
  }
}

// one CTA per position: d_cand rows written, d_pred reduced over the n_cand candidates (no atomics)
__global__ void __launch_bounds__(256)
mul_pred_bwd_kernel(const float4* __restrict__ d_prod, const float4* __restrict__ cand, const float4* __restrict__ pred,
                    int64_t n_cand, int C4, int cand_act, float4* __restrict__ d_cand, float4* __restrict__ d_pred) {
  const int64_t l = blockIdx.x;
  for (int c = threadIdx.x; c < C4; c += blockDim.x) {
    const float4 p = pred[l * C4 + c];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t j = 0; j < n_cand; ++j) {
      const int64_t i = (l * n_cand + j) * C4 + c;
      const float4 d = d_prod[i]; const float4 e = cand[i];
      // optionally straight through the activation that produced cand (CAR tanh): d_cand is then d(pre-activation)
      d_cand[i] = make_float4(d.x * p.x * act_grad_from_output(e.x, cand_act), d.y * p.y * act_grad_from_output(e.y, cand_act),
                              d.z * p.z * act_grad_from_output(e.z, cand_act), d.w * p.w * act_grad_from_output(e.w, cand_act));
      acc.x = fmaf(d.x, e.x, acc.x); acc.y = fmaf(d.y, e.y, acc.y); acc.z = fmaf(d.z, e.z, acc.z); acc.w = fmaf(d.w, e.w, acc.w);
    }
    d_pred[l * C4 + c] = acc;
  }
}

// Novelty regulariser (nar_model.py:517, :531-544, :673-683): total_loss -= factor * sum_l mask_l * sum_k q_lk * nov_lk
// / sum(mask), q = softmax over the NEGATIVES only of the scaled scores, nov = -log_base(articles_recent_pop_norm[id]).
// d/d(scaled score k) = -factor * inv_count * q_k * (nov_k - sum_j q_j nov_j); fused into the two softmax-CE kernels.
struct NovArgs { float factor, inv_log_base; const float* pop_norm; const int64_t* cand_ids; float* loss_nov; };

__device__ __forceinline__ float nov_of(const NovArgs& nv, int64_t l, int64_t n_cand, int64_t j) {
  return -__fmul_rn(logf(nv.pop_norm[nv.cand_ids[l * n_cand + j]]), nv.inv_log_base);
}
// warp-cooperative: log-sum-exp of the negatives' scaled scores and their probability-weighted mean novelty
__device__ __forceinline__ void nov_stats(const NovArgs& nv, const float* lg, int64_t l, int64_t n_cand, int lane, float& lse_n,
                                          float& nbar) {
  float mx = -INFINITY;
  for (int64_t j = 1 + lane; j < n_cand; j += 32) mx = fmaxf(mx, lg[j]);
  mx = warp_max(mx);
  float se = 0.f, sn = 0.f;
  for (int64_t j = 1 + lane; j < n_cand; j += 32) { const float e = expf(lg[j] - mx); se += e; sn = fmaf(e, nov_of(nv, l, n_cand, j), sn); }
  se = warp_sum(se); sn = warp_sum(sn);
  lse_n = mx + logf(se);
  nbar = sn / se;
}

// one warp per position
constexpr int CE_WARPS = 4;

__global__ void __launch_bounds__(CE_WARPS * 32)
score_softmax_ce_kernel(const float* __restrict__ z3, int64_t ld_z, int width, const float* __restrict__ m4, int64_t ld_m4,
                        const float* __restrict__ c4, int64_t n_pos, int64_t n_cand, float inv_temp, float inv_count,
                        float* __restrict__ logits, float* __restrict__ loss_sum, float* __restrict__ d_z3,
                        float* __restrict__ d_m4, float* __restrict__ d_c4, const NovArgs nv) {
  const int lane = threadIdx.x & 31;
  const int64_t l = (int64_t)blockIdx.x * CE_WARPS + (threadIdx.x >> 5);
  if (l >= n_pos) return;
  const float bias = c4[0];
  float* lg = logits + l * n_cand;
  float mx = -INFINITY;
  for (int64_t j = lane; j < n_cand; j += 32) {
    const float* z = z3 + (l * n_cand + j) * ld_z;
    float s = bias;
    for (int k = 0; k < width; ++k) s = fmaf(z[k], __ldg(m4 + (int64_t)k * ld_m4), s);
    s *= inv_temp;
    lg[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  __syncwarp();
  float se = 0.f;
  for (int64_t j = lane; j < n_cand; j += 32) se += expf(lg[j] - mx);
  se = warp_sum(se);
  const float lse = mx + logf(se);
  if (lane == 0) atomicAdd(loss_sum, -(lg[0] - lse) * inv_count);
  float lse_n = 0.f, nbar = 0.f;
  const bool use_nov = nv.factor > 0.f && n_cand > 1;
  if (use_nov) {
    __syncwarp();
    nov_stats(nv, lg, l, n_cand, lane, lse_n, nbar);
    if (lane == 0) atomicAdd(nv.loss_nov, nv.factor * nbar * inv_count);
  }
  if (d_z3 == nullptr) return;
  // gradient: d logit_j = (softmax_j - [j==0]) * inv_count ; ds_j = d logit_j * inv_temp
  float dc = 0.f;
  for (int64_t j = lane; j < n_cand; j += 32) {
    const float pj = expf(lg[j] - lse);
    float ds = (pj - (j == 0 ? 1.f : 0.f)) * inv_count * inv_temp;
    if (use_nov && j > 0) ds -= nv.factor * inv_count * inv_temp * expf(lg[j] - lse_n) * (nov_of(nv, l, n_cand, j) - nbar);
    dc += ds;
    const float* z = z3 + (l * n_cand + j) * ld_z;
    float* dz = d_z3 + (l * n_cand + j) * ld_z;
    for (int k = 0; k < width; ++k) {
      const float zk = z[k];
      dz[k] = ds * __ldg(m4 + (int64_t)k * ld_m4) * (zk > 0.f ? 1.f : 0.2f);    // leaky' of matching_dense_layer_3
    }
  }
  dc = warp_sum(dc);
  if (lane == 0) atomicAdd(d_c4, dc);
  // d_m4[k] = sum_j ds_j * z3[j,k] : lane k (width <= 32 handled per 32-chunk)
  for (int k0 = 0; k0 < width; k0 += 32) {
    const int k = k0 + lane;
    float acc = 0.f;
    if (k < width) {
      for (int64_t j = 0; j < n_cand; ++j) {
        const float pj = expf(lg[j] - lse);
        float ds = (pj - (j == 0 ? 1.f : 0.f)) * inv_count * inv_temp;
        if (use_nov && j > 0) ds -= nv.factor * inv_count * inv_temp * expf(lg[j] - lse_n) * (nov_of(nv, l, n_cand, j) - nbar);
        acc = fmaf(ds, z3[(l * n_cand + j) * ld_z + k], acc);
      }
      atomicAdd(d_m4 + (int64_t)k * ld_m4, acc);
    }
  }
}

// cosine mode: one CTA (128 threads = 4 warps) per position; pred row staged in shared memory,
// each warp walks candidates, warp-shuffle dot products, then the same softmax-CE.
constexpr int COS_THREADS = 128;
// l2-normalisation floor on the norm, x / max(|x|, eps) (the oracle's F.normalize).  A norm held at the floor is a
// constant: the gradient of its row has no normalisation term.
constexpr float COS_EPS = 1e-12f;

__global__ void __launch_bounds__(COS_THREADS)
cosine_softmax_ce_kernel(const float* __restrict__ cand, const float* __restrict__ pred, int64_t n_cand, int C,
                         float inv_temp, float inv_count, float* __restrict__ logits, float* __restrict__ loss_sum,
                         float* __restrict__ d_cand, float* __restrict__ d_pred, const NovArgs nv) {
  extern __shared__ float sh[];
  float* sp = sh;                       // [C] pred row
  float* s_dot = sh + C;                // [n_cand] <cand_j, pred>
  float* s_nrm = s_dot + n_cand;        // [n_cand] |cand_j| (before the floor)
  float* s_ds = s_nrm + n_cand;         // [n_cand] d loss / d cos_j
  __shared__ float s_red[8];
  const int64_t l = blockIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float pp = 0.f;
  for (int c = threadIdx.x; c < C; c += COS_THREADS) { const float v = pred[l * C + c]; sp[c] = v; pp = fmaf(v, v, pp); }
  pp = warp_sum(pp);
  if (lane == 0) s_red[w] = pp;
  __syncthreads();
  const float pn_raw = sqrtf(s_red[0] + s_red[1] + s_red[2] + s_red[3]), pn = fmaxf(pn_raw, COS_EPS);
  const bool pn_live = pn_raw >= COS_EPS;
  for (int64_t j = w; j < n_cand; j += COS_THREADS / 32) {
    const float* e = cand + (l * n_cand + j) * C;
    float d = 0.f, n = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = e[c]; d = fmaf(v, sp[c], d); n = fmaf(v, v, n); }
    d = warp_sum(d); n = warp_sum(n);
    if (lane == 0) { s_dot[j] = d; s_nrm[j] = sqrtf(n); }
  }
  __syncthreads();
  float* lg = logits + l * n_cand;
  if (w == 0) {
    float mx = -INFINITY;
    for (int64_t j = lane; j < n_cand; j += 32) {
      const float s = s_dot[j] / (fmaxf(s_nrm[j], COS_EPS) * pn) * inv_temp;
      lg[j] = s; mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    __syncwarp();
    float se = 0.f;
    for (int64_t j = lane; j < n_cand; j += 32) se += expf(lg[j] - mx);
    se = warp_sum(se);
    const float lse = mx + logf(se);
    if (lane == 0) atomicAdd(loss_sum, -(lg[0] - lse) * inv_count);
    float lse_n = 0.f, nbar = 0.f;
    const bool use_nov = nv.factor > 0.f && n_cand > 1;
    if (use_nov) {
      __syncwarp();
      nov_stats(nv, lg, l, n_cand, lane, lse_n, nbar);
      if (lane == 0) atomicAdd(nv.loss_nov, nv.factor * nbar * inv_count);
    }
    for (int64_t j = lane; j < n_cand; j += 32) {
      float ds = (expf(lg[j] - lse) - (j == 0 ? 1.f : 0.f)) * inv_count * inv_temp;
      if (use_nov && j > 0) ds -= nv.factor * inv_count * inv_temp * expf(lg[j] - lse_n) * (nov_of(nv, l, n_cand, j) - nbar);
      s_ds[j] = ds;
    }
  }
  __syncthreads();
  if (d_cand == nullptr) return;
  // cos = <e,p>/(|e||p|) : d/de = p/(|e||p|) - cos * e/|e|^2 ; d/dp = e/(|e||p|) - cos * p/|p|^2 (no second term for a
  // floored norm)
  for (int c = threadIdx.x; c < C; c += COS_THREADS) {
    const float pc = sp[c];
    float dp = 0.f;
    for (int64_t j = 0; j < n_cand; ++j) {
      const float en = fmaxf(s_nrm[j], COS_EPS), cs = s_dot[j] / (en * pn), ds = s_ds[j];
      const float ce = s_nrm[j] >= COS_EPS ? cs : 0.f, cp = pn_live ? cs : 0.f;
      const float ec = cand[(l * n_cand + j) * C + c];
      d_cand[(l * n_cand + j) * C + c] = ds * (pc / (en * pn) - ce * ec / (en * en));
      dp = fmaf(ds, ec / (en * pn) - cp * pc / (pn * pn), dp);
    }
    d_pred[l * C + c] = dp;
  }
}


// ---------------------------------------------------------------- evaluation ranking
// one warp per position: softmax probabilities in shared memory, rank of candidate i = number of candidates that
// precede it in tf.nn.top_k order (higher probability, or equal probability and lower index).
constexpr int RANK_WARPS = 4;

__global__ void __launch_bounds__(RANK_WARPS * 32)
rank_candidates_kernel(const float* __restrict__ logits, const int64_t* __restrict__ cand_ids, int64_t n_pos, int n_cand,
                       int top_n, int64_t* __restrict__ pred_ids, float* __restrict__ pred_probs, double* __restrict__ metrics) {
  extern __shared__ float sh[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t l = (int64_t)blockIdx.x * RANK_WARPS + w;
  if (l >= n_pos) return;
  float* p = sh + (size_t)w * n_cand;
  const float* lg = logits + l * n_cand;
  float mx = -INFINITY;
  for (int j = lane; j < n_cand; j += 32) mx = fmaxf(mx, lg[j]);
  mx = warp_max(mx);
  float se = 0.f;
  for (int j = lane; j < n_cand; j += 32) { const float e = expf(lg[j] - mx); p[j] = e; se += e; }
  se = warp_sum(se);
  __syncwarp();
  for (int j = lane; j < n_cand; j += 32) p[j] = p[j] / se;
  __syncwarp();
  for (int i = lane; i < n_cand; i += 32) {
    const float pi = p[i];
    int rank = 0;
    for (int j = 0; j < n_cand; ++j) { const float pj = p[j]; rank += (pj > pi || (pj == pi && j < i)) ? 1 : 0; }
    if (pred_ids) pred_ids[l * n_cand + rank] = cand_ids[l * n_cand + i];
    if (pred_probs) pred_probs[l * n_cand + rank] = pi;
    if (i == 0 && metrics) {
      // float64 accumulators: hit / label counts stay exact (integers below 2^53), the reciprocal-rank sum keeps
      // ~1e-16 relative rounding whatever the order of the atomics
      if (rank < top_n) { atomicAdd(metrics + 0, 1.0); atomicAdd(metrics + 1, 1.0 / (double)(rank + 1)); }
      atomicAdd(metrics + 2, 1.0);
    }
  }
}

}  // namespace loss
}  // namespace nar

extern "C" int nar_mul_pred(const float* cand, const float* pred, int64_t n_pos, int64_t n_cand, int64_t C, float* prod, void* stream) {
  if (!cand || !pred || !prod || (C & 3)) return NAR_ERR_INVALID;
  const int64_t rows = n_pos * n_cand;
  if (rows <= 0) return NAR_OK;
  const int64_t total = rows * (C / 4);
  const unsigned grid = (unsigned)((total + 255) / 256 > NAR_GRID_SMS * 16 ? NAR_GRID_SMS * 16 : (total + 255) / 256);
  nar::loss::mul_pred_kernel<<<grid, 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(cand), reinterpret_cast<const float4*>(pred),
                                                                   rows, n_cand, (int)(C / 4), reinterpret_cast<float4*>(prod));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_mul_pred_bwd(const float* d_prod, const float* cand, const float* pred, int64_t n_pos, int64_t n_cand, int64_t C,
                                int cand_act, float* d_cand, float* d_pred, void* stream) {
  if (!d_prod || !cand || !pred || !d_cand || !d_pred || (C & 3)) return NAR_ERR_INVALID;
  if (n_pos <= 0) return NAR_OK;
  nar::loss::mul_pred_bwd_kernel<<<(unsigned)n_pos, 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(d_prod), reinterpret_cast<const float4*>(cand), reinterpret_cast<const float4*>(pred), n_cand,
      (int)(C / 4), cand_act, reinterpret_cast<float4*>(d_cand), reinterpret_cast<float4*>(d_pred));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_score_softmax_ce(const float* z3, int64_t ld_z, int64_t width, const float* m4, int64_t ld_m4, const float* c4,
                                    int64_t n_pos, int64_t n_cand, float inv_temperature, float inv_count, float* logits,
                                    float* loss_sum, float* d_z3, float* d_m4, float* d_c4, const nar_novelty_reg* nov,
                                    void* stream) {
  if (!z3 || !m4 || !c4 || !logits || !loss_sum) return NAR_ERR_INVALID;
  nar::loss::NovArgs nv = {0.f, 0.f, nullptr, nullptr, nullptr};
  if (nov && nov->factor > 0.f) {
    if (!nov->pop_norm || !nov->cand_ids || !nov->loss_nov || !(nov->log_base > 1.f)) return NAR_ERR_INVALID;
    nv.factor = nov->factor; nv.inv_log_base = 1.0f / logf(nov->log_base); nv.pop_norm = nov->pop_norm; nv.cand_ids = nov->cand_ids;
    nv.loss_nov = nov->loss_nov;
  }
  if (d_z3 && (!d_m4 || !d_c4)) return NAR_ERR_INVALID;
  if (n_pos <= 0) return NAR_OK;
  const unsigned grid = (unsigned)((n_pos + nar::loss::CE_WARPS - 1) / nar::loss::CE_WARPS);
  nar::loss::score_softmax_ce_kernel<<<grid, nar::loss::CE_WARPS * 32, 0, as_stream(stream)>>>(
      z3, ld_z, (int)width, m4, ld_m4, c4, n_pos, n_cand, inv_temperature, inv_count, logits, loss_sum, d_z3, d_m4, d_c4, nv);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_cosine_softmax_ce(const float* cand, const float* pred, int64_t n_pos, int64_t n_cand, int64_t C, float inv_temperature,
                                     float inv_count, float* logits, float* loss_sum, float* d_cand, float* d_pred,
                                     const nar_novelty_reg* nov, void* stream) {
  if (!cand || !pred || !logits || !loss_sum) return NAR_ERR_INVALID;
  nar::loss::NovArgs nv = {0.f, 0.f, nullptr, nullptr, nullptr};
  if (nov && nov->factor > 0.f) {
    if (!nov->pop_norm || !nov->cand_ids || !nov->loss_nov || !(nov->log_base > 1.f)) return NAR_ERR_INVALID;
    nv.factor = nov->factor; nv.inv_log_base = 1.0f / logf(nov->log_base); nv.pop_norm = nov->pop_norm; nv.cand_ids = nov->cand_ids;
    nv.loss_nov = nov->loss_nov;
  }
  if (d_cand && !d_pred) return NAR_ERR_INVALID;
  if (n_pos <= 0) return NAR_OK;
  const size_t smem = (size_t)(C + 3 * n_cand) * sizeof(float);
  if (smem > 48 * 1024) return NAR_ERR_UNSUPPORTED;
  // with the kernel's static s_red, the top 32 bytes of that range (which the engine's cosine_chunk_cap reaches) exceed
  // the 48 KB a launch gets without opting in
  if (smem > 48 * 1024 - 8 * sizeof(float))
    NAR_CHECK_CUDA(cudaFuncSetAttribute(nar::loss::cosine_softmax_ce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nar::loss::cosine_softmax_ce_kernel<<<(unsigned)n_pos, nar::loss::COS_THREADS, smem, as_stream(stream)>>>(
      cand, pred, n_cand, (int)C, inv_temperature, inv_count, logits, loss_sum, d_cand, d_pred, nv);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_rank_candidates(const float* logits, const int64_t* cand_ids, int64_t n_pos, int64_t n_cand, int32_t top_n,
                                   int64_t* pred_ids, float* pred_probs, double* metrics, void* stream) {
  if (!logits || !cand_ids) return NAR_ERR_INVALID;
  if (n_pos <= 0) return NAR_OK;
  if (n_cand <= 0 || top_n < 0) return NAR_ERR_INVALID;
  const size_t smem = (size_t)nar::loss::RANK_WARPS * n_cand * sizeof(float);
  if (smem > 48 * 1024) return NAR_ERR_UNSUPPORTED;
  const unsigned grid = (unsigned)((n_pos + nar::loss::RANK_WARPS - 1) / nar::loss::RANK_WARPS);
  nar::loss::rank_candidates_kernel<<<grid, nar::loss::RANK_WARPS * 32, smem, as_stream(stream)>>>(
      logits, cand_ids, n_pos, (int)n_cand, (int)top_n, pred_ids, pred_probs, metrics);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
