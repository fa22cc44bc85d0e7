// The evaluation hook's ranking-quality metrics beyond HR / MRR (the reference's ItemsStateUpdaterHook.create_eval_metrics,
// metrics.py): NDCG, item coverage, ESI-R / ESI-RR novelty and EILD-R / EILD-RR content diversity, computed from the
// top-n id lists the model and the baselines already leave on the device.  Spec: oracle/eval_metrics_ref.py.
//
// Per (recommender row, query) one CTA stages the list's ACR rows in shared memory, computes the m x m fp64 cosine
// distances and the five per-query values, and marks the ids in the row's recommended-items bitmap.  The per-query
// values go to a scratch array; a second launch sums them per row in a fixed order (no float atomics: the sums are
// bit-identical run to run).  Coverage sets are bitmaps over [0, V) set with integer atomicOr and counted by popcount.
#include "common.cuh"

namespace nar {
namespace em {

constexpr int LIST_THREADS = 128;
constexpr int REDUCE_THREADS = 256;
constexpr int MAX_M = 64;                  // list positions scored per query (top_n)
constexpr int N_VALUES = 6;                // per query: ndcg, esi-r, esi-rr, eild-r, eild-rr, 1 (the query count)
constexpr size_t MAX_LIST_SMEM = 200 * 1024;   // list_kernel's dynamic shared memory: [m, m] fp64 + [m, acr_dim] fp32

__device__ __forceinline__ double disc(int k) { return 1.0 / log2((double)(k + 2)); }

__global__ void mark_kernel(const int64_t* ids, int64_t n, int64_t num_items, int skip_zero, unsigned* bitmap, int* err) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t id = ids[i];
    if (id == 0 && skip_zero) continue;
    if (id < 0 || id >= num_items) { atomicExch(err, 1); continue; }
    atomicOr(bitmap + (id >> 5), 1u << (id & 31));
  }
}

struct ListArgs {
  const int64_t* ids; int64_t row_stride, q_stride, nq, len; int m;
  const int64_t* labels; int64_t label_stride;
  const float* pop; const float* acr; int64_t acr_dim, acr_ld; const double* acr_norm; int64_t num_items;
  double neg_rel; long long row_mask;
  double* per_query;                       // [rows, nq, N_VALUES]
  unsigned* rec; int64_t words;            // [rows, words]
  int* err;
};

// grid (nq, rows): one CTA per (query, recommender row)
__global__ void __launch_bounds__(LIST_THREADS) list_kernel(ListArgs a) {
  extern __shared__ unsigned char smem[];
  const int64_t q = blockIdx.x;
  const int row = blockIdx.y;
  if (!((a.row_mask >> row) & 1)) return;
  const int m = a.m, dim = (int)a.acr_dim;
  double* s_D = reinterpret_cast<double*>(smem);                           // [m, m] cosine distance / 2
  float* s_acr = reinterpret_cast<float*>(smem + sizeof(double) * m * m);  // [m, dim]
  __shared__ int64_t s_id[MAX_M];
  __shared__ double s_er[MAX_M], s_err[MAX_M];
  __shared__ int s_occ, s_bad;
  double* out = a.per_query + ((int64_t)row * a.nq + q) * N_VALUES;
  const int64_t label = a.labels[q * a.label_stride];
  if (label == 0) {
    if (threadIdx.x < N_VALUES) out[threadIdx.x] = 0.0;
    return;
  }
  const int64_t* list = a.ids + row * a.row_stride + q * a.q_stride;
  if (threadIdx.x == 0) { s_occ = 0; s_bad = label < 0 || label >= a.num_items; }
  __syncthreads();
  int occ = 0;
  for (int64_t j = threadIdx.x; j < a.len; j += blockDim.x) {
    const int64_t id = list[j];
    occ += id == label;
    if (j < m) {
      s_id[j] = id;
      if (id < 0 || id >= a.num_items) s_bad = 1;
    }
  }
  if (occ) atomicAdd(&s_occ, occ);
  __syncthreads();
  if (s_bad) {
    if (threadIdx.x == 0) atomicExch(a.err, 1);
    if (threadIdx.x < N_VALUES) out[threadIdx.x] = 0.0;
    return;
  }
  if (threadIdx.x < m) {
    const int64_t id = s_id[threadIdx.x];
    atomicOr(a.rec + row * a.words + (id >> 5), 1u << (id & 31));
  }
  for (int idx = threadIdx.x; idx < m * dim; idx += blockDim.x) {
    const int i = idx / dim, k = idx - i * dim;
    s_acr[idx] = a.acr[s_id[i] * a.acr_ld + k];
  }
  __syncthreads();
  // pairwise distances, sklearn's cosine_distances / 2: clip(1 - cos, 0, 2) / 2, cos = 0 when a row has norm 0
  for (int p = threadIdx.x; p < m * m; p += blockDim.x) {
    const int i = p / m, j = p - i * m;
    if (i >= j) continue;
    const float* x = s_acr + i * dim;
    const float* y = s_acr + j * dim;
    double dot = 0.0;
    for (int k = 0; k < dim; ++k) dot = fma((double)x[k], (double)y[k], dot);
    const double nn = a.acr_norm[s_id[i]] * a.acr_norm[s_id[j]];
    const double cs = nn > 0.0 ? dot / nn : 0.0;
    const double d = fmin(fmax(1.0 - cs, 0.0), 2.0) * 0.5;
    s_D[i * m + j] = d;
    s_D[j * m + i] = d;
  }
  __syncthreads();
  // inner (per list position i < m - 1) averages of the two EILD variants
  if (threadIdx.x < m - 1) {
    const int i = threadIdx.x;
    double num = 0.0, den = 0.0, num_rr = 0.0, den_rr = 0.0;
    for (int j = 0; j < m; ++j) {
      if (j == i) continue;
      const double w = disc(j - i - 1 > 0 ? j - i - 1 : 0);
      num += s_D[i * m + j] * w;
      den += w;
      if (j > i) {
        const double rj = s_id[j] == label ? 1.0 : a.neg_rel;
        num_rr += s_D[i * m + j] * w * rj;
        den_rr += w * rj;
      }
    }
    s_er[i] = num / den;
    s_err[i] = num_rr / den_rr;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double dcg = 0.0, idcg = 0.0;
  const int ideal = s_occ < m ? s_occ : m;
  for (int i = 0; i < m; ++i) {
    if (s_id[i] == label) dcg += disc(i);
    if (i < ideal) idcg += disc(i);
  }
  double w = 0.0, esi = 0.0, esi_rr = 0.0, eild = 0.0, eild_rr = 0.0;
  for (int i = 0; i < m - 1; ++i) {                  // the reference's range(0, len - 1): the last item never counts
    const double di = disc(i);
    const double ri = s_id[i] == label ? 1.0 : a.neg_rel;
    const double nov = -log2((double)a.pop[s_id[i]]) * di;
    esi += nov;
    esi_rr += nov * ri;
    eild += s_er[i] * di;
    eild_rr += s_err[i] * di * ri;
    w += di;
  }
  out[0] = idcg > 0.0 ? dcg / idcg : 0.0;
  out[1] = esi / w;
  out[2] = esi_rr / w;
  out[3] = eild / w;
  out[4] = eild_rr / w;
  out[5] = 1.0;
}

// acc[row, c] += sum over q of per_query[row, q, c]: per-thread strided partial sums, then a shared-memory tree, both in
// a fixed order.  One CTA per row.
__global__ void __launch_bounds__(REDUCE_THREADS) reduce_kernel(const double* per_query, int64_t nq, long long row_mask,
                                                                double* acc) {
  __shared__ double s[N_VALUES][REDUCE_THREADS];
  const int row = blockIdx.x;
  if (!((row_mask >> row) & 1)) return;
  const double* src = per_query + (int64_t)row * nq * N_VALUES;
  double part[N_VALUES] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t q = threadIdx.x; q < nq; q += REDUCE_THREADS)
#pragma unroll
    for (int c = 0; c < N_VALUES; ++c) part[c] += src[q * N_VALUES + c];
#pragma unroll
  for (int c = 0; c < N_VALUES; ++c) s[c][threadIdx.x] = part[c];
  __syncthreads();
  for (int h = REDUCE_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h)
#pragma unroll
      for (int c = 0; c < N_VALUES; ++c) s[c][threadIdx.x] += s[c][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < N_VALUES) acc[row * N_VALUES + threadIdx.x] += s[threadIdx.x][0];
}

// counts[i] = set bits of bitmap i (one CTA per bitmap)
__global__ void popcount_kernel(const unsigned* bitmaps, int64_t words, unsigned long long* counts) {
  __shared__ unsigned long long s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const unsigned* b = bitmaps + blockIdx.x * words;
  unsigned long long n = 0;
  for (int64_t w = threadIdx.x; w < words; w += blockDim.x) n += __popc(b[w]);
  atomicAdd(&s_n, n);
  __syncthreads();
  if (threadIdx.x == 0) counts[blockIdx.x] = s_n;
}

// ---- hit rate by session position (the reference's HitRateBySessionPosition, metrics.py:136-168; spec
// oracle/by_position_ref.py).  Rows y < rows: a grid-stride loop over the queries of recommender row y builds per-CTA
// position histograms in shared memory and adds them to hits / total with integer atomics (exact in any order).  Row
// y == rows (only when pop is given, one CTA): chunk by chunk of sessions, the CTA gathers pop[label] of every (session,
// position) cell into shared memory in parallel, then one thread per position t adds the chunk's values for b in order
// - a sequential float32 sum with no FMA, carried in norm_pop from batch to batch: the reference's own order.
constexpr int POS_THREADS = 256;
constexpr int MAX_POS = 1024;              // positions T per batch (shared-memory histograms)
constexpr int POP_CHUNK = 4096;            // (session, position) cells gathered per round
constexpr int GATHER_UNROLL = 8;           // cells whose loads one thread has in flight at once

struct PosArgs {
  const int64_t* ids; int64_t row_stride, q_stride, nq; int m; long long row_mask; int rows;
  const int64_t* labels; int64_t label_stride;
  const int32_t* pos_idx; int T;           // pos_idx null: query q sits at position q % T
  const int32_t* sess_off; int64_t n_sess; const float* pop;
  int64_t num_items;
  unsigned long long* hits; unsigned long long* total; int64_t ld;   // [rows, ld]
  float* norm_pop;                         // [T]
  int* err;
};

__device__ void norm_pop_pass(const PosArgs& a) {
  __shared__ float s_v[POP_CHUNK];
  constexpr int PER = MAX_POS / POS_THREADS;
  const int T = a.T, per_chunk = POP_CHUNK / T;
  float sum[PER];
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int t = threadIdx.x + k * POS_THREADS;
    sum[k] = t < T ? a.norm_pop[t] : 0.f;
  }
  bool bad = false;
  for (int64_t b0 = 0; b0 < a.n_sess; b0 += per_chunk) {
    const int nb = (int)(a.n_sess - b0 < per_chunk ? a.n_sess - b0 : per_chunk), n = nb * T;
    // three rounds of independent loads (offsets, labels, pop) over GATHER_UNROLL cells per thread
    for (int i0 = threadIdx.x; i0 < n; i0 += POS_THREADS * GATHER_UNROLL) {
      int32_t off[GATHER_UNROLL], end[GATHER_UNROLL];
      int tt[GATHER_UNROLL];
#pragma unroll
      for (int u = 0; u < GATHER_UNROLL; ++u) {
        const int i = i0 + u * POS_THREADS;
        const int64_t b = i < n ? b0 + i / T : a.n_sess;     // past the chunk: an empty session
        tt[u] = i % T;
        off[u] = a.sess_off[b];
        end[u] = a.sess_off[b < a.n_sess ? b + 1 : b];
      }
      int64_t label[GATHER_UNROLL];
#pragma unroll
      for (int u = 0; u < GATHER_UNROLL; ++u)
        label[u] = tt[u] < end[u] - off[u] ? a.labels[(int64_t)(off[u] + tt[u]) * a.label_stride] : 0;
#pragma unroll
      for (int u = 0; u < GATHER_UNROLL; ++u) {
        const bool ok = label[u] > 0 && label[u] < a.num_items;
        bad |= label[u] != 0 && !ok;
        const int i = i0 + u * POS_THREADS;
        const float v = ok ? a.pop[label[u]] : 0.f;
        if (i < n) s_v[i] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int t = threadIdx.x + k * POS_THREADS;
      if (t < T)
        for (int b = 0; b < nb; ++b) sum[k] = __fadd_rn(sum[k], s_v[b * T + t]);   // s + 0 == s (s is never -0)
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int t = threadIdx.x + k * POS_THREADS;
    if (t < T) a.norm_pop[t] = sum[k];
  }
  if (bad) atomicExch(a.err, 1);
}

__global__ void __launch_bounds__(POS_THREADS) by_position_kernel(PosArgs a) {
  const int row = blockIdx.y;
  if (row == a.rows) {                     // the model's label popularity per position
    if (blockIdx.x == 0) norm_pop_pass(a);
    return;
  }
  if (!((a.row_mask >> row) & 1)) return;
  __shared__ unsigned s_hit[MAX_POS], s_tot[MAX_POS];
  for (int t = threadIdx.x; t < a.T; t += POS_THREADS) { s_hit[t] = 0; s_tot[t] = 0; }
  __syncthreads();
  const int64_t* lists = a.ids + row * a.row_stride;
  for (int64_t q = blockIdx.x * (int64_t)POS_THREADS + threadIdx.x; q < a.nq; q += (int64_t)gridDim.x * POS_THREADS) {
    const int64_t label = a.labels[q * a.label_stride];
    if (label == 0) continue;
    bool bad = label < 0 || label >= a.num_items, hit = false;
    const int64_t* list = lists + q * a.q_stride;
    for (int j = 0; j < a.m; ++j) {
      const int64_t id = list[j];
      hit |= id == label;
      bad |= id < 0 || id >= a.num_items;
    }
    if (bad) { atomicExch(a.err, 1); continue; }
    const int t = (int)((a.pos_idx ? (int64_t)a.pos_idx[q] : q) % a.T);
    atomicAdd(&s_tot[t], 1u);
    if (hit) atomicAdd(&s_hit[t], 1u);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < a.T; t += POS_THREADS) {
    if (s_tot[t]) atomicAdd(a.total + row * a.ld + t, (unsigned long long)s_tot[t]);
    if (s_hit[t]) atomicAdd(a.hits + row * a.ld + t, (unsigned long long)s_hit[t]);
  }
}

static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  return (int)(g < 1 ? 1 : (g > 8 * NAR_GRID_SMS ? 8 * NAR_GRID_SMS : g));
}

}  // namespace em
}  // namespace nar

using namespace nar::em;

extern "C" int nar_eval_metrics_mark(const int64_t* ids, int64_t n, int64_t num_items, int32_t skip_zero, uint32_t* bitmap,
                                     int* err, void* stream) {
  if ((!ids && n > 0) || !bitmap || !err || n < 0 || num_items <= 0) return NAR_ERR_INVALID;
  if (n == 0) return NAR_OK;
  mark_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(ids, n, num_items, skip_zero, bitmap, err);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_eval_metrics_lists(const int64_t* ids, int64_t row_stride, int64_t q_stride, int64_t rows, int64_t row_mask,
                                      int64_t nq, int64_t len, int32_t top_n, const int64_t* labels, int64_t label_stride,
                                      const float* pop, const float* acr, int64_t acr_dim, int64_t acr_ld,
                                      const double* acr_norm, int64_t num_items, double neg_relevance, double* per_query,
                                      uint32_t* rec_bitmaps, int* err, void* stream) {
  if (!ids || !labels || !pop || !acr || !acr_norm || !per_query || !rec_bitmaps || !err || rows < 1 || rows > 63 ||
      nq < 0 || len < 1 || q_stride < len || label_stride < 1 || acr_dim <= 0 || acr_ld < acr_dim || num_items <= 0 ||
      !(neg_relevance > 0.0))
    return NAR_ERR_INVALID;
  const int64_t m = top_n < len ? top_n : len;
  if (m < 2) return NAR_ERR_INVALID;                      // the reference divides by an empty sum below two items
  if (m > MAX_M || nq > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  const size_t smem = sizeof(double) * m * m + sizeof(float) * m * acr_dim;
  if (smem > MAX_LIST_SMEM) return NAR_ERR_UNSUPPORTED;
  if (nq == 0 || (row_mask & ((1LL << rows) - 1)) == 0) return NAR_OK;
  // the kernel's static arrays count against the 48 KB a launch gets without opting in, so a dynamic size just below
  // 48 KB needs the attribute too: raise it once to the cap
  static bool attr = false;
  if (!attr) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(list_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MAX_LIST_SMEM));
    attr = true;
  }
  ListArgs a;
  a.ids = ids; a.row_stride = row_stride; a.q_stride = q_stride; a.nq = nq; a.len = len; a.m = (int)m;
  a.labels = labels; a.label_stride = label_stride;
  a.pop = pop; a.acr = acr; a.acr_dim = acr_dim; a.acr_ld = acr_ld; a.acr_norm = acr_norm; a.num_items = num_items;
  a.neg_rel = neg_relevance; a.row_mask = row_mask & ((1LL << rows) - 1);
  a.per_query = per_query; a.rec = rec_bitmaps; a.words = (num_items + 31) / 32; a.err = err;
  list_kernel<<<dim3((unsigned)nq, (unsigned)rows), LIST_THREADS, smem, as_stream(stream)>>>(a);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_eval_metrics_reduce(const double* per_query, int64_t rows, int64_t row_mask, int64_t nq, double* acc,
                                       void* stream) {
  if (!per_query || !acc || rows < 1 || rows > 63 || nq < 0) return NAR_ERR_INVALID;
  if (nq == 0) return NAR_OK;
  reduce_kernel<<<(unsigned)rows, REDUCE_THREADS, 0, as_stream(stream)>>>(per_query, nq, row_mask, acc);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_eval_by_position(const int64_t* ids, int64_t row_stride, int64_t q_stride, int64_t rows, int64_t row_mask,
                                    int64_t nq, int64_t len, int32_t top_n, const int64_t* labels, int64_t label_stride,
                                    const int32_t* pos_idx, int64_t T, const int32_t* sess_off, int64_t n_sess,
                                    const float* pop, int64_t num_items, int64_t* hits, int64_t* total, int64_t ld,
                                    float* norm_pop, int* err, void* stream) {
  if (!ids || !labels || !hits || !total || !err || rows < 1 || rows > 63 || nq < 0 || len < 1 || q_stride < len ||
      label_stride < 1 || top_n < 1 || T < 1 || ld < T || num_items <= 0 || (nq > 0 && !pos_idx && nq % T) ||
      (pop && (!pos_idx || !sess_off || !norm_pop || n_sess < 0)))
    return NAR_ERR_INVALID;
  if (T > MAX_POS || nq > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  const long long mask = row_mask & ((1LL << rows) - 1);
  if (nq == 0 || (mask == 0 && !pop)) return NAR_OK;
  PosArgs a;
  a.ids = ids; a.row_stride = row_stride; a.q_stride = q_stride; a.nq = nq; a.m = (int)(top_n < len ? top_n : len);
  a.row_mask = mask; a.rows = (int)rows;
  a.labels = labels; a.label_stride = label_stride; a.pos_idx = pos_idx; a.T = (int)T;
  a.sess_off = sess_off; a.n_sess = n_sess; a.pop = pop; a.num_items = num_items;
  a.hits = reinterpret_cast<unsigned long long*>(hits); a.total = reinterpret_cast<unsigned long long*>(total); a.ld = ld;
  a.norm_pop = norm_pop; a.err = err;
  const dim3 grid((unsigned)grid_for(nq, POS_THREADS), (unsigned)(rows + (pop ? 1 : 0)));
  by_position_kernel<<<grid, POS_THREADS, 0, as_stream(stream)>>>(a);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_eval_metrics_popcount(const uint32_t* bitmaps, int64_t n_maps, int64_t words, int64_t* counts,
                                         void* stream) {
  if (!bitmaps || !counts || n_maps < 1 || n_maps > 0x7fffffffLL || words < 1) return NAR_ERR_INVALID;
  popcount_kernel<<<(unsigned)n_maps, 256, 0, as_stream(stream)>>>(bitmaps, words,
                                                                  reinterpret_cast<unsigned long long*>(counts));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
