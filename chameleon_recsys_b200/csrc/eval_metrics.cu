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
  if (smem > 200 * 1024) return NAR_ERR_UNSUPPORTED;
  if (nq == 0 || (row_mask & ((1LL << rows) - 1)) == 0) return NAR_OK;
  if (smem > 48 * 1024)
    NAR_CHECK_CUDA(cudaFuncSetAttribute(list_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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

extern "C" int nar_eval_metrics_popcount(const uint32_t* bitmaps, int64_t n_maps, int64_t words, int64_t* counts,
                                         void* stream) {
  if (!bitmaps || !counts || n_maps < 1 || n_maps > 0x7fffffffLL || words < 1) return NAR_ERR_INVALID;
  popcount_kernel<<<(unsigned)n_maps, 256, 0, as_stream(stream)>>>(bitmaps, words,
                                                                  reinterpret_cast<unsigned long long*>(counts));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
