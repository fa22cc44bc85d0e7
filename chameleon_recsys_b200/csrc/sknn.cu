// Session-based kNN baseline of the evaluation hook (the reference's benchmarks/session_knn.py: V-SkNN with the 'div'
// decay, SkNN with 'same'), driven like the other baselines (nar_model.py:1609-1632).  Spec: oracle/sknn_ref.py.
//
// State: a ring of S slots holding the last S sessions in insertion order (logical index 0 = oldest; head and count are
// tracked by the caller, which knows them from the batch sizes).  Slot: session id (int64), length, and up to W item ids
// (int32, sorted ascending, deduplicated).  An item is stored as +x while (x, id) is in the reference's item -> sessions
// map ("live") and as -x once an eviction has discarded that pair; the similarity always uses |x| (the full set).
// Update, per batch: stage the new entries (sorted sets), evict the oldest max(0, count + B - S) entries (clearing the
// live bits of their items in every surviving slot, staged ones included, with the same session id: the reference's
// discard also drops the pair of a newer entry with that id), then copy the staged entries into their slots.
// Score, one CTA per query: candidates with multiplicity from the live sets and the reference's binary search over the
// ring in insertion order, the 'recent' cut, fp64 similarities in the reference's association, the neighbour cut, item
// scores of the query's own candidates summed copy by copy, exact ranking and an integer rank histogram.
#include "common.cuh"

namespace nar {
namespace sknn {

constexpr int MAX_W = 128;                 // slot width bound (the staging CTA holds one row)
constexpr int MAX_T = 64;                  // positions of the active session: one uint64 mask bit each
constexpr int MAX_SESSIONS = 4096;         // ring slots the score kernel's shared memory holds
constexpr int MAX_CAND = 1024;             // 1 + K candidates of one query
constexpr int ST = 512;                    // score kernel threads
constexpr int NW = ST / 32;
constexpr uint16_t NONE = 0xFFFF;

__global__ void __launch_bounds__(MAX_W) stage_kernel(const int64_t* all_items, int64_t T1, const int64_t* sids,
                                                      int64_t num_items, int64_t* st_ids, int* st_lens, int* st_items,
                                                      int W, int* err) {
  __shared__ int64_t s_x[MAX_W];
  __shared__ int s_first[MAX_W];
  const int64_t b = blockIdx.x;
  const int p = threadIdx.x;
  int64_t x = 0;
  if (p < T1) {
    x = all_items[b * T1 + p];
    if (x < 0 || x >= num_items) { atomicExch(err, 1); x = 0; }
    s_x[p] = x;
  }
  __syncthreads();
  int first = 0;
  if (p < T1 && x != 0) {
    first = 1;
    for (int q = 0; q < p; ++q) first &= (s_x[q] != x);
  }
  s_first[p] = first;
  __syncthreads();
  if (first) {
    int rank = 0;
    for (int q = 0; q < T1; ++q) rank += s_first[q] && s_x[q] < x;
    st_items[b * W + rank] = (int)x;
  }
  const int n = __syncthreads_count(first);
  if (p == 0) { st_lens[b] = n; st_ids[b] = sids[b]; }
}

__device__ __forceinline__ bool contains(const int* set, int n, int x) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (set[mid] < x) lo = mid + 1; else hi = mid; }
  return lo < n && set[lo] == x;
}

// one CTA per evicted entry e (logical e < E): survivors are the old entries E..count-1 and the staged ones
__global__ void evict_kernel(const int64_t* ids, const int* lens, int* items, int64_t S, int W, int64_t head,
                             int64_t count, int64_t E, const int64_t* st_ids, const int* st_lens, int* st_items,
                             int64_t B) {
  __shared__ int s_set[MAX_W];
  __shared__ int s_n;
  __shared__ int64_t s_id;
  const int64_t ph = (head + blockIdx.x) % S;
  if (threadIdx.x == 0) { s_n = lens[ph]; s_id = ids[ph]; }
  __syncthreads();
  for (int k = threadIdx.x; k < s_n; k += blockDim.x) s_set[k] = abs(items[ph * W + k]);
  __syncthreads();
  const int64_t old = count - E;
  for (int64_t i = threadIdx.x; i < old + B; i += blockDim.x) {
    int* row; int L;
    if (i < old) {
      const int64_t p = (head + E + i) % S;
      if (ids[p] != s_id) continue;
      row = items + p * W; L = lens[p];
    } else {
      const int64_t b = i - old;
      if (st_ids[b] != s_id) continue;
      row = st_items + b * W; L = st_lens[b];
    }
    for (int k = 0; k < L; ++k) {
      const int x = row[k];
      if (x > 0 && contains(s_set, s_n, x)) row[k] = -x;     // every writer stores the same value
    }
  }
}

__global__ void copy_kernel(int64_t* ids, int* lens, int* items, int64_t S, int W, int64_t head, int64_t count,
                            const int64_t* st_ids, const int* st_lens, const int* st_items) {
  const int64_t b = blockIdx.x;
  const int64_t ph = (head + count + b) % S;
  const int L = st_lens[b];
  for (int k = threadIdx.x; k < W; k += blockDim.x) items[ph * W + k] = k < L ? st_items[b * W + k] : 0;
  if (threadIdx.x == 0) { ids[ph] = st_ids[b]; lens[ph] = L; }
}

struct ScoreArgs {
  const int64_t* ids; const int* lens; const int* items; int64_t S; int W; int64_t head, count;
  const int64_t *item_clicked, *label_next, *negatives; int64_t B, T, K, num_items;
  int64_t sample_size, nn; int decay_div, jaccard, top_n;
  unsigned long long* rank_hist;   // [top_n + 1]: queries whose label ranked r (< top_n), and all queries
  int64_t* out_ids;                // [B*T, top_n] or null
  int* err;
};

template <typename V>
__device__ __forceinline__ int find_sorted(const V* arr, int n, int64_t x) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if ((int64_t)arr[mid] < x) lo = mid + 1; else hi = mid; }
  return (lo < n && (int64_t)arr[lo] == x) ? lo : -1;
}

// neighbour order: higher similarity, then higher session id; NONE pads the sort
__device__ __forceinline__ bool nb_before(const double* sim, const int64_t* cid, uint16_t x, uint16_t y) {
  if (x == NONE) return false;
  if (y == NONE) return true;
  const double sx = sim[x], sy = sim[y];
  if (sx != sy) return sx > sy;
  return cid[x] > cid[y];
}

// perm[0..n) = 0..n-1 sorted by nb_before (bitonic, keys unique: session ids are distinct among the candidates)
__device__ void sort_perm(uint16_t* perm, int n, const double* sim, const int64_t* cid) {
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int i = threadIdx.x; i < n2; i += ST) perm[i] = i < n ? (uint16_t)i : NONE;
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += ST) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint16_t x = perm[i], y = perm[ixj];
          if ((i & k) == 0 ? nb_before(sim, cid, y, x) : nb_before(sim, cid, x, y)) { perm[i] = y; perm[ixj] = x; }
        }
      }
      __syncthreads();
    }
}

// in perm order over the first n entries: cnt[k] = number of its copies among the first `limit` copies
__device__ void keep_prefix(const uint16_t* perm, uint16_t* cnt, int n, int64_t limit, int* s_warp) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (n + ST - 1) / ST;
  const int beg = min(tid * per, n), end = min(beg + per, n);
  int local = 0;
  for (int r = beg; r < end; ++r) local += cnt[perm[r]];
  int v = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  if (lane == 31) s_warp[wid] = v;
  __syncthreads();
  int64_t excl = v - local;
  for (int w = 0; w < wid; ++w) excl += s_warp[w];
  for (int r = beg; r < end; ++r) {
    const int k = perm[r], c = cnt[k];
    const int64_t keep = limit - excl;
    cnt[k] = (uint16_t)(keep < 0 ? 0 : (keep > c ? c : keep));
    excl += c;
  }
  __syncthreads();
}

// dynamic shared memory for `count` ring entries
static inline size_t score_smem(int64_t count) {
  const int64_t sc = count > 0 ? count : 1;
  int64_t n2 = 1;
  while (n2 < sc) n2 <<= 1;
  return (size_t)(28 * sc + 2 * n2);
}

// one CTA per query (b, t) with label != 0
__global__ void __launch_bounds__(ST) score_kernel(ScoreArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int n = (int)a.count;
  const int sc = n > 0 ? n : 1;
  unsigned long long* s_acc = reinterpret_cast<unsigned long long*>(smem);  // position masks; later neighbour masks
  int64_t* s_cid = reinterpret_cast<int64_t*>(smem + 8 * (size_t)sc);       // candidate session ids
  double* s_sim = reinterpret_cast<double*>(smem + 16 * (size_t)sc);        // similarities; ring ids during the scan
  uint16_t* s_slot = reinterpret_cast<uint16_t*>(smem + 24 * (size_t)sc);   // candidate -> logical slot
  uint16_t* s_cnt = s_slot + sc;                                             // candidate -> copies
  uint16_t* s_perm = s_cnt + sc;
  __shared__ int64_t s_P[MAX_T], s_pd[MAX_T];
  __shared__ unsigned long long s_pdm[MAX_T];      // distinct item of P -> positions holding it
  __shared__ int s_pfirst[MAX_T];
  __shared__ int s_q[MAX_CAND], s_qf[MAX_CAND], s_qfirst[MAX_CAND];
  __shared__ double s_qs[MAX_CAND];
  __shared__ int s_warp[NW];
  __shared__ int s_n, s_total, s_kept, s_nb;
  const int tid = threadIdx.x;
  const int64_t q = blockIdx.x;
  const int64_t label = a.label_next[q];
  if (label == 0) return;                                            // block-uniform
  const int64_t b = q / a.T, t = q % a.T;
  const int np = (int)t + 1;
  {
    const int64_t item = a.item_clicked[q];
    if (item <= 0 || item >= a.num_items || label < 0 || label >= a.num_items) {
      if (tid == 0) atomicExch(a.err, 1);
      return;
    }
  }
  // ---- the active session P = item_clicked[b, :t+1]: distinct items (sorted) with their position masks
  if (tid < np) {
    int64_t x = a.item_clicked[b * a.T + tid];
    if (x < 0 || x >= a.num_items) { atomicExch(a.err, 1); x = 0; }
    s_P[tid] = x;
  }
  // ---- the query's candidates: label + K negatives, distinct nonzero ids, sorted
  const int nc = (int)a.K + 1;
  for (int j = tid; j < nc; j += ST) {
    int64_t id = j == 0 ? label : a.negatives[q * a.K + (j - 1)];
    if (id < 0 || id >= a.num_items) { atomicExch(a.err, 1); id = 0; }
    s_qf[j] = (int)id;
  }
  if (tid == 0) { s_n = 0; s_total = 0; s_kept = 0; s_nb = 0; }
  __syncthreads();
  if (tid < np) {
    int first = 1;
    for (int p = 0; p < tid; ++p) first &= s_P[p] != s_P[tid];
    s_pfirst[tid] = first;
  }
  for (int j = tid; j < nc; j += ST) {
    const int x = s_qf[j];
    int first = x != 0;
    for (int k = 0; k < j && first; ++k) first = s_qf[k] != x;
    s_qfirst[j] = first;
  }
  __syncthreads();
  if (tid < np && s_pfirst[tid]) {
    const int64_t x = s_P[tid];
    int rank = 0;
    unsigned long long m = 0;
    for (int p = 0; p < np; ++p) {
      rank += s_pfirst[p] && s_P[p] < x;
      if (s_P[p] == x) m |= 1ull << p;
    }
    s_pd[rank] = x; s_pdm[rank] = m;
  }
  for (int j = tid; j < nc; j += ST) {
    if (!s_qfirst[j]) continue;
    const int x = s_qf[j];
    int rank = 0;
    for (int k = 0; k < nc; ++k) rank += s_qfirst[k] && s_qf[k] < x;
    s_q[rank] = x;
  }
  int nP = 0, nq = 0;
  for (int p = 0; p < np; ++p) nP += s_pfirst[p];
  for (int j = 0; j < nc; ++j) nq += s_qfirst[j];
  // ---- scan the ring: positions of P whose item is live in the slot, OR-ed into the slot the binary search finds
  int64_t* s_idc = reinterpret_cast<int64_t*>(s_sim);
  for (int i = tid; i < n; i += ST) { s_idc[i] = a.ids[(a.head + i) % a.S]; s_acc[i] = 0; }
  __syncthreads();
  for (int i = tid; i < n; i += ST) {
    const int64_t ph = (a.head + i) % a.S;
    const int L = a.lens[ph];
    const int* row = a.items + ph * a.W;
    unsigned long long m = 0;
    for (int k = 0; k < L; ++k) {
      const int x = row[k];
      if (x > 0) { const int d = find_sorted(s_pd, nP, x); if (d >= 0) m |= s_pdm[d]; }
    }
    if (m) {
      const int64_t sid = s_idc[i];
      int lo = 0, hi = n;                                            // find_session_on_buffer
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (sid > s_idc[mid]) lo = mid + 1; else hi = mid; }
      if (lo != n && s_idc[lo] == sid) atomicOr(s_acc + lo, m);
    }
  }
  __syncthreads();
  for (int j = tid; j < n; j += ST) {
    const unsigned long long m = s_acc[j];
    if (!m) continue;
    const int k = atomicAdd(&s_n, 1), c = __popcll(m);
    s_slot[k] = (uint16_t)j; s_cnt[k] = (uint16_t)c; s_cid[k] = s_idc[j];
    atomicAdd(&s_total, c);
  }
  __syncthreads();
  const int ncand = s_n;
  // ---- 'recent' cut: the sample_size copies of the highest session ids
  if (a.sample_size > 0 && s_total > a.sample_size) {
    for (int k = tid; k < ncand; k += ST) s_sim[k] = 0.0;
    __syncthreads();
    sort_perm(s_perm, ncand, s_sim, s_cid);
    keep_prefix(s_perm, s_cnt, ncand, a.sample_size, s_warp);
  }
  // ---- similarities against the full set of the slot, in the reference's fp64 association; kept: 0 < sim < 1
  for (int k = tid; k < ncand; k += ST) {
    double sim = -1.0;
    if (s_cnt[k] > 0) {
      const int64_t ph = (a.head + s_slot[k]) % a.S;
      const int L = a.lens[ph];
      const int* row = a.items + ph * a.W;
      unsigned long long dm = 0, pm = 0;
      for (int kk = 0; kk < L; ++kk) {
        const int d = find_sorted(s_pd, nP, abs(row[kk]));
        if (d >= 0) { dm |= 1ull << d; pm |= s_pdm[d]; }
      }
      const int inter = __popcll(dm);
      double num;
      if (a.decay_div) {
        num = 0.0;
        for (int pos = 1; pos <= np; ++pos)
          if ((pm >> (np - pos)) & 1ull) num = __dadd_rn(num, __ddiv_rn(1.0, (double)pos));
      } else {
        num = (double)inter;
      }
      const double den = a.jaccard ? (double)(nP + L - inter) : __dmul_rn(__dsqrt_rn((double)nP), __dsqrt_rn((double)L));
      const double v = __ddiv_rn(num, den);
      if (v > 0.0 && v < 1.0) { sim = v; atomicAdd(&s_kept, 1); }
    }
    s_sim[k] = sim;
  }
  __syncthreads();
  const int kept = s_kept;
  sort_perm(s_perm, ncand, s_sim, s_cid);                            // kept candidates first
  keep_prefix(s_perm, s_cnt, kept, a.nn, s_warp);
  for (int r = tid; r < kept; r += ST)
    if (s_cnt[s_perm[r]] > 0) atomicAdd(&s_nb, 1);
  __syncthreads();
  const int nb = s_nb;                                               // the kept neighbours: a prefix of perm
  // ---- item scores of the query's candidates, 64 at a time: neighbour masks, then sums copy by copy in order
  for (int c0 = 0; c0 < nq; c0 += 64) {
    const int cn = min(64, nq - c0);
    for (int r = tid; r < nb; r += ST) {
      const int64_t ph = (a.head + s_slot[s_perm[r]]) % a.S;
      const int L = a.lens[ph];
      const int* row = a.items + ph * a.W;
      unsigned long long m = 0;
      for (int kk = 0; kk < L; ++kk) {
        const int d = find_sorted(s_q + c0, cn, abs(row[kk]));
        if (d >= 0) m |= 1ull << d;
      }
      s_acc[r] = m;
    }
    __syncthreads();
    if (tid < cn) {
      double sc_ = 0.0;
      int first = -1;
      for (int r = 0; r < nb; ++r) {
        if (!((s_acc[r] >> tid) & 1ull)) continue;
        if (first < 0) first = r;
        const int k = s_perm[r];
        const double v = s_sim[k];
        for (int c = 0; c < s_cnt[k]; ++c) sc_ = __dadd_rn(sc_, v);
      }
      s_qs[c0 + tid] = sc_; s_qf[c0 + tid] = first;
    }
    __syncthreads();
  }
  // ---- rank: score desc, first neighbour asc, id asc; only items some kept neighbour holds
  int64_t* out = a.out_ids ? a.out_ids + q * a.top_n : nullptr;
  if (out) for (int r = tid; r < a.top_n; r += ST) out[r] = 0;
  __syncthreads();
  for (int c = tid; c < nq; c += ST) {
    if (s_qf[c] < 0) continue;
    const double sc_ = s_qs[c];
    const int f = s_qf[c], id = s_q[c];
    int rank = 0;
    for (int o = 0; o < nq; ++o) {
      if (o == c || s_qf[o] < 0) continue;
      const double so = s_qs[o];
      rank += so > sc_ || (so == sc_ && (s_qf[o] < f || (s_qf[o] == f && s_q[o] < id)));
    }
    if (rank < a.top_n) {
      if (out) out[rank] = id;
      if (id == label) atomicAdd(a.rank_hist + rank, 1ull);
    }
  }
  if (tid == 0) atomicAdd(a.rank_hist + a.top_n, 1ull);
}

// metrics += {hits, sum of reciprocal ranks, queries}, summed over the rank histogram in a fixed order
__global__ void finalize_kernel(const unsigned long long* h, int top_n, double* metrics) {
  unsigned long long hits = 0; double rr = 0.0;
  for (int r = 0; r < top_n; ++r) { hits += h[r]; rr += (double)h[r] / (double)(r + 1); }
  metrics[0] += (double)hits;
  metrics[1] += rr;
  metrics[2] += (double)h[top_n];
}

}  // namespace sknn
}  // namespace nar

using namespace nar::sknn;

extern "C" int nar_sknn_update(int64_t* ids, int32_t* lens, int32_t* items, int64_t S, int64_t W, int64_t head,
                               int64_t count, int64_t* st_ids, int32_t* st_lens, int32_t* st_items,
                               const int64_t* all_items, const int64_t* session_ids, int64_t B, int64_t T1,
                               int64_t num_items, int* err, void* stream) {
  if (!ids || !lens || !items || !st_ids || !st_lens || !st_items || !err || S <= 0 || W <= 0 || W > MAX_W || head < 0 ||
      head >= S || count < 0 || count > S || B < 0 || T1 <= 0 || num_items <= 0 || num_items > 0x7fffffffLL)
    return NAR_ERR_INVALID;
  if (B > S || T1 > W) return NAR_ERR_INVALID;
  if (B == 0) return NAR_OK;
  if (!all_items || !session_ids) return NAR_ERR_INVALID;
  cudaStream_t s = as_stream(stream);
  stage_kernel<<<(unsigned)B, MAX_W, 0, s>>>(all_items, T1, session_ids, num_items, st_ids, st_lens, st_items, (int)W, err);
  NAR_LAUNCH_CHECK();
  const int64_t E = count + B - S > 0 ? count + B - S : 0;
  if (E > 0) {
    evict_kernel<<<(unsigned)E, 256, 0, s>>>(ids, lens, items, S, (int)W, head, count, E, st_ids, st_lens, st_items, B);
    NAR_LAUNCH_CHECK();
  }
  copy_kernel<<<(unsigned)B, MAX_W, 0, s>>>(ids, lens, items, S, (int)W, head, count, st_ids, st_lens, st_items);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_sknn_score(const int64_t* ids, const int32_t* lens, const int32_t* items, int64_t S, int64_t W,
                              int64_t head, int64_t count, const int64_t* item_clicked, const int64_t* label_next,
                              const int64_t* negatives, int64_t B, int64_t T, int64_t K, int64_t num_items,
                              int64_t sample_size, int64_t nn, int32_t decay_div, int32_t jaccard, int32_t top_n,
                              int64_t* rank_hist, double* metrics, int64_t* out_ids, int* err, void* stream) {
  if (!ids || !lens || !items || !item_clicked || !label_next || (!negatives && K > 0) || !rank_hist || !metrics || !err ||
      S <= 0 || W <= 0 || head < 0 || head >= S || count < 0 || count > S || B < 0 || T <= 0 || K < 0 || top_n < 1 ||
      num_items <= 0 || num_items > 0x7fffffffLL || sample_size < 0 || nn < 0)
    return NAR_ERR_INVALID;
  if (S > MAX_SESSIONS || T > MAX_T || K + 1 > MAX_CAND) return NAR_ERR_UNSUPPORTED;
  cudaStream_t s = as_stream(stream);
  static bool attr = false;
  if (!attr) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)score_smem(MAX_SESSIONS)));
    attr = true;
  }
  NAR_CHECK_CUDA(cudaMemsetAsync(rank_hist, 0, sizeof(int64_t) * (top_n + 1), s));
  ScoreArgs a;
  a.ids = ids; a.lens = lens; a.items = items; a.S = S; a.W = (int)W; a.head = head; a.count = count;
  a.item_clicked = item_clicked; a.label_next = label_next; a.negatives = negatives; a.B = B; a.T = T; a.K = K;
  a.num_items = num_items; a.sample_size = sample_size; a.nn = nn; a.decay_div = decay_div; a.jaccard = jaccard;
  a.top_n = top_n; a.rank_hist = reinterpret_cast<unsigned long long*>(rank_hist); a.out_ids = out_ids; a.err = err;
  if (B * T > 0) {
    score_kernel<<<(unsigned)(B * T), ST, score_smem(count), s>>>(a);
    NAR_LAUNCH_CHECK();
  }
  finalize_kernel<<<1, 1, 0, s>>>(a.rank_hist, top_n, metrics);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
