// Baseline recommenders of the evaluation hook (nar_model.py:1399-1407, 1609-1632 of the reference): the pair table
// shared by the co-occurrence, item-kNN and sequential-rules baselines, the recent-clicks histogram of the popularity
// baseline, and one scoring + ranking + metrics kernel for all five baselines.  Spec: oracle/baselines_ref.py.
//
// Pair table: open addressing with linear probing in HBM, capacity a power of two.  Key (a << 32) | c of the ordered
// pair (a = current click, c = candidate), -1 = empty slot.  Values (structure of arrays, int64):
//   cooc     sessions in which a and c occur at two different positions (each distinct ordered pair once per session)
//   sr_w     sequential-rules weight in units of 1 / lcm(1..max_clicks_dist): a 'div' decay 1/d is lcm/d units, exact
//   sr_first first insertion key of the rule a -> c: min over its occurrences of (batch_seq << 32) | ordinal, the ordinal
//            running over (session, i, j) in the reference's loop order
// Integer atomics only: the table contents do not depend on thread scheduling (slot placement does; exports sort).
#include "common.cuh"
#include "select_topn.cuh"

namespace nar {
namespace bl {

constexpr unsigned long long EMPTY = ~0ull;
constexpr int UPDATE_THREADS = 256;
constexpr int MAX_SESSION = 1024;          // clicks of one session the update kernel holds in shared memory
constexpr int MAX_CAND = 1024;             // 1 + K candidates of one query
constexpr int N_BASELINES = 5;             // pop_recent, coocurrent, item_knn, cb, sr (rows of the metrics accumulator)

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// slot of `key`, inserting it when absent; -1 when the table is full
__device__ __forceinline__ int64_t find_or_insert(unsigned long long* keys, int64_t cap, unsigned long long key,
                                                  unsigned long long* count) {
  const unsigned long long mask = (unsigned long long)cap - 1;
  unsigned long long h = mix64(key) & mask;
  for (int64_t probe = 0; probe < cap; ++probe) {
    unsigned long long k = *(volatile unsigned long long*)(keys + h);
    if (k == key) return (int64_t)h;
    if (k == EMPTY) {
      const unsigned long long old = atomicCAS(keys + h, EMPTY, key);
      if (old == EMPTY) {
        if (count) atomicAdd(count, 1ull);
        return (int64_t)h;
      }
      if (old == key) return (int64_t)h;
    }
    h = (h + 1) & mask;
  }
  return -1;
}

__device__ __forceinline__ int64_t find(const unsigned long long* keys, int64_t cap, unsigned long long key) {
  const unsigned long long mask = (unsigned long long)cap - 1;
  unsigned long long h = mix64(key) & mask;
  for (int64_t probe = 0; probe < cap; ++probe) {
    const unsigned long long k = keys[h];
    if (k == key) return (int64_t)h;
    if (k == EMPTY) return -1;
    h = (h + 1) & mask;
  }
  return -1;
}

__global__ void clear_kernel(unsigned long long* keys, long long* cooc, long long* sr_w, long long* sr_first, int64_t cap) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = EMPTY; cooc[i] = 0; sr_w[i] = 0; sr_first[i] = 0x7fffffffffffffffLL;
  }
}

__global__ void rehash_kernel(const unsigned long long* keys, const long long* cooc, const long long* sr_w,
                              const long long* sr_first, int64_t cap, unsigned long long* nkeys, long long* ncooc,
                              long long* nsr_w, long long* nsr_first, int64_t ncap, int* err) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == EMPTY) continue;
    const int64_t s = find_or_insert(nkeys, ncap, k, nullptr);
    if (s < 0) { atomicExch(err, 2); continue; }
    ncooc[s] = cooc[i]; nsr_w[s] = sr_w[i]; nsr_first[s] = sr_first[i];
  }
}

// one CTA per session of the batch: all_items [Bg, T1] = item_clicked | label_last_item, padding 0 dropped
__global__ void __launch_bounds__(UPDATE_THREADS) update_kernel(
    unsigned long long* keys, long long* cooc, long long* sr_w, long long* sr_first, int64_t cap,
    unsigned long long* count, const int64_t* all_items, int64_t T1, int64_t num_items, int max_dist, long long unit,
    unsigned long long batch_seq, int* err) {
  __shared__ int64_t s_x[MAX_SESSION];
  __shared__ int s_first[MAX_SESSION];       // 1: no earlier position holds the same id
  __shared__ int s_next[MAX_SESSION];        // next position holding the same id, -1 if none
  __shared__ int s_len;
  const int64_t b = blockIdx.x;
  const int64_t* row = all_items + b * T1;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int64_t t = 0; t < T1; ++t) {
      const int64_t id = row[t];
      if (id == 0) continue;
      if (id < 0 || id >= num_items || n == MAX_SESSION) { atomicExch(err, 1); continue; }
      s_x[n++] = id;
    }
    s_len = n;
  }
  __syncthreads();
  const int L = s_len;
  if (L < 2) return;
  for (int p = threadIdx.x; p < L; p += blockDim.x) {
    int first = 1, nxt = -1;
    for (int q = 0; q < p; ++q) first &= (s_x[q] != s_x[p]);
    for (int q = L - 1; q > p; --q) if (s_x[q] == s_x[p]) nxt = q;
    s_first[p] = first; s_next[p] = nxt;
  }
  __syncthreads();
  // co-occurrence: one canonical (p, q) per distinct ordered pair of ids: p the first position of a, q the first position
  // of c (c != a) or the second position of a (c == a)
  for (int64_t idx = threadIdx.x; idx < (int64_t)L * L; idx += blockDim.x) {
    const int p = (int)(idx / L), q = (int)(idx % L);
    if (p == q || !s_first[p]) continue;
    const bool canon = (s_x[q] != s_x[p]) ? (s_first[q] != 0) : (q == s_next[p]);
    if (!canon) continue;
    const unsigned long long key = ((unsigned long long)s_x[p] << 32) | (unsigned long long)s_x[q];
    const int64_t s = find_or_insert(keys, cap, key, count);
    if (s < 0) { atomicExch(err, 2); continue; }
    atomicAdd(reinterpret_cast<unsigned long long*>(cooc + s), 1ull);
  }
  // sequential rules: every (j, i) with j < i <= j + max_dist, past = x_j, active = x_i
  const int D = max_dist;
  for (int64_t idx = threadIdx.x; idx < (int64_t)(L - 1) * D; idx += blockDim.x) {
    const int i = 1 + (int)(idx / D), d = 1 + (int)(idx % D), j = i - d;
    if (j < 0) continue;
    const unsigned long long key = ((unsigned long long)s_x[j] << 32) | (unsigned long long)s_x[i];
    const int64_t s = find_or_insert(keys, cap, key, count);
    if (s < 0) { atomicExch(err, 2); continue; }
    atomicAdd(reinterpret_cast<unsigned long long*>(sr_w + s), (unsigned long long)(unit / d));
    const long long ord = (long long)((b * T1 + i) * T1 + j);
    atomicMin(sr_first + s, (long long)((batch_seq << 32) | (unsigned long long)ord));
  }
}

// recent-clicks histogram: count and first index of every nonzero id of the buffer (Counter.most_common order)
__global__ void hist_kernel(const int64_t* buf, int64_t n, int64_t num_items, int* count, int* first, int* err) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t id = buf[i];
    if (id == 0) continue;
    if (id < 0 || id >= num_items) { atomicExch(err, 1); continue; }
    atomicAdd(count + id, 1);
    atomicMin(first + id, (int)i);
  }
}

__global__ void row_norms_kernel(const float* acr, int64_t V, int64_t dim, int64_t ld, double* norms) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t v = w; v < V; v += nw) {
    double s = 0.0;
    for (int64_t k = lane; k < dim; k += 32) { const double x = acr[v * ld + k]; s = fma(x, x, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) norms[v] = sqrt(s);
  }
}

struct ScoreArgs {
  const unsigned long long* keys; const long long *cooc, *sr_w, *sr_first; int64_t cap;
  const int64_t *item_clicked, *label_next, *negatives; int64_t B, T, K;
  const int* buf_count; const int* buf_first; const int64_t* articles_pop;
  const float* acr; int64_t acr_dim, acr_ld; const double* acr_norm; int64_t num_items;
  double knn_lambda, knn_alpha; int enabled; int top_n;
  unsigned long long* rank_hist;   // sampled: [N_BASELINES, top_n + 1]: queries whose label ranked r (< top_n), all queries
                                   // unsampled: [N_BASELINES, top_n + 2]: the same, then the competitor sum
  int64_t* out_ids;                // [N_BASELINES, B*T, top_n] or null
  int* err;
  // unsampled ranking only
  const int64_t* all_items;        // [B, T + 1] = item_clicked | label_last_item: the rows whose ids are not competitors
  const int64_t* pool; int64_t n_pool;
  int* rank;                       // [N_BASELINES, B*T] or null
};

// candidate x ranks before y: higher score, then lower tie key
__device__ __forceinline__ bool before(double sx, long long tx, double sy, long long ty) {
  return sx > sy || (sx == sy && tx < ty);
}

// Score, tie key and admissibility of candidate c (-1: an invalid id) of a query whose current click is `item`, for the
// pop_recent, coocurrent, item_knn and sr baselines (bl = 0, 1, 2, 4).  The sampled and the unsampled ranking both score
// through here, so a (query, id) pair gets the same score in both.
__device__ __forceinline__ void pair_score(const ScoreArgs& a, int bl, int64_t item, int64_t c, double& sc, long long& tie,
                                           int& ok) {
  sc = 0.0; tie = 0; ok = 0;
  if (c < 0) return;
  if (bl == 0) {                                                // pop_recent
    const int cnt = a.buf_count[c];
    sc = (double)cnt; tie = a.buf_first[c]; ok = cnt > 0;
    return;
  }
  const int64_t s = find(a.keys, a.cap, ((unsigned long long)item << 32) | (unsigned long long)c);
  if (s < 0) return;
  const long long co = a.cooc[s];
  if (bl == 1) { sc = (double)co; tie = -(long long)c; ok = co > 0; }
  else if (bl == 2) {                                           // item_knn (fp64, the reference's association)
    const double pc = pow((double)a.articles_pop[c] + a.knn_lambda, a.knn_alpha);
    const double pa = pow((double)a.articles_pop[item] + a.knn_lambda, 1.0 - a.knn_alpha);
    sc = __ddiv_rn((double)co, __dmul_rn(pc, pa)); tie = -(long long)c; ok = co > 0;
  } else {                                                      // sr
    const long long w = a.sr_w[s];
    sc = (double)w; tie = a.sr_first[s]; ok = w > 0;
  }
}

// cb: fp64 cosine of the ACR rows of `item` and c (-1: an invalid id, scores 0), one warp: lane-strided fma, then the
// xor-shuffle tree (every lane ends with the same sum).  A zero row scores 0.
__device__ __forceinline__ double cb_score(const ScoreArgs& a, int64_t item, int64_t c, int lane) {
  double dot = 0.0;
  if (c >= 0)
    for (int64_t k = lane; k < a.acr_dim; k += 32)
      dot = fma((double)a.acr[item * a.acr_ld + k], (double)a.acr[c * a.acr_ld + k], dot);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  const double nn = c >= 0 ? a.acr_norm[item] * a.acr_norm[c] : 0.0;
  return nn > 0.0 ? dot / nn : 0.0;
}

// one warp per query (b, t) with a nonzero label; candidates = label + the position's K negatives, first occurrence
// of each id only.  Per baseline: score + tie key + admissibility per candidate, then each admissible candidate's rank
// is the number of admissible candidates before it (a strict total order), ranks < top_n are written out.
__global__ void score_kernel(ScoreArgs a) {
  extern __shared__ unsigned char smem[];
  const int warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nc = (int)a.K + 1, ncp = (nc + 1) & ~1;        // ncp: 8-byte alignment of every warp's slice
  unsigned char* base = smem + (size_t)wid * ncp * (8 + 8 + 8 + 4);
  int64_t* s_id = reinterpret_cast<int64_t*>(base);
  double* s_score = reinterpret_cast<double*>(base + 8 * ncp);
  long long* s_tie = reinterpret_cast<long long*>(base + 16 * ncp);
  int* s_ok = reinterpret_cast<int*>(base + 24 * ncp);
  const int64_t nq = a.B * a.T;
  for (int64_t q = (int64_t)blockIdx.x * warps + wid; q < nq; q += (int64_t)gridDim.x * warps) {
    const int64_t label = a.label_next[q];
    if (label == 0) continue;                                   // warp-uniform
    const int64_t item = a.item_clicked[q];
    if (item <= 0 || item >= a.num_items || label < 0 || label >= a.num_items) {
      if (lane == 0) atomicExch(a.err, 1);
      continue;
    }
    for (int j = lane; j < nc; j += 32) {
      const int64_t id = j == 0 ? label : a.negatives[q * a.K + (j - 1)];
      s_id[j] = (id < 0 || id >= a.num_items) ? -1 : id;
      if (id < 0 || id >= a.num_items) atomicExch(a.err, 1);
    }
    __syncwarp();
    for (int bl = 0; bl < N_BASELINES; ++bl) {
      if (!((a.enabled >> bl) & 1)) continue;
      if (bl == 3) {                                            // cb: cosine of the ACR rows, warp-cooperative dots
        for (int j = 0; j < nc; ++j) {
          const int64_t c = s_id[j];
          const double sc = cb_score(a, item, c, lane);
          if (lane == 0) {
            s_score[j] = sc;
            s_tie[j] = -(long long)c;
            s_ok[j] = c >= 0;
          }
        }
        __syncwarp();
      } else {
        for (int j = lane; j < nc; j += 32) {
          double sc; long long tie; int ok;
          pair_score(a, bl, item, s_id[j], sc, tie, ok);
          s_score[j] = sc; s_tie[j] = tie; s_ok[j] = ok;
        }
        __syncwarp();
      }
      // duplicates: only the first occurrence of an id is a candidate
      for (int j = lane; j < nc; j += 32) {
        if (!s_ok[j]) continue;
        for (int k = 0; k < j; ++k) if (s_id[k] == s_id[j]) { s_ok[j] = 0; break; }
      }
      __syncwarp();
      int64_t* out = a.out_ids ? a.out_ids + ((int64_t)bl * nq + q) * a.top_n : nullptr;
      if (out) for (int r = lane; r < a.top_n; r += 32) out[r] = 0;
      __syncwarp();
      for (int j = lane; j < nc; j += 32) {
        if (!s_ok[j]) continue;
        int rank = 0;
        for (int k = 0; k < nc; ++k)
          if (k != j && s_ok[k] && before(s_score[k], s_tie[k], s_score[j], s_tie[j])) ++rank;
        if (rank < a.top_n) {
          if (out) out[rank] = s_id[j];
          if (j == 0) atomicAdd(a.rank_hist + bl * (a.top_n + 1) + rank, 1ull);
        }
      }
      if (lane == 0) atomicAdd(a.rank_hist + bl * (a.top_n + 1) + a.top_n, 1ull);
      __syncwarp();
    }
  }
}

// metrics[bl] += {hits, sum of reciprocal ranks, queries}, summed over the rank histogram in a fixed order
__global__ void finalize_kernel(const unsigned long long* rank_hist, int top_n, int enabled, double* metrics) {
  const int bl = threadIdx.x;
  if (bl >= N_BASELINES || !((enabled >> bl) & 1)) return;
  const unsigned long long* h = rank_hist + bl * (top_n + 1);
  unsigned long long hits = 0; double rr = 0.0;
  for (int r = 0; r < top_n; ++r) { hits += h[r]; rr += (double)h[r] / (double)(r + 1); }
  metrics[bl * 3 + 0] += (double)hits;
  metrics[bl * 3 + 1] += rr;
  metrics[bl * 3 + 2] += (double)h[top_n];
}

// ---- unsampled ranking (DESIGN.md section 14): each label against the pool minus its session's row
constexpr int RANK_NT = 256;
constexpr int RANK_WARPS = RANK_NT / 32;
constexpr int BLOOM_WORDS = 128;
constexpr int MISS = 0x7fffffff;           // rank of a label the baseline does not admit: a miss at every n

// One CTA per query (b, t) with label != 0 (grid-stride over the queries when the grid is capped).  The label is scored
// first; then every pool id outside the session row all_items[b] (behind a Bloom filter) other than the label is a
// competitor, scored as pair_score / cb_score score it (cb: one warp per id), and rank = the admissible competitors
// before the label in the baseline's strict order.  Integer histograms only.
__global__ void __launch_bounds__(RANK_NT) rank_unsampled_kernel(ScoreArgs a) {
  __shared__ int64_t s_excl[MAX_SESSION];
  __shared__ uint32_t s_bloom[BLOOM_WORDS];
  __shared__ double s_lsc[N_BASELINES];
  __shared__ long long s_ltie[N_BASELINES];
  __shared__ int s_lok[N_BASELINES];
  __shared__ int s_red[RANK_WARPS][N_BASELINES + 1];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t nq = a.B * a.T, T1 = a.T + 1;
  const int n_excl = (int)T1;
  for (int64_t q = blockIdx.x; q < nq; q += gridDim.x) {
    const int64_t label = a.label_next[q];
    const int64_t item = a.item_clicked[q];
    const bool bad = label != 0 && (item <= 0 || item >= a.num_items || label < 0 || label >= a.num_items);
    if (label == 0 || bad) {                                    // block-uniform
      if (tid == 0) {
        if (bad) atomicExch(a.err, 1);
        if (a.rank)
          for (int bl = 0; bl < N_BASELINES; ++bl) a.rank[bl * nq + q] = -1;
      }
      continue;
    }
    const int64_t b = q / a.T;
    __syncthreads();                                            // the previous query is done with the shared arrays
    for (int i = tid; i < BLOOM_WORDS; i += RANK_NT) s_bloom[i] = 0u;
    __syncthreads();
    for (int i = tid; i < n_excl; i += RANK_NT) {
      const int64_t id = a.all_items[b * T1 + i];
      s_excl[i] = id;
      const uint32_t h = bloom_slot(id);
      atomicOr(&s_bloom[h >> 5], 1u << (h & 31));
    }
    if (w == 0) {
      for (int bl = 0; bl < N_BASELINES; ++bl) {
        if (!((a.enabled >> bl) & 1)) continue;
        double sc; long long tie; int ok;
        if (bl == 3) { sc = cb_score(a, item, label, lane); tie = -(long long)label; ok = 1; }
        else pair_score(a, bl, item, label, sc, tie, ok);
        if (lane == 0) { s_lsc[bl] = sc; s_ltie[bl] = tie; s_lok[bl] = ok; }
      }
    }
    __syncthreads();
    auto competitor = [&](int64_t c) -> bool {
      if (c == label) return false;
      const uint32_t h = bloom_slot(c);
      if (s_bloom[h >> 5] & (1u << (h & 31)))
        for (int i = 0; i < n_excl; ++i)
          if (s_excl[i] == c) return false;
      return true;
    };
    int above[N_BASELINES], comp = 0;
#pragma unroll
    for (int bl = 0; bl < N_BASELINES; ++bl) above[bl] = 0;
    for (int64_t j = tid; j < a.n_pool; j += RANK_NT) {
      const int64_t c = a.pool[j];
      if (c <= 0 || c >= a.num_items) { atomicExch(a.err, 1); continue; }
      if (!competitor(c)) continue;
      ++comp;
#pragma unroll
      for (int bl = 0; bl < N_BASELINES; ++bl) {
        if (bl == 3 || !((a.enabled >> bl) & 1)) continue;
        double sc; long long tie; int ok;
        pair_score(a, bl, item, c, sc, tie, ok);
        above[bl] += ok && before(sc, tie, s_lsc[bl], s_ltie[bl]);
      }
    }
    if ((a.enabled >> 3) & 1) {
      for (int64_t j = w; j < a.n_pool; j += RANK_WARPS) {    // warp-uniform
        const int64_t c = a.pool[j];
        if (c <= 0 || c >= a.num_items || !competitor(c)) continue;
        const double sc = cb_score(a, item, c, lane);
        if (lane == 0) above[3] += before(sc, -(long long)c, s_lsc[3], s_ltie[3]);
      }
    }
#pragma unroll
    for (int bl = 0; bl <= N_BASELINES; ++bl) {
      int v = bl < N_BASELINES ? above[bl] : comp;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) s_red[w][bl] = v;
    }
    __syncthreads();
    if (tid < N_BASELINES && ((a.enabled >> tid) & 1)) {
      const int bl = tid;
      int ab = 0, cm = 0;
      for (int i = 0; i < RANK_WARPS; ++i) { ab += s_red[i][bl]; cm += s_red[i][N_BASELINES]; }
      const int r = s_lok[bl] ? ab : MISS;
      if (a.rank) a.rank[bl * nq + q] = r;
      unsigned long long* h = a.rank_hist + bl * (a.top_n + 2);
      if (r < a.top_n) atomicAdd(h + r, 1ull);
      atomicAdd(h + a.top_n, 1ull);
      atomicAdd(h + a.top_n + 1, (unsigned long long)cm);
    }
  }
}

// ---- recommendations (DESIGN.md section 16): the top n of one baseline's order over a candidate set
constexpr int REC_NT = 256;

struct RecArgs {
  const int32_t* q_pos; int64_t n_q;     // queries: flat positions b*T + t of item_clicked [B, T]
  const int64_t* cand; int64_t N;        // distinct candidate ids in [1, num_items)
  int exclude;                           // drop the query's clicks item_clicked[b, 0..t]
  int bl;                                // baseline: 0 pop_recent, 1 coocurrent, 2 item_knn, 3 cb, 4 sr
  int top_n;
  int64_t* out_ids; double* out_scores;  // [n_q, top_n]
};

// One CTA per query (grid-stride over the queries when the grid is capped).  The query's clicks sit behind the Bloom
// filter of rank_unsampled_kernel; the candidates are walked in tiles of REC_NT, each id scored as pair_score / cb_score
// score it (cb: one warp per id, 32 ids per warp and tile), and the admissible ones go through sel::offer.
__global__ void __launch_bounds__(REC_NT) recommend_kernel(ScoreArgs a, RecArgs r) {
  extern __shared__ __align__(16) unsigned char smem[];
  sel::KeySel& S = *reinterpret_cast<sel::KeySel*>(smem);
  __shared__ int64_t s_excl[MAX_SESSION];
  __shared__ uint32_t s_bloom[BLOOM_WORDS];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int bl = r.bl;
  for (int64_t q = blockIdx.x; q < r.n_q; q += gridDim.x) {
    const int64_t pos = r.q_pos[q];
    const int64_t b = pos / a.T, t = pos - b * a.T;
    const int64_t item = pos >= 0 && b < a.B ? a.item_clicked[pos] : 0;
    __syncthreads();                                            // the previous query is done with shared memory
    if (item <= 0 || item >= a.num_items) {                     // block-uniform
      if (tid == 0) atomicExch(a.err, 1);
      for (int i = tid; i < r.top_n; i += REC_NT) {
        r.out_ids[q * r.top_n + i] = 0;
        r.out_scores[q * r.top_n + i] = __longlong_as_double(0x7ff8000000000000LL);
      }
      continue;
    }
    for (int i = tid; i < BLOOM_WORDS; i += REC_NT) s_bloom[i] = 0u;
    sel::begin<REC_NT>(S);
    const int n_excl = r.exclude ? (int)(t + 1) : 0;
    for (int i = tid; i < n_excl; i += REC_NT) {
      const int64_t id = a.item_clicked[b * a.T + i];
      s_excl[i] = id;
      const uint32_t h = bloom_slot(id);
      atomicOr(&s_bloom[h >> 5], 1u << (h & 31));
    }
    __syncthreads();
    auto excluded = [&](int64_t c) -> bool {
      const uint32_t h = bloom_slot(c);
      if (s_bloom[h >> 5] & (1u << (h & 31)))
        for (int i = 0; i < n_excl; ++i)
          if (s_excl[i] == c) return true;
      return false;
    };
    if (q == 0)                                                 // the selection's key is strict only over distinct ids
      for (int64_t j = tid + 1; j < r.N; j += REC_NT)
        if (r.cand[j] <= r.cand[j - 1]) atomicExch(a.err, 3);
    for (int64_t j0 = 0; j0 < r.N; j0 += REC_NT) {
      bool ok = false; double sc = 0.0; long long tie = 0; int64_t c = 0;
      if (bl == 3) {                                            // block-uniform
        for (int k = 0; k < 32; ++k) {
          const int64_t j = j0 + w * 32 + k;
          if (j >= r.N) break;                                  // warp-uniform
          const int64_t cc = r.cand[j];
          if (cc <= 0 || cc >= a.num_items) { if (lane == 0) atomicExch(a.err, 1); continue; }
          if (excluded(cc)) continue;
          const double s = cb_score(a, item, cc, lane);
          if (lane == k) { sc = s; tie = -(long long)cc; ok = true; c = cc; }
        }
      } else if (j0 + tid < r.N) {
        c = r.cand[j0 + tid];
        if (c <= 0 || c >= a.num_items) atomicExch(a.err, 1);
        else if (!excluded(c)) { int o; pair_score(a, bl, item, c, sc, tie, o); ok = o; }
      }
      sel::offer<REC_NT, REC_NT>(S, r.top_n, ok, sc, tie, (int)c);
    }
    sel::finish<REC_NT>(S, r.top_n, r.out_ids + q * r.top_n, r.out_scores + q * r.top_n);
  }
}

static inline bool pow2(int64_t x) { return x > 0 && (x & (x - 1)) == 0; }
static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  return (int)(g < 1 ? 1 : (g > 8 * NAR_GRID_SMS ? 8 * NAR_GRID_SMS : g));
}

}  // namespace bl
}  // namespace nar

using namespace nar::bl;

extern "C" int nar_baselines_clear(int64_t* keys, int64_t* cooc, int64_t* sr_w, int64_t* sr_first, int64_t cap,
                                   void* stream) {
  if (!keys || !cooc || !sr_w || !sr_first || !pow2(cap) || cap > (1LL << 40)) return NAR_ERR_INVALID;
  clear_kernel<<<grid_for(cap, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<unsigned long long*>(keys),
                                                                   (long long*)cooc, (long long*)sr_w, (long long*)sr_first, cap);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_rehash(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first,
                                    int64_t cap, int64_t* new_keys, int64_t* new_cooc, int64_t* new_sr_w,
                                    int64_t* new_sr_first, int64_t new_cap, int* err, void* stream) {
  if (!keys || !cooc || !sr_w || !sr_first || !new_keys || !new_cooc || !new_sr_w || !new_sr_first || !err || !pow2(cap) ||
      !pow2(new_cap) || new_cap < cap)
    return NAR_ERR_INVALID;
  const int rc = nar_baselines_clear(new_keys, new_cooc, new_sr_w, new_sr_first, new_cap, stream);
  if (rc != NAR_OK) return rc;
  rehash_kernel<<<grid_for(cap, 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const unsigned long long*>(keys), (const long long*)cooc, (const long long*)sr_w,
      (const long long*)sr_first, cap, reinterpret_cast<unsigned long long*>(new_keys), (long long*)new_cooc,
      (long long*)new_sr_w, (long long*)new_sr_first, new_cap, err);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_update(int64_t* keys, int64_t* cooc, int64_t* sr_w, int64_t* sr_first, int64_t cap,
                                    int64_t* count, const int64_t* all_items, int64_t Bg, int64_t T1, int64_t num_items,
                                    int32_t max_clicks_dist, int64_t batch_seq, int* err, void* stream) {
  if (!keys || !cooc || !sr_w || !sr_first || !count || !all_items || !err || !pow2(cap) || Bg < 0 || T1 <= 0 ||
      num_items <= 0 || num_items > 0x7fffffffLL || batch_seq < 0 || batch_seq > 0x7fffffffLL)
    return NAR_ERR_INVALID;
  if (max_clicks_dist < 1 || max_clicks_dist > 20 || T1 > MAX_SESSION || Bg * T1 * T1 > 0xffffffffLL)
    return NAR_ERR_UNSUPPORTED;
  if (Bg == 0) return NAR_OK;
  long long unit = 1;                                    // lcm(1..max_clicks_dist)
  for (long long d = 2; d <= max_clicks_dist; ++d) {
    long long x = unit, y = d;
    while (y) { const long long r = x % y; x = y; y = r; }
    unit = unit / x * d;
  }
  update_kernel<<<(unsigned)Bg, UPDATE_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<unsigned long long*>(keys), (long long*)cooc, (long long*)sr_w, (long long*)sr_first, cap,
      reinterpret_cast<unsigned long long*>(count), all_items, T1, num_items, max_clicks_dist, unit,
      (unsigned long long)batch_seq, err);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_buffer_hist(const int64_t* buffer, int64_t n, int64_t num_items, int32_t* count,
                                         int32_t* first, int* err, void* stream) {
  if (!buffer || !count || !first || !err || n < 0 || n > 0x7fffffffLL || num_items <= 0) return NAR_ERR_INVALID;
  NAR_CHECK_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t) * num_items, as_stream(stream)));
  NAR_CHECK_CUDA(cudaMemsetAsync(first, 0x7f, sizeof(int32_t) * num_items, as_stream(stream)));
  if (n == 0) return NAR_OK;
  hist_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(buffer, n, num_items, count, first, err);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_row_norms(const float* acr, int64_t V, int64_t dim, int64_t ld, double* norms, void* stream) {
  if (!acr || !norms || V <= 0 || dim <= 0 || ld < dim) return NAR_ERR_INVALID;
  row_norms_kernel<<<grid_for(V * 32, 256), 256, 0, as_stream(stream)>>>(acr, V, dim, ld, norms);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_score(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first,
                                   int64_t cap, const int64_t* item_clicked, const int64_t* label_next,
                                   const int64_t* negatives, int64_t B, int64_t T, int64_t K, const int32_t* buf_count,
                                   const int32_t* buf_first, const int64_t* articles_pop, const float* acr, int64_t acr_dim,
                                   int64_t acr_ld, const double* acr_norm, int64_t num_items, double knn_lambda,
                                   double knn_alpha, int32_t enabled, int32_t top_n, int64_t* rank_hist, double* metrics,
                                   int64_t* out_ids, int* err, void* stream) {
  if (!item_clicked || !label_next || (!negatives && K > 0) || !rank_hist || !metrics || !err || B < 0 || T <= 0 || K < 0 ||
      top_n < 1 || num_items <= 0 || (enabled & ~31))
    return NAR_ERR_INVALID;
  if ((enabled & 1) && (!buf_count || !buf_first)) return NAR_ERR_INVALID;
  if ((enabled & (2 | 4 | 16)) && (!keys || !cooc || !sr_w || !sr_first || !pow2(cap))) return NAR_ERR_INVALID;
  if ((enabled & 4) && !articles_pop) return NAR_ERR_INVALID;
  if ((enabled & 8) && (!acr || !acr_norm || acr_dim <= 0 || acr_ld < acr_dim)) return NAR_ERR_INVALID;
  if (K + 1 > MAX_CAND) return NAR_ERR_UNSUPPORTED;
  cudaStream_t s = as_stream(stream);
  NAR_CHECK_CUDA(cudaMemsetAsync(rank_hist, 0, sizeof(int64_t) * N_BASELINES * (top_n + 1), s));
  if (enabled == 0) return NAR_OK;
  ScoreArgs a;
  a.keys = reinterpret_cast<const unsigned long long*>(keys); a.cooc = (const long long*)cooc;
  a.sr_w = (const long long*)sr_w; a.sr_first = (const long long*)sr_first; a.cap = cap;
  a.item_clicked = item_clicked; a.label_next = label_next; a.negatives = negatives; a.B = B; a.T = T; a.K = K;
  a.buf_count = buf_count; a.buf_first = buf_first; a.articles_pop = articles_pop;
  a.acr = acr; a.acr_dim = acr_dim; a.acr_ld = acr_ld; a.acr_norm = acr_norm; a.num_items = num_items;
  a.knn_lambda = knn_lambda; a.knn_alpha = knn_alpha; a.enabled = enabled; a.top_n = top_n;
  a.rank_hist = reinterpret_cast<unsigned long long*>(rank_hist); a.out_ids = out_ids; a.err = err;
  const int64_t per_warp = ((K + 2) & ~1LL) * 28;
  int warps = (int)(40960 / per_warp);
  warps = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
  const int64_t nq = B * T;
  if (nq > 0) {
    int64_t grid = (nq + warps - 1) / warps;
    if (grid > 16 * NAR_GRID_SMS) grid = 16 * NAR_GRID_SMS;
    score_kernel<<<(unsigned)grid, warps * 32, (size_t)(warps * per_warp), s>>>(a);
    NAR_LAUNCH_CHECK();
  }
  finalize_kernel<<<1, 32, 0, s>>>(a.rank_hist, top_n, enabled, metrics);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_rank_unsampled(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w,
                                            const int64_t* sr_first, int64_t cap, const int64_t* item_clicked,
                                            const int64_t* label_next, const int64_t* all_items, int64_t B, int64_t T,
                                            const int64_t* pool, int64_t N, const int32_t* buf_count,
                                            const int32_t* buf_first, const int64_t* articles_pop, const float* acr,
                                            int64_t acr_dim, int64_t acr_ld, const double* acr_norm, int64_t num_items,
                                            double knn_lambda, double knn_alpha, int32_t enabled, int32_t top_n,
                                            int64_t max_blocks, int32_t* rank, int64_t* hist, int* err, void* stream) {
  if (!item_clicked || !label_next || !all_items || (!pool && N > 0) || !hist || !err || B < 0 || T <= 0 || N < 0 ||
      top_n < 1 || num_items <= 0 || num_items > 0x7fffffffLL || (enabled & ~31))
    return NAR_ERR_INVALID;
  if ((enabled & 1) && (!buf_count || !buf_first)) return NAR_ERR_INVALID;
  if ((enabled & (2 | 4 | 16)) && (!keys || !cooc || !sr_w || !sr_first || !pow2(cap))) return NAR_ERR_INVALID;
  if ((enabled & 4) && !articles_pop) return NAR_ERR_INVALID;
  if ((enabled & 8) && (!acr || !acr_norm || acr_dim <= 0 || acr_ld < acr_dim)) return NAR_ERR_INVALID;
  if (T + 1 > MAX_SESSION || N > 0x7fffffffLL || B * T > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  cudaStream_t s = as_stream(stream);
  const int64_t nq = B * T;
  if (rank && nq > 0) NAR_CHECK_CUDA(cudaMemsetAsync(rank, 0xff, sizeof(int32_t) * N_BASELINES * nq, s));
  if (enabled == 0 || nq == 0) return NAR_OK;
  ScoreArgs a = {};
  a.keys = reinterpret_cast<const unsigned long long*>(keys); a.cooc = (const long long*)cooc;
  a.sr_w = (const long long*)sr_w; a.sr_first = (const long long*)sr_first; a.cap = cap;
  a.item_clicked = item_clicked; a.label_next = label_next; a.B = B; a.T = T;
  a.buf_count = buf_count; a.buf_first = buf_first; a.articles_pop = articles_pop;
  a.acr = acr; a.acr_dim = acr_dim; a.acr_ld = acr_ld; a.acr_norm = acr_norm; a.num_items = num_items;
  a.knn_lambda = knn_lambda; a.knn_alpha = knn_alpha; a.enabled = enabled; a.top_n = top_n;
  a.rank_hist = reinterpret_cast<unsigned long long*>(hist); a.err = err;
  a.all_items = all_items; a.pool = pool; a.n_pool = N; a.rank = rank;
  const int64_t grid = max_blocks > 0 && max_blocks < nq ? max_blocks : nq;
  rank_unsampled_kernel<<<(unsigned)grid, RANK_NT, 0, s>>>(a);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_baselines_recommend(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w,
                                       const int64_t* sr_first, int64_t cap, const int64_t* item_clicked, int64_t B,
                                       int64_t T, const int32_t* q_pos, int64_t Q, const int64_t* cand, int64_t N,
                                       int32_t exclude, const int32_t* buf_count, const int32_t* buf_first,
                                       const int64_t* articles_pop, const float* acr, int64_t acr_dim, int64_t acr_ld,
                                       const double* acr_norm, int64_t num_items, double knn_lambda, double knn_alpha,
                                       int32_t baseline, int32_t top_n, int64_t max_blocks, int64_t* out_ids,
                                       double* out_scores, int* err, void* stream) {
  if (!item_clicked || (!q_pos && Q > 0) || (!cand && N > 0) || !out_ids || !out_scores || !err || B < 0 || T <= 0 ||
      Q < 0 || N < 0 || top_n < 1 || num_items <= 0 || num_items > 0x7fffffffLL || baseline < 0 || baseline >= N_BASELINES)
    return NAR_ERR_INVALID;
  if (baseline == 0 && (!buf_count || !buf_first)) return NAR_ERR_INVALID;
  if ((baseline == 1 || baseline == 2 || baseline == 4) && (!keys || !cooc || !sr_w || !sr_first || !pow2(cap)))
    return NAR_ERR_INVALID;
  if (baseline == 2 && !articles_pop) return NAR_ERR_INVALID;
  if (baseline == 3 && (!acr || !acr_norm || acr_dim <= 0 || acr_ld < acr_dim)) return NAR_ERR_INVALID;
  if (top_n > nar::sel::MAX_TOP || T > MAX_SESSION || Q > 0x7fffffffLL || B * T > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  if (Q == 0) return NAR_OK;
  cudaStream_t s = as_stream(stream);
  constexpr size_t smem = sizeof(nar::sel::KeySel);
  static bool attr = false;
  if (!attr) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(recommend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  ScoreArgs a = {};
  a.keys = reinterpret_cast<const unsigned long long*>(keys); a.cooc = (const long long*)cooc;
  a.sr_w = (const long long*)sr_w; a.sr_first = (const long long*)sr_first; a.cap = cap;
  a.item_clicked = item_clicked; a.B = B; a.T = T;
  a.buf_count = buf_count; a.buf_first = buf_first; a.articles_pop = articles_pop;
  a.acr = acr; a.acr_dim = acr_dim; a.acr_ld = acr_ld; a.acr_norm = acr_norm; a.num_items = num_items;
  a.knn_lambda = knn_lambda; a.knn_alpha = knn_alpha; a.enabled = 1 << baseline; a.top_n = top_n; a.err = err;
  RecArgs r;
  r.q_pos = q_pos; r.n_q = Q; r.cand = cand; r.N = N; r.exclude = exclude != 0; r.bl = baseline; r.top_n = top_n;
  r.out_ids = out_ids; r.out_scores = out_scores;
  const int64_t grid = max_blocks > 0 && max_blocks < Q ? max_blocks : Q;
  recommend_kernel<<<(unsigned)grid, REC_NT, smem, s>>>(a, r);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
