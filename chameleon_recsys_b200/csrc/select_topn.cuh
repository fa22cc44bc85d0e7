// Exact top n of a stream of keyed candidates for the baselines' recommendations (nar_baselines_recommend,
// nar_sknn_recommend; DESIGN.md section 16).  One CTA owns one query.  A key is (score desc, tie asc, id asc), a strict
// total order because candidate ids are distinct, so the result is the same for any tile size, grid or arrival order.
//
// Shared state: a sorted list [0, m) of at most top_n entries and a staging area [m, m + nb) behind it.  Every tile the
// CTA offers one candidate per thread; an admissible candidate that orders before the list's n-th entry (any admissible
// one while the list is short) is appended to the staging area.  A flush sorts list + staging (bitonic, best first) and
// keeps the first top_n.  It runs when the next tile might not fit and as soon as the list can first be filled, so the
// n-th entry becomes a filter early.  Shared memory does not bound the candidates: only top_n + one tile are held.
#pragma once
#include "common.cuh"

namespace nar {
namespace sel {

constexpr int CAP = 2048;                  // list + staging entries
constexpr int MAX_TOP = 1024;              // top_n bound: CAP - MAX_TOP entries are left for staging

struct KeySel {
  double sc[CAP];
  long long tie[CAP];
  int id[CAP];
  int m, nb;
};

__device__ __forceinline__ bool key_before(double sx, long long tx, int ix, double sy, long long ty, int iy) {
  return sx > sy || (sx == sy && (tx < ty || (tx == ty && ix < iy)));
}

__device__ __forceinline__ bool entry_before(const KeySel& S, int i, int j) {
  return key_before(S.sc[i], S.tie[i], S.id[i], S.sc[j], S.tie[j], S.id[j]);
}

// Sort entries [0, n) best first: the bitonic network whose comparators all point one way (the first step of each stage
// compares mirrored pairs), over the next power of two.  Slots >= n act as entries after every real one and never move,
// so a comparator with its upper slot >= n is skipped.  Called by all NT threads; ends with a barrier.
template <int NT>
__device__ void sort_entries(KeySel& S, int n) {
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      const bool flip = j == (k >> 1);
      for (int i = threadIdx.x; i < (n2 >> 1); i += NT) {
        const int blk = i / j, off = i - blk * j;
        const int lo = blk * 2 * j + off;
        const int hi = flip ? blk * 2 * j + 2 * j - 1 - off : lo + j;
        if (hi < n && entry_before(S, hi, lo)) {
          const double s = S.sc[lo]; S.sc[lo] = S.sc[hi]; S.sc[hi] = s;
          const long long t = S.tie[lo]; S.tie[lo] = S.tie[hi]; S.tie[hi] = t;
          const int d = S.id[lo]; S.id[lo] = S.id[hi]; S.id[hi] = d;
        }
      }
      __syncthreads();
    }
  }
}

template <int NT>
__device__ void flush(KeySel& S, int top_n) {
  const int n = S.m + S.nb;
  __syncthreads();                                     // every thread has read m and nb
  sort_entries<NT>(S, n);
  if (threadIdx.x == 0) { S.m = n < top_n ? n : top_n; S.nb = 0; }
  __syncthreads();
}

template <int NT>
__device__ __forceinline__ void begin(KeySel& S) {
  if (threadIdx.x == 0) { S.m = 0; S.nb = 0; }
  __syncthreads();
}

// One tile: every thread of the CTA calls it with its candidate (ok = admissible).  TILE: the most candidates one call
// can append (threads that may pass ok).  Ends with a barrier after every thread has read nb, so the flush decision is
// the same in every warp whatever the caller does before the next call (whose atomicAdd changes nb).
template <int NT, int TILE>
__device__ void offer(KeySel& S, int top_n, bool ok, double sc, long long tie, int id) {
  const int lane = threadIdx.x & 31;
  const int m = S.m;
  if (ok && m == top_n) ok = key_before(sc, tie, id, S.sc[m - 1], S.tie[m - 1], S.id[m - 1]);
  const unsigned bal = __ballot_sync(0xffffffffu, ok);
  int base = 0;
  if (lane == 0 && bal) base = atomicAdd(&S.nb, __popc(bal));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (ok) {
    const int p = m + base + __popc(bal & ((1u << lane) - 1u));
    S.sc[p] = sc; S.tie[p] = tie; S.id[p] = id;
  }
  __syncthreads();
  const int nb = S.nb;
  const bool full = m + nb + TILE > CAP || (m < top_n && m + nb >= top_n);
  __syncthreads();                                     // every thread has read nb before anyone can change it
  if (full) flush<NT>(S, top_n);                       // block-uniform
}

// Sorts what is staged and writes the query's row: the first top_n entries, then id 0 with score NaN.
template <int NT>
__device__ void finish(KeySel& S, int top_n, int64_t* out_ids, double* out_scores) {
  if (S.nb > 0) flush<NT>(S, top_n);                   // block-uniform (nb read after offer's barrier)
  const int m = S.m;
  for (int r = threadIdx.x; r < top_n; r += NT) {
    out_ids[r] = r < m ? (int64_t)S.id[r] : 0;
    out_scores[r] = r < m ? S.sc[r] : __longlong_as_double(0x7ff8000000000000LL);
  }
}

}  // namespace sel
}  // namespace nar
