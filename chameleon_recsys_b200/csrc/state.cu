// Device-resident ClickedItemsState (SURVEY.md section 8f #1): the recent-clicks buffer and the recent-popularity
// vector stay in HBM and are advanced by ONE single-CTA kernel per step instead of being recomputed on the host and
// re-uploaded (0.34 MB per step at G1).  Same arithmetic as clicked_items_state.py:187-250 / nar_model.py:1635-1646
// (spec: chameleon_recsys_b200/clicked_items_state.py, C host version csrc/host_state.cu):
//   batch clicks  = [item_clicked | label_last_item] flattened row-major, id 0 dropped, the last label carrying its
//                   session's maximum timestamp;
//   new buffer    = batch clicks reversed (newest first) ++ old entries with ts >= min(batch ts) - hours, clipped to
//                   `cap`, zero padded;
//   recent_pop    = bincount of the non-zero ids of the new buffer;  pop_norm = max(pop / (sum + 1), min_norm) in
//                   float64, stored as float32 (what the graph is fed) and optionally as float64;
//   articles_pop += bincount(batch clicks).
// Estimator.train advances the state with this kernel on every step (NAR_DEVICE_STATE=0 switches back to the host
// update and its per-step upload).  Checked bit for bit against oracle/clicked_items_state_ref.py by
// tests/test_device_state.py.
#include <limits.h>
#include "common.cuh"

namespace nar {
namespace state {

constexpr int THREADS = 1024;

// exclusive prefix over the block's threads (serial pass by thread 0: 1024 adds); *total = sum
__device__ int block_exclusive(int v, int* sh, int* total) {
  __syncthreads();
  sh[threadIdx.x] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < THREADS; ++i) { const int x = sh[i]; sh[i] = run; run += x; }
    *total = run;
  }
  __syncthreads();
  return sh[threadIdx.x];
}

__device__ __forceinline__ int64_t click_ts(const int64_t* __restrict__ event_ts, int64_t T, int64_t f) {
  const int64_t b = f / (T + 1), p = f - b * (T + 1);
  if (p < T) return event_ts[b * T + p];
  int64_t mx = 0;                                   // the last label inherits the session's maximum timestamp
  for (int64_t q = 0; q < T; ++q) { const int64_t v = event_ts[b * T + q]; mx = (q == 0 || v > mx) ? v : mx; }
  return mx;
}

__global__ void __launch_bounds__(THREADS)
state_update_kernel(const int64_t* __restrict__ old_items, const int64_t* __restrict__ old_ts, int64_t cap,
                    const int64_t* __restrict__ all_items, const int64_t* __restrict__ event_ts, int64_t Bg, int64_t T,
                    int64_t hours_ms, int64_t* __restrict__ new_items, int64_t* __restrict__ new_ts,
                    int64_t* __restrict__ recent_pop, float* __restrict__ pop_norm, double* __restrict__ pop_norm64,
                    int64_t* __restrict__ articles_pop, int64_t V, double min_norm, int* __restrict__ err) {
  __shared__ int s_scan[THREADS];
  __shared__ long long s_red[THREADS / 32];
  __shared__ int s_total;
  __shared__ long long s_min;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  // ---- batch clicks: count + minimum timestamp
  const int64_t nb = Bg * (T + 1);
  const int64_t chunk = (nb + THREADS - 1) / THREADS;
  const int64_t lo = min(nb, (int64_t)t * chunk), hi = min(nb, lo + chunk);
  int c = 0;
  long long mn = LLONG_MAX;
  for (int64_t f = lo; f < hi; ++f) {
    if (all_items[f] != 0) { ++c; const long long ts = click_ts(event_ts, T, f); mn = ts < mn ? ts : mn; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const long long x = __shfl_xor_sync(0xffffffffu, mn, o); mn = x < mn ? x : mn; }
  if (lane == 0) s_red[w] = mn;
  const int first = block_exclusive(c, s_scan, &s_total);          // (syncs: s_red is complete afterwards)
  if (t == 0) { long long m = LLONG_MAX; for (int i = 0; i < THREADS / 32; ++i) m = s_red[i] < m ? s_red[i] : m; s_min = m; }
  __syncthreads();
  const int n_batch = s_total;
  if (n_batch == 0) return;                                          // the hook leaves the state alone (host checks too)
  const long long thr = s_min - hours_ms;
  // ---- reversed batch -> head of the new buffer ; articles_pop += bincount(batch)
  int r = first;
  for (int64_t f = lo; f < hi; ++f) {
    const int64_t id = all_items[f];
    if (id == 0) continue;
    if (id < 0 || id >= V) { atomicExch(err, 1); ++r; continue; }
    const int64_t pos = (int64_t)n_batch - 1 - r;
    if (pos < cap) { new_items[pos] = id; new_ts[pos] = click_ts(event_ts, T, f); }
    atomicAdd(reinterpret_cast<unsigned long long*>(articles_pop + id), 1ULL);
    ++r;
  }
  // ---- old entries with ts >= thr, order kept
  const int64_t chunk2 = (cap + THREADS - 1) / THREADS;
  const int64_t lo2 = min(cap, (int64_t)t * chunk2), hi2 = min(cap, lo2 + chunk2);
  int k = 0;
  for (int64_t i = lo2; i < hi2; ++i) k += (old_ts[i] >= thr) ? 1 : 0;
  int kept_total;
  {
    __shared__ int s_kept;
    int pre = block_exclusive(k, s_scan, &s_kept);
    kept_total = s_kept;
    for (int64_t i = lo2; i < hi2; ++i) {
      if (old_ts[i] >= thr) {
        const int64_t pos = (int64_t)n_batch + pre;
        if (pos < cap) { new_items[pos] = old_items[i]; new_ts[pos] = old_ts[i]; }
        ++pre;
      }
    }
  }
  const int64_t filled = min(cap, (int64_t)n_batch + kept_total);
  for (int64_t i = filled + t; i < cap; i += THREADS) { new_items[i] = 0; new_ts[i] = 0; }
  for (int64_t v = t; v < V; v += THREADS) recent_pop[v] = 0;
  __syncthreads();                                                   // the new buffer and the zeroed counters are visible
  // ---- recent popularity
  int nz = 0;
  for (int64_t i = t; i < filled; i += THREADS) {
    const int64_t id = new_items[i];
    if (id != 0) {
      if (id < 0 || id >= V) { atomicExch(err, 1); continue; }
      atomicAdd(reinterpret_cast<unsigned long long*>(recent_pop + id), 1ULL);
      ++nz;
    }
  }
  int total_nz;
  {
    __shared__ int s_nz;
    block_exclusive(nz, s_scan, &s_nz);
    total_nz = s_nz;
  }
  const double denom = (double)(total_nz + 1);
  for (int64_t v = t; v < V; v += THREADS) {
    const double x = (double)recent_pop[v] / denom;
    const double y = x > min_norm ? x : min_norm;
    pop_norm[v] = (float)y;
    if (pop_norm64) pop_norm64[v] = y;
  }
}

}  // namespace state
}  // namespace nar

extern "C" int nar_state_update(const int64_t* old_items, const int64_t* old_ts, int64_t cap, const int64_t* all_items,
                                const int64_t* event_ts, int64_t Bg, int64_t T, int64_t hours_ms, int64_t* new_items,
                                int64_t* new_ts, int64_t* recent_pop, float* pop_norm, double* pop_norm64,
                                int64_t* articles_pop, int64_t num_items, double min_norm_pop, int* err, void* stream) {
  if (!old_items || !old_ts || !all_items || !event_ts || !new_items || !new_ts || !recent_pop || !pop_norm ||
      !articles_pop || !err)
    return NAR_ERR_INVALID;
  if (cap <= 0 || num_items <= 0 || Bg < 0 || T <= 0 || old_items == new_items || old_ts == new_ts) return NAR_ERR_INVALID;
  if (Bg * (T + 1) > 0x7fffffffLL || cap > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  if (Bg == 0) return NAR_OK;
  nar::state::state_update_kernel<<<1, nar::state::THREADS, 0, as_stream(stream)>>>(
      old_items, old_ts, cap, all_items, event_ts, Bg, T, hours_ms, new_items, new_ts, recent_pop, pop_norm, pop_norm64,
      articles_pop, num_items, min_norm_pop, err);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
