// Negative sampler of the NAR hot path (integer work; bit-exact against oracle/sampler_ref.py).
//
// Replaces nar_model.py:1220-1304 (tf.random_shuffle x (2 + one per click), tf.unique,
// tf.unsorted_segment_min, tf.setdiff1d inside nested tf.map_fn - a serial CPU while_loop in
// the reference).  "shuffle, keep first n" == keep the n smallest 64-bit keys
// (philox32 << 32 | idx); "shuffle, first-occurrence unique, first K" == per-item min key, K
// smallest items.  Order-independent, so every (session, click) is an independent CTA.
//
// kernel 1 (one CTA): stream 1 buffer sample -> stream 2 candidate pool (K*20 smallest keys,
//   sorted = shuffled order) -> unique item table + per-occurrence unique index.
// kernel 2 (one CTA per click): stream 3 keys for the pool occurrences, atomicMin per unique
//   item in shared memory, session items excluded (ListDiff), bitonic sort, first K.
#include "common.cuh"

namespace nar {
namespace sampler {

constexpr uint64_t KEY_MAX = 0xFFFFFFFFFFFFFFFFull;
constexpr int POOL_THREADS = 1024;
constexpr int CLICK_THREADS = 256;
constexpr int MAX_POOL = 16384;

struct PoolWs {
  uint64_t* key1;       // [buf_len]
  uint64_t* key2;       // [NB + buf_len]
  uint64_t* pool_key;   // [n_pool_cap] sorted stream-2 keys
  int64_t* pool_item;   // [n_pool_cap] item of pool position i
  int32_t* pool_uidx;   // [n_pool_cap] unique index of pool position i
  int64_t* uitems;      // [n_pool_cap] sorted unique items
  int32_t* counters;    // [4]: n_pool, n_unique
};

__device__ __forceinline__ uint32_t next_pow2(uint32_t x) {
  uint32_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

// block-wide bitonic sort of n (power of two) 64-bit keys in shared memory, ascending
__device__ void bitonic_sort(uint64_t* a, uint32_t n) {
  for (uint32_t k = 2; k <= n; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint64_t x = a[i], y = a[ixj];
          const bool up = (i & k) == 0;
          if ((x > y) == up) { a[i] = y; a[ixj] = x; }
        }
      }
      __syncthreads();
    }
  }
}

// bitonic sort of exactly blockDim.x (= 1024) keys, one per thread, a[] in shared memory (in and out).
// Compare-exchange distances below 32 stay inside a warp (shuffles, no barrier): 15 block barriers instead of 55.
__device__ void bitonic_sort_block1024(uint64_t* a, uint64_t* scratch /*[1024]*/) {
  const uint32_t i = threadIdx.x;
  uint64_t x = a[i];
  uint64_t* bufs[2] = {a, scratch};
  int cur = 0;
  for (uint32_t k = 2; k <= 1024u; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      uint64_t y;
      if (j >= 32u) {
        bufs[cur][i] = x;
        __syncthreads();
        y = bufs[cur][i ^ j];
        cur ^= 1;                     // next exchange writes the other buffer: no second barrier needed
      } else {
        y = __shfl_xor_sync(0xffffffffu, x, (int)j);
      }
      const bool up = (i & k) == 0;
      const bool lower = (i & j) == 0;
      const uint64_t mn = x < y ? x : y, mx = x < y ? y : x;
      x = (lower == up) ? mn : mx;
    }
  }
  __syncthreads();
  a[i] = x;
  __syncthreads();
}

// exclusive block scan of one int per thread (blockDim.x <= 1024); returns the exclusive prefix, total in *total
__device__ int block_exclusive_scan(int v, int* sh /*[33]*/, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    int s = (lane < (int)(blockDim.x >> 5)) ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sh[lane] = s;     // inclusive warp totals
  }
  __syncthreads();
  const int base = w == 0 ? 0 : sh[w - 1];
  *total = sh[(blockDim.x >> 5) - 1];
  const int res = base + x - v;
  __syncthreads();
  return res;
}

// threshold T such that exactly k of the (unique, != KEY_MAX) keys are <= T.  Requires 1 <= k <= #valid.
// MSB-first radix select, 11-bit digits; stops as soon as the k-th key is alone in its bucket.
__device__ uint64_t select_kth(const uint64_t* __restrict__ keys, int64_t n, int64_t k, int* hist /*[2048]*/,
                               int* scan_sh /*[33]*/, unsigned long long* sh_key) {
  uint64_t prefix = 0;       // bits above `shift` already fixed
  int shift = 64;
  int64_t kk = k;            // rank inside the current bucket (1-based)
  while (shift > 0) {
    const int bits = shift >= 11 ? 11 : shift;
    const int nshift = shift - bits;
    const int nb = 1 << bits;
    for (int i = threadIdx.x; i < nb; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint64_t key = keys[i];
      if (key == KEY_MAX) continue;
      const bool match = shift == 64 ? true : ((key >> shift) == prefix);
      if (match) atomicAdd(&hist[(int)((key >> nshift) & (uint64_t)(nb - 1))], 1);
    }
    __syncthreads();
    // locate the digit whose cumulative count crosses kk: each thread owns 2 consecutive bins
    const int b0 = threadIdx.x * 2;
    const int c0 = b0 < nb ? hist[b0] : 0, c1 = b0 + 1 < nb ? hist[b0 + 1] : 0;
    int total;
    const int ex = block_exclusive_scan(c0 + c1, scan_sh, &total);
    __shared__ int s_digit, s_below, s_count;
    if (c0 > 0 && ex < kk && kk <= ex + c0) { s_digit = b0; s_below = ex; s_count = c0; }
    if (c1 > 0 && ex + c0 < kk && kk <= ex + c0 + c1) { s_digit = b0 + 1; s_below = ex + c0; s_count = c1; }
    __syncthreads();
    prefix = (shift == 64 ? 0ull : (prefix << bits)) | (uint64_t)s_digit;
    kk -= s_below;
    const int cnt = s_count;
    shift = nshift;
    __syncthreads();
    if (cnt == 1 && shift > 0) {
      // the k-th key is the only one with this prefix: fetch it
      for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint64_t key = keys[i];
        if (key != KEY_MAX && (key >> shift) == prefix) *sh_key = key;
      }
      __syncthreads();
      const uint64_t r = *sh_key;
      __syncthreads();
      return r;
    }
  }
  return prefix;
}

__global__ void __launch_bounds__(POOL_THREADS, 1)
pool_kernel(const int64_t* __restrict__ all_items, int64_t NB, const int64_t* __restrict__ buffer, int64_t buf_len,
            int64_t n_from_buffer, int64_t n_pool_cap, uint64_t seed, uint32_t step, PoolWs ws) {
  extern __shared__ uint64_t sort_buf[];            // [next_pow2(n_pool_cap)]
  __shared__ int hist[2048];
  __shared__ int scan_sh[33];
  __shared__ unsigned long long sh_key;
  __shared__ int s_count;
  const int t = threadIdx.x;

  // ---- stream 1: buffer sample
  if (t == 0) s_count = 0;
  __syncthreads();
  int local = 0;
  for (int64_t i = t; i < buf_len; i += POOL_THREADS) {
    const bool ok = buffer[i] != 0;
    ws.key1[i] = ok ? shuffle_key(seed, step, 1u, 0u, (uint32_t)i) : KEY_MAX;
    local += ok;
  }
  atomicAdd(&s_count, local);
  __syncthreads();
  const int64_t n1 = min((int64_t)s_count, n_from_buffer);
  __syncthreads();
  uint64_t thr1 = 0;
  if (n1 > 0) thr1 = select_kth(ws.key1, buf_len, n1, hist, scan_sh, &sh_key);

  // ---- stream 2: candidate pool = batch clicks (with repetition) ++ buffer sample
  if (t == 0) s_count = 0;
  __syncthreads();
  local = 0;
  const int64_t n2 = NB + buf_len;
  for (int64_t i = t; i < n2; i += POOL_THREADS) {
    bool ok;
    if (i < NB) ok = all_items[i] != 0;
    else ok = n1 > 0 && ws.key1[i - NB] <= thr1;     // KEY_MAX entries never pass (thr1 < KEY_MAX)
    ws.key2[i] = ok ? shuffle_key(seed, step, 2u, 0u, (uint32_t)i) : KEY_MAX;
    local += ok;
  }
  atomicAdd(&s_count, local);
  __syncthreads();
  const int n_pool = (int)min((int64_t)s_count, n_pool_cap);
  __syncthreads();
  if (n_pool == 0) {
    if (t == 0) { ws.counters[0] = 0; ws.counters[1] = 0; }
    return;
  }
  const uint64_t thr2 = select_kth(ws.key2, n2, n_pool, hist, scan_sh, &sh_key);
  const uint32_t np2 = next_pow2((uint32_t)n_pool);
  for (uint32_t i = t; i < np2; i += POOL_THREADS) sort_buf[i] = KEY_MAX;
  if (t == 0) s_count = 0;
  __syncthreads();
  for (int64_t i = t; i < n2; i += POOL_THREADS) {
    const uint64_t key = ws.key2[i];
    if (key <= thr2) {                                           // exactly n_pool keys (keys are unique)
      const int slot = atomicAdd(&s_count, 1);
      if (slot < (int)np2) sort_buf[slot] = key;                 // (bounded anyway: corrupted keys must not become a wild store)
    }
  }
  __syncthreads();
  if (np2 <= 1024u) {                       // common case (K*20 <= 1024): register / shuffle bitonic network
    for (uint32_t i = np2 + t; i < 1024u; i += POOL_THREADS) sort_buf[i] = KEY_MAX;
    __syncthreads();
    bitonic_sort_block1024(sort_buf, sort_buf + 1024);
  } else {
    bitonic_sort(sort_buf, np2);
  }
  for (int i = t; i < n_pool; i += POOL_THREADS) {
    const uint64_t key = sort_buf[i];
    const int64_t ident = (int64_t)(key & 0xFFFFFFFFull);
    const int64_t item = ident < NB ? all_items[ident] : buffer[ident - NB];
    ws.pool_key[i] = key;
    ws.pool_item[i] = item;
  }
  __syncthreads();
  // ---- unique items: sort (item << 20 | pool position)
  for (uint32_t i = t; i < np2; i += POOL_THREADS)
    sort_buf[i] = i < (uint32_t)n_pool ? (((uint64_t)ws.pool_item[i] << 20) | (uint64_t)i) : KEY_MAX;
  __syncthreads();
  if (np2 <= 1024u) {
    for (uint32_t i = np2 + t; i < 1024u; i += POOL_THREADS) sort_buf[i] = KEY_MAX;
    __syncthreads();
    bitonic_sort_block1024(sort_buf, sort_buf + 1024);
  } else {
    bitonic_sort(sort_buf, np2);
  }
  // heads of runs -> unique index (contiguous chunk per thread keeps order)
  const int chunk = (n_pool + POOL_THREADS - 1) / POOL_THREADS;
  const int lo = min(n_pool, t * chunk), hi = min(n_pool, lo + chunk);
  int heads = 0;
  for (int i = lo; i < hi; ++i) heads += (i == 0) || ((sort_buf[i] >> 20) != (sort_buf[i - 1] >> 20));
  int total;
  int u = block_exclusive_scan(heads, scan_sh, &total);
  for (int i = lo; i < hi; ++i) {
    const bool head = (i == 0) || ((sort_buf[i] >> 20) != (sort_buf[i - 1] >> 20));
    if (head) { ws.uitems[u] = (int64_t)(sort_buf[i] >> 20); ++u; }
    ws.pool_uidx[(int)(sort_buf[i] & 0xFFFFFull)] = u - 1;
  }
  if (t == 0) { ws.counters[0] = n_pool; ws.counters[1] = total; }
}

__global__ void __launch_bounds__(CLICK_THREADS)
click_kernel(const int64_t* __restrict__ all_items, int64_t T1, int64_t sess0, int64_t K, uint64_t seed, uint32_t step,
             PoolWs ws, int64_t* __restrict__ out, int32_t* __restrict__ out_uidx, int32_t zero_slot) {
  extern __shared__ uint64_t ukey[];               // [next_pow2(n_unique)]
  const int64_t T = T1 - 1;
  const int64_t b = blockIdx.x / T, p = blockIdx.x % T;
  const int64_t* sess = all_items + (sess0 + b) * T1;
  int64_t* o = out + ((int64_t)blockIdx.x) * K;
  // optional second output: the index of each negative in the pool's sorted unique-item table (ws.uitems), or
  // zero_slot for a padding negative (id 0) - what the per-unique-id CAR layer 1 is keyed by
  int32_t* ou = out_uidx ? out_uidx + ((int64_t)blockIdx.x) * K : nullptr;
  const int n_pool = ws.counters[0], n_unique = ws.counters[1];
  if (sess[p] == 0 || n_unique == 0) {
    for (int64_t r = threadIdx.x; r < K; r += CLICK_THREADS) { o[r] = 0; if (ou) ou[r] = zero_slot; }
    return;
  }
  const uint32_t np2 = next_pow2((uint32_t)n_unique);
  for (uint32_t i = threadIdx.x; i < np2; i += CLICK_THREADS) ukey[i] = KEY_MAX;
  __syncthreads();
  const uint32_t ctx = (uint32_t)((sess0 + b) * T1 + p);
  // four pool positions share one Philox block
  for (int i4 = threadIdx.x * 4; i4 < n_pool; i4 += CLICK_THREADS * 4) {
    const Philox4 ph = philox4x32_10((uint32_t)i4 >> 2, ctx, 3u, step, (uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i4 + q;
      if (i < n_pool) {
        const uint64_t key = ((uint64_t)philox_word(ph, q) << 32) | (uint64_t)i;
        atomicMin(reinterpret_cast<unsigned long long*>(&ukey[ws.pool_uidx[i]]), (unsigned long long)key);
      }
    }
  }
  __syncthreads();
  // ListDiff: items clicked anywhere in this session are not candidates
  for (int64_t q = threadIdx.x; q < T1; q += CLICK_THREADS) {
    const int64_t it = sess[q];
    if (it == 0) continue;
    int lo = 0, hi = n_unique - 1;
    while (lo <= hi) {
      const int mid = (lo + hi) >> 1;
      const int64_t v = ws.uitems[mid];
      if (v == it) { ukey[mid] = KEY_MAX; break; }
      if (v < it) lo = mid + 1; else hi = mid - 1;
    }
  }
  __syncthreads();
  bitonic_sort(ukey, np2);
  for (int64_t r = threadIdx.x; r < K; r += CLICK_THREADS) {
    const uint64_t key = r < np2 ? ukey[r] : KEY_MAX;
    o[r] = key == KEY_MAX ? 0 : ws.pool_item[(int)(key & 0xFFFFFFFFull)];
    if (ou) ou[r] = key == KEY_MAX ? zero_slot : ws.pool_uidx[(int)(key & 0xFFFFFFFFull)];
  }
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

static int carve(void* base, int64_t bytes, int64_t NB, int64_t buf_len, int64_t cap, PoolWs* ws, int64_t* need) {
  int64_t off = 0;
  auto take = [&](int64_t n) { int64_t o = off; off = align_up(off + n, 256); return o; };
  const int64_t o1 = take(buf_len * 8), o2 = take((NB + buf_len) * 8), o3 = take(cap * 8), o4 = take(cap * 8),
                o5 = take(cap * 4), o6 = take(cap * 8), o7 = take(16);
  *need = off;
  if (!base) return NAR_OK;
  if (bytes < off) return NAR_ERR_WORKSPACE;
  char* b = static_cast<char*>(base);
  ws->key1 = reinterpret_cast<uint64_t*>(b + o1); ws->key2 = reinterpret_cast<uint64_t*>(b + o2);
  ws->pool_key = reinterpret_cast<uint64_t*>(b + o3); ws->pool_item = reinterpret_cast<int64_t*>(b + o4);
  ws->pool_uidx = reinterpret_cast<int32_t*>(b + o5); ws->uitems = reinterpret_cast<int64_t*>(b + o6);
  ws->counters = reinterpret_cast<int32_t*>(b + o7);
  return NAR_OK;
}

}  // namespace sampler
}  // namespace nar

extern "C" int nar_sample_negatives_workspace(int64_t Bg, int64_t T1, int64_t buf_len, int64_t K, int64_t* bytes) {
  if (!bytes || buf_len < 0) return NAR_ERR_INVALID;
  nar::sampler::PoolWs ws;
  return nar::sampler::carve(nullptr, 0, Bg * T1, buf_len, K * 20, &ws, bytes);
}

extern "C" int nar_sample_negatives(nar_ctx* ctx, const int64_t* all_items_global, int64_t Bg, int64_t T1, int64_t sess0,
                                    int64_t B, const int64_t* buffer, int64_t buf_len, int64_t K, int64_t n_from_buffer,
                                    uint64_t seed, uint32_t step, int64_t* out, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
  return nar_sample_negatives_uidx(ctx, all_items_global, Bg, T1, sess0, B, buffer, buf_len, K, n_from_buffer, seed, step, out,
                                   nullptr, nullptr, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int nar_sample_negatives_uidx(nar_ctx* ctx, const int64_t* all_items_global, int64_t Bg, int64_t T1, int64_t sess0,
                                         int64_t B, const int64_t* buffer, int64_t buf_len, int64_t K, int64_t n_from_buffer,
                                         uint64_t seed, uint32_t step, int64_t* out, int32_t* out_uidx,
                                         const int64_t** unique_items, const int32_t** n_unique, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  using namespace nar::sampler;
  if (!ctx || !all_items_global || !buffer || !out || !workspace) return NAR_ERR_INVALID;
  if (T1 < 2 || K <= 0 || B < 0 || sess0 < 0 || sess0 + B > Bg) return NAR_ERR_INVALID;
  // a negative buffer length would shrink the pool's stream and carve the workspace from negative sizes; a negative
  // sample count has no meaning (the oracle's slice would drop entries from the end)
  if (buf_len < 0 || n_from_buffer < 0) return NAR_ERR_INVALID;
  const int64_t cap = K * 20;
  if (cap > MAX_POOL) return NAR_ERR_UNSUPPORTED;
  if (Bg * T1 + buf_len >= (1ll << 32)) return NAR_ERR_UNSUPPORTED;
  PoolWs ws; int64_t need;
  int rc = carve(workspace, workspace_bytes, Bg * T1, buf_len, cap, &ws, &need);
  if (rc) return rc;
  uint32_t np2 = 1; while (np2 < (uint32_t)cap) np2 <<= 1;
  const size_t smem = (size_t)(np2 < 2048u ? 2048u : np2) * 8;     // pool kernel: 1024 keys + 1024 scratch at least
  static bool attr_set = false;
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_POOL * 8));
    NAR_CHECK_CUDA(cudaFuncSetAttribute(click_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_POOL * 8));
    attr_set = true;
  }
  cudaStream_t st = as_stream(stream);
  pool_kernel<<<1, POOL_THREADS, smem, st>>>(all_items_global, Bg * T1, buffer, buf_len, n_from_buffer, cap, seed, step, ws);
  NAR_LAUNCH_CHECK();
  if (B > 0) {
    click_kernel<<<(unsigned)(B * (T1 - 1)), CLICK_THREADS, smem, st>>>(all_items_global, T1, sess0, K, seed, step, ws, out,
                                                                         out_uidx, (int32_t)cap);
    NAR_LAUNCH_CHECK();
  }
  if (unique_items) *unique_items = ws.uitems;
  if (n_unique) *n_unique = ws.counters + 1;
  return NAR_OK;
}
