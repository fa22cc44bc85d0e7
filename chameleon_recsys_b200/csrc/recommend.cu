// Inference path: score a candidate set for every query position and keep the top n (NarEngine.recommend).
//
// A query is a valid position (b, t) of a batch; its candidate rows are concat(context(b, t), item_features(id)) * gamma
// + beta, scored exactly like a sampled negative (nar_model.py:356-364, :374-405, :444-515).  The first CAR layer splits
// as in csrc/car.cu: pre(q, j) = PC[q] + PI[j], so per (query, candidate) pair only the combine and the layers after it
// run.  This file holds the two kernels around the engine's GEMMs (csrc/engine.cu, run_recommend):
//   car_combine_grid_kernel  H1[q*Nc + j] = act(PC[q] + PI[j])  for a block of queries x a chunk of candidates
//   topn_kernel              per query row of logits [Q, N]: softmax statistics over the non-excluded candidates and an
//                            exact top n (radix select on order-preserving keys, compaction, bitonic sort of <= 4096)
//   rank_labels_kernel       per query row of logits [Q, N]: the label's rank among its non-excluded competitors and an
//                            integer histogram of the ranks below n (unsampled evaluation, DESIGN.md section 13)
#include "common.cuh"

namespace nar {
namespace rec {

constexpr int CG_NT = 256;
constexpr int CG_ROWS = 16;                 // candidate rows per CTA (the query's PC row is read once for all of them)

__global__ void __launch_bounds__(CG_NT)
car_combine_grid_kernel(const float* __restrict__ PC, const float* __restrict__ PI, int64_t Nc, int C, int act,
                        int64_t row_blocks, float* __restrict__ H1) {
  const int64_t q = blockIdx.x / row_blocks;
  const int64_t j0 = (blockIdx.x - q * row_blocks) * CG_ROWS;
  const int64_t j1 = j0 + CG_ROWS < Nc ? j0 + CG_ROWS : Nc;
  for (int c = threadIdx.x * 4; c < C; c += CG_NT * 4) {
    const float4 pc = *reinterpret_cast<const float4*>(PC + q * C + c);
    for (int64_t j = j0; j < j1; ++j) {
      float4 v = *reinterpret_cast<const float4*>(PI + j * C + c);
      // same operand order as car_combine_kernel (PI + PC): the layer-1 pre-activation of a pair is bit-identical
      v.x += pc.x; v.y += pc.y; v.z += pc.z; v.w += pc.w;
      *reinterpret_cast<float4*>(H1 + (q * Nc + j) * C + c) =
          make_float4(apply_act(v.x, act), apply_act(v.y, act), apply_act(v.z, act), apply_act(v.w, act));
    }
  }
}

// ------------------------------------------------------------------------------------------------ top n
constexpr int TOPN_NT = 512;
constexpr int TOPN_WARPS = TOPN_NT / 32;
constexpr int TOPN_MAX = 4096;
constexpr int BLOOM_WORDS = 128;            // 4096-bit filter in front of the exclusion list
constexpr int MAX_EXCL = 1024;

// float -> uint32 with the same order (larger float, larger key); key 0 is never produced by a non-NaN float
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t b = __float_as_uint(__fadd_rn(f, 0.0f));     // -0 -> +0: equal scores get equal keys

  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint32_t bloom_slot(int64_t id) { return ((uint32_t)id * 2654435761u) >> 20; }

struct TopnShared {
  unsigned long long sel[TOPN_MAX];         // (key << 32) | (0xffffffff - index): descending order = score desc, index asc
  int64_t excl[MAX_EXCL];
  uint32_t bloom[BLOOM_WORDS];
  int hist[256];
  double red_d[TOPN_WARPS];
  float red_f[TOPN_WARPS];
  int red_i[TOPN_WARPS];
  int warp_cnt[TOPN_WARPS];
  uint32_t prefix;
  int k_rem, n_above, tie_base, n_excl;
};

__global__ void __launch_bounds__(TOPN_NT)
topn_kernel(const float* __restrict__ logits, const int64_t* __restrict__ cand_ids, int64_t N, int top_n,
            const int64_t* __restrict__ item_clicked, const int32_t* __restrict__ q_pos, int64_t T,
            int64_t* __restrict__ out_ids, float* __restrict__ out_scores, float* __restrict__ out_probs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TopnShared& S = *reinterpret_cast<TopnShared*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t q = blockIdx.x;
  const float* lg = logits + q * N;

  // ---- exclusion list: the query's own clicks item_clicked[b, 0..t]
  for (int i = tid; i < BLOOM_WORDS; i += TOPN_NT) S.bloom[i] = 0u;
  if (tid == 0) S.n_excl = 0;
  __syncthreads();
  if (item_clicked) {
    const int64_t pos = q_pos[q], b = pos / T, t = pos - b * T;
    const int n = (int)(t + 1);
    for (int i = tid; i < n; i += TOPN_NT) {
      const int64_t id = item_clicked[b * T + i];
      S.excl[i] = id;
      const uint32_t h = bloom_slot(id);
      atomicOr(&S.bloom[h >> 5], 1u << (h & 31));
    }
    if (tid == 0) S.n_excl = n;
  }
  __syncthreads();
  const int n_excl = S.n_excl;
  auto excluded = [&](int64_t j) -> bool {
    if (n_excl == 0) return false;
    const int64_t id = cand_ids[j];
    const uint32_t h = bloom_slot(id);
    if (!(S.bloom[h >> 5] & (1u << (h & 31)))) return false;
    for (int i = 0; i < n_excl; ++i) if (S.excl[i] == id) return true;
    return false;
  };

  // ---- pass 1: max and count of the non-excluded candidates
  float mx = -INFINITY;
  int cnt = 0;
  for (int64_t j = tid; j < N; j += TOPN_NT) {
    if (excluded(j)) continue;
    mx = fmaxf(mx, lg[j]);
    ++cnt;
  }
  mx = warp_max(mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) { S.red_f[w] = mx; S.red_i[w] = cnt; }
  for (int i = tid; i < 256; i += TOPN_NT) S.hist[i] = 0;
  __syncthreads();
  mx = -INFINITY; cnt = 0;
  for (int i = 0; i < TOPN_WARPS; ++i) { mx = fmaxf(mx, S.red_f[i]); cnt += S.red_i[i]; }
  const int k_eff = cnt < top_n ? cnt : top_n;

  // warp-aggregated histogram increment (every lane of the warp calls it)
  auto hist_add = [&](bool valid, uint32_t bin) {
    const unsigned act = __ballot_sync(0xffffffffu, valid);
    if (valid) {
      const unsigned peers = __match_any_sync(act, bin);
      if (lane == __ffs(peers) - 1) atomicAdd(&S.hist[bin], __popc(peers));
    }
  };
  // warp 0: the bin holding the k-th largest key of the histogram, and how many of that bin are still needed
  auto select_bin = [&](int shift) {
    if (w == 0) {
      const int k = S.k_rem;
      int s = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += S.hist[255 - 8 * lane - i];
      int incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      int above = incl - s;
      if (above < k && k <= incl) {
        for (int i = 0; i < 8; ++i) {
          const int bin = 255 - 8 * lane - i, c = S.hist[bin];
          if (above + c >= k) { S.prefix |= (uint32_t)bin << shift; S.k_rem = k - above; break; }
          above += c;
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < 256; i += TOPN_NT) S.hist[i] = 0;
    __syncthreads();
  };

  // ---- pass 2: sum of exp (float64 accumulation) and the histogram of the top key byte
  if (tid == 0) { S.prefix = 0u; S.k_rem = k_eff; S.n_above = 0; S.tie_base = 0; }
  double se = 0.0;
  for (int64_t j0 = 0; j0 < N; j0 += TOPN_NT) {
    const int64_t j = j0 + tid;
    const bool ok = j < N && !excluded(j);
    uint32_t key = 0u;
    if (ok) { const float x = lg[j]; se += (double)expf(x - mx); key = order_key(x); }
    hist_add(ok, key >> 24);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  if (lane == 0) S.red_d[w] = se;
  __syncthreads();
  se = 0.0;
  for (int i = 0; i < TOPN_WARPS; ++i) se += S.red_d[i];

  if (k_eff > 0) {
    select_bin(24);
    // ---- passes 3-5: the lower key bytes among the keys that share the prefix chosen so far
    for (int shift = 16; shift >= 0; shift -= 8) {
      const uint32_t pre = S.prefix, pmask = 0xffffffffu << (shift + 8);
      for (int64_t j0 = 0; j0 < N; j0 += TOPN_NT) {
        const int64_t j = j0 + tid;
        bool ok = false; uint32_t key = 0u;
        if (j < N) { key = order_key(lg[j]); ok = (key & pmask) == pre && !excluded(j); }
        hist_add(ok, (key >> shift) & 255u);
      }
      __syncthreads();
      select_bin(shift);
    }
    // ---- compaction: every key above the pivot, then the k_rem lowest-index keys equal to it
    const uint32_t pivot = S.prefix;
    const int k_tie = S.k_rem, n_above = k_eff - k_tie;
    for (int64_t j0 = 0; j0 < N; j0 += TOPN_NT) {
      const int64_t j = j0 + tid;
      uint32_t key = 0u; bool ok = false;
      if (j < N) { key = order_key(lg[j]); ok = key >= pivot && !excluded(j); }
      const unsigned long long v = ((unsigned long long)key << 32) | (unsigned long long)(0xffffffffu - (uint32_t)j);
      if (ok && key > pivot) S.sel[atomicAdd(&S.n_above, 1)] = v;
      const bool tie = ok && key == pivot;
      const unsigned bt = __ballot_sync(0xffffffffu, tie);
      if (lane == 0) S.warp_cnt[w] = __popc(bt);
      __syncthreads();
      int base = S.tie_base;
      for (int i = 0; i < w; ++i) base += S.warp_cnt[i];
      const int rank = base + __popc(bt & ((1u << lane) - 1u));
      if (tie && rank < k_tie) S.sel[n_above + rank] = v;
      int tile = 0;
      if (tid == 0) for (int i = 0; i < TOPN_WARPS; ++i) tile += S.warp_cnt[i];
      __syncthreads();
      if (tid == 0) S.tie_base += tile;           // read again only after the next tile's first barrier
    }
  }
  // ---- bitonic sort (descending) of the k_eff selected entries, padded to a power of two
  int size = 1;
  while (size < k_eff) size <<= 1;
  __syncthreads();
  for (int i = k_eff + tid; i < size; i += TOPN_NT) S.sel[i] = 0ull;
  __syncthreads();
  for (int k = 2; k <= size; k <<= 1) {
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = tid; i < size; i += TOPN_NT) {
        const int ixj = i ^ jj;
        if (ixj > i) {
          const unsigned long long a = S.sel[i], b = S.sel[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? a < b : a > b) { S.sel[i] = b; S.sel[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int r = tid; r < top_n; r += TOPN_NT) {
    const int64_t o = q * top_n + r;
    if (r < k_eff) {
      const uint32_t j = 0xffffffffu - (uint32_t)(S.sel[r] & 0xffffffffull);
      const float s = lg[j];
      out_ids[o] = cand_ids[j];
      if (out_scores) out_scores[o] = s;
      if (out_probs) out_probs[o] = (float)(exp((double)s - (double)mx) / se);
    } else {                                 // fewer non-excluded candidates than top_n
      out_ids[o] = 0;
      if (out_scores) out_scores[o] = -INFINITY;
      if (out_probs) out_probs[o] = 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------ label rank
// Unsampled evaluation (NarEngine.rank_labels): per query row of logits [Q, N], the number of competitors whose key is
// above the label's.  Competitors are the candidates other than the label that are not in the session's row
// all_items[b, 0..T] (its clicks and its last label); ties go to the label.
constexpr int RANK_NT = 256;
constexpr int RANK_WARPS = RANK_NT / 32;

__global__ void __launch_bounds__(RANK_NT)
rank_labels_kernel(const float* __restrict__ logits, const int64_t* __restrict__ cand_ids, int64_t N,
                   const int64_t* __restrict__ label_next, const int64_t* __restrict__ all_items,
                   const int32_t* __restrict__ q_pos, int64_t T, int top_n, int32_t* __restrict__ rank,
                   unsigned long long* __restrict__ hist) {
  __shared__ int64_t excl[MAX_EXCL];
  __shared__ uint32_t bloom[BLOOM_WORDS];
  __shared__ int red_above[RANK_WARPS], red_comp[RANK_WARPS];
  __shared__ int64_t s_lab;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t q = blockIdx.x;
  const int64_t pos = q_pos[q], b = pos / T;
  const int n_excl = (int)(T + 1);
  for (int i = tid; i < BLOOM_WORDS; i += RANK_NT) bloom[i] = 0u;
  if (tid == 0) {                                  // the label's index in the ascending candidate ids, -1 when absent
    const int64_t id = label_next[pos];
    int64_t lo = 0, hi = N;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (cand_ids[mid] < id) lo = mid + 1; else hi = mid; }
    s_lab = (id != 0 && lo < N && cand_ids[lo] == id) ? lo : -1;
  }
  __syncthreads();
  const int64_t* row = all_items + b * (T + 1);
  for (int i = tid; i < n_excl; i += RANK_NT) {
    const int64_t id = row[i];
    excl[i] = id;
    const uint32_t h = bloom_slot(id);
    atomicOr(&bloom[h >> 5], 1u << (h & 31));
  }
  __syncthreads();
  const int64_t lab = s_lab;
  if (lab < 0) {                                   // a label outside the candidates is not ranked
    if (tid == 0) rank[q] = -1;
    return;
  }
  const float* lg = logits + q * N;
  const uint32_t key_lab = order_key(lg[lab]);
  int above = 0, comp = 0;
  for (int64_t j = tid; j < N; j += RANK_NT) {
    if (j == lab) continue;
    const int64_t id = cand_ids[j];
    const uint32_t h = bloom_slot(id);
    if (bloom[h >> 5] & (1u << (h & 31))) {
      bool hit = false;
      for (int i = 0; i < n_excl && !hit; ++i) hit = excl[i] == id;
      if (hit) continue;
    }
    ++comp;
    above += order_key(lg[j]) > key_lab;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    above += __shfl_xor_sync(0xffffffffu, above, o);
    comp += __shfl_xor_sync(0xffffffffu, comp, o);
  }
  if (lane == 0) { red_above[w] = above; red_comp[w] = comp; }
  __syncthreads();
  if (tid == 0) {
    above = 0; comp = 0;
    for (int i = 0; i < RANK_WARPS; ++i) { above += red_above[i]; comp += red_comp[i]; }
    rank[q] = above;
    if (above < top_n) atomicAdd(&hist[above], 1ull);
    atomicAdd(&hist[top_n], 1ull);
    atomicAdd(&hist[top_n + 1], (unsigned long long)comp);
  }
}

}  // namespace rec
}  // namespace nar

// Row lists of a recommend call: rows [0, L) = the clicked rows (row_pos = pos_idx[l], row_item = item_clicked[pos]),
// rows [L, L+N) = one item-only row per candidate (row_pos 0: no context is read for them).
namespace nar {
namespace rec {
__global__ void recommend_rows_kernel(const int32_t* __restrict__ pos_idx, int64_t L, const int64_t* __restrict__ item_clicked,
                                      const int64_t* __restrict__ cand_ids, int64_t N, int32_t* __restrict__ row_pos,
                                      int64_t* __restrict__ row_item) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < L + N; r += (int64_t)gridDim.x * blockDim.x) {
    if (r < L) { const int32_t p = pos_idx[r]; row_pos[r] = p; row_item[r] = item_clicked[p]; }
    else { row_pos[r] = 0; row_item[r] = cand_ids[r - L]; }
  }
}
}  // namespace rec
int recommend_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* cand_ids, int64_t N,
                   int32_t* row_pos, int64_t* row_item, cudaStream_t st) {
  const int64_t n = L + N;
  if (n <= 0) return NAR_OK;
  const int64_t blocks = (n + 255) / 256;
  rec::recommend_rows_kernel<<<(unsigned)(blocks > NAR_GRID_SMS * 8 ? NAR_GRID_SMS * 8 : blocks), 256, 0, st>>>(
      pos_idx, L, item_clicked, cand_ids, N, row_pos, row_item);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
}  // namespace nar

extern "C" int nar_car_combine_grid(const float* PC, const float* PI, int64_t Q, int64_t Nc, int64_t C, int act, float* H1,
                                    void* stream) {
  if (!PC || !PI || !H1 || (C & 3) || C <= 0) return NAR_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(PC) | reinterpret_cast<uintptr_t>(PI) | reinterpret_cast<uintptr_t>(H1)) & 15u) return NAR_ERR_INVALID;
  if (Q <= 0 || Nc <= 0) return NAR_OK;
  const int64_t row_blocks = (Nc + nar::rec::CG_ROWS - 1) / nar::rec::CG_ROWS;
  if (Q * row_blocks > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  nar::rec::car_combine_grid_kernel<<<(unsigned)(Q * row_blocks), nar::rec::CG_NT, 0, as_stream(stream)>>>(
      PC, PI, Nc, (int)C, act, row_blocks, H1);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_topn_candidates(const float* logits, const int64_t* cand_ids, int64_t Q, int64_t N, int32_t top_n,
                                   const int64_t* item_clicked, const int32_t* q_pos, int64_t T, int64_t* out_ids,
                                   float* out_scores, float* out_probs, void* stream) {
  if (!logits || !cand_ids || !out_ids) return NAR_ERR_INVALID;
  if (Q <= 0) return NAR_OK;
  if (N <= 0 || N >= 0xffffffffLL || top_n < 1 || top_n > nar::rec::TOPN_MAX || top_n > N) return NAR_ERR_INVALID;
  if (item_clicked && (!q_pos || T <= 0)) return NAR_ERR_INVALID;
  if (item_clicked && T > nar::rec::MAX_EXCL) return NAR_ERR_UNSUPPORTED;
  if (Q > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  const size_t smem = sizeof(nar::rec::TopnShared);
  static_assert(sizeof(nar::rec::TopnShared) <= 48 * 1024, "top-n scratch must fit the default shared-memory window");
  nar::rec::topn_kernel<<<(unsigned)Q, nar::rec::TOPN_NT, smem, as_stream(stream)>>>(
      logits, cand_ids, N, top_n, item_clicked, q_pos, T, out_ids, out_scores, out_probs);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_rank_labels(const float* logits, const int64_t* cand_ids, int64_t Q, int64_t N, const int64_t* label_next,
                               const int64_t* all_items, const int32_t* q_pos, int64_t T, int32_t top_n, int32_t* rank,
                               int64_t* hist, void* stream) {
  if (!logits || !cand_ids || !label_next || !all_items || !q_pos || !rank || !hist) return NAR_ERR_INVALID;
  if (Q <= 0) return NAR_OK;
  if (N <= 0 || N > 0x7fffffffLL || T <= 0 || top_n < 1) return NAR_ERR_INVALID;
  if (T + 1 > nar::rec::MAX_EXCL || Q > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  nar::rec::rank_labels_kernel<<<(unsigned)Q, nar::rec::RANK_NT, 0, as_stream(stream)>>>(
      logits, cand_ids, N, label_next, all_items, q_pos, T, top_n, rank, reinterpret_cast<unsigned long long*>(hist));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
