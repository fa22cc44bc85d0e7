// Per-session evaluation logs of the reference hook (nar_model.py:1529-1581), packed on the GPU: the eval negatives of
// every query and / or its ranked candidates with their rounded probabilities and rounded normalised popularity, filtered
// to the cells with a nonzero label and laid out so that one device-to-host copy brings exactly what the host turns into
// lists.  Spec: oracle/session_logs_ref.py; layout and copy discipline: DESIGN.md section 12.
#include "common.cuh"

namespace nar {
namespace sl {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int ROWS = 16;                 // compact rows per CTA (<= 32: one ballot holds the chunk's query flags)
constexpr int HEADER_BYTES = 16;         // {Q, err, 0, 0} int32, then the per-session query counts

struct Args {
  const int64_t* pred_ids;               // [L, W] ranked candidate ids
  const float* pred_probs;               // [L, W]
  const int64_t* cand;                   // label of compact row r at cand[r * cand_stride]
  int64_t cand_stride;
  const int32_t* pos_idx;                // [L] flat b * T + t of compact row r
  const int32_t* sess_off;               // [B + 1]
  const float* pop;                      // [V]
  const int64_t* neg;                    // [B * T, K]
  const int64_t* label_next;             // [B * T]
  int B, L, K, W, Kp, Wp;
  int64_t V;
  int* hdr;
  int* counts;
  int64_t* o_neg;                        // [rows, Kp]   (null: log off)
  int64_t* o_labels;                     // [rows]       (null with o_ids, o_probs, o_pops: log off)
  int64_t* o_ids;                        // [rows, Wp]
  float* o_probs;                        // [rows, Wp]
  float* o_pops;                         // [rows, Wp]
};

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// ndarray.round(decimals=7) of a float32 array: rint(x * 1e7) / 1e7, every step rounded to float32 (1e7 is exact in it)
__device__ __forceinline__ float round7(float x) { return __fdiv_rn(rintf(__fmul_rn(x, 1e7f)), 1e7f); }

__device__ __forceinline__ int is_query(const Args& a, int r) { return a.label_next[a.pos_idx[r]] != 0; }

__global__ void __launch_bounds__(THREADS) nar_eval_session_logs_pack_kernel(Args a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row0 = blockIdx.x * ROWS;
  __shared__ int s_cnt[WARPS];

  // queries among the compact rows before this CTA's chunk: its first output row
  int c = 0;
  for (int r = threadIdx.x; r < row0; r += THREADS) c += is_query(a, r);
  c = __reduce_add_sync(0xffffffffu, c);
  if (lane == 0) s_cnt[warp] = c;
  __syncthreads();
  int before = 0;
#pragma unroll
  for (int w = 0; w < WARPS; ++w) before += s_cnt[w];
  const unsigned flags = __ballot_sync(0xffffffffu, lane < ROWS && row0 + lane < a.L && is_query(a, row0 + lane));

  // header: every session's query count (one thread per session over the whole grid), and Q from the last chunk
  for (int b = blockIdx.x * THREADS + threadIdx.x; b < a.B; b += gridDim.x * THREADS) {
    int n = 0;
    for (int r = a.sess_off[b]; r < a.sess_off[b + 1]; ++r) n += is_query(a, r);
    a.counts[b] = n;
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) a.hdr[0] = before + __popc(flags);

  bool bad = false;
  for (int i = warp; i < ROWS; i += WARPS) {
    if (!((flags >> i) & 1u)) continue;
    const int r = row0 + i;
    const int64_t q = before + __popc(flags & ((1u << i) - 1u));
    if (a.o_neg) {
      const int64_t* src = a.neg + (int64_t)a.pos_idx[r] * a.K;
      int64_t* dst = a.o_neg + q * a.Kp;
      for (int j = 2 * lane; j < a.Kp; j += 64) {
        longlong2 x;
        x.x = src[j];
        x.y = j + 1 < a.K ? src[j + 1] : 0;
        *reinterpret_cast<longlong2*>(dst + j) = x;
      }
    }
    if (a.o_ids) {
      const int64_t* ids = a.pred_ids + (int64_t)r * a.W;
      const float* probs = a.pred_probs + (int64_t)r * a.W;
      if (lane == 0) a.o_labels[q] = a.cand[(int64_t)r * a.cand_stride];
      int64_t* dst = a.o_ids + q * a.Wp;
      for (int j = 2 * lane; j < a.Wp; j += 64) {
        longlong2 x;
        x.x = j < a.W ? ids[j] : 0;
        x.y = j + 1 < a.W ? ids[j + 1] : 0;
        *reinterpret_cast<longlong2*>(dst + j) = x;
      }
      // one float4 per lane: the row's probabilities first, then its popularities
      const int nv = a.Wp / 4;
      for (int u = lane; u < 2 * nv; u += 32) {
        const bool is_pop = u >= nv;
        const int j0 = 4 * (is_pop ? u - nv : u);
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = j0 + e;
          float x = 0.f;
          if (j < a.W) {
            if (is_pop) {
              const int64_t id = ids[j];
              const bool ok = id >= 0 && id < a.V;
              bad |= !ok;
              x = ok ? round7(a.pop[id]) : 0.f;
            } else {
              x = round7(probs[j]);
            }
          }
          v[e] = x;
        }
        float* out = (is_pop ? a.o_pops : a.o_probs) + q * a.Wp + j0;
        *reinterpret_cast<float4*>(out) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  }
  if (bad) atomicExch(a.hdr + 1, 1);
}

}  // namespace sl
}  // namespace nar

using namespace nar::sl;

extern "C" int nar_eval_session_logs_layout(int64_t B, int64_t rows, int64_t K, int32_t flags, int64_t* offsets) {
  if (!offsets || B < 0 || rows < 0 || K < 1 || (flags & ~3)) return NAR_ERR_INVALID;
  const int64_t Kp = round_up(K, 2), Wp = round_up(K + 1, 4);
  int64_t off = round_up(HEADER_BYTES + 4 * B, 16);
  offsets[0] = HEADER_BYTES;
  offsets[1] = off;  if (flags & 1) off += rows * Kp * 8;
  offsets[2] = off;  if (flags & 2) off += round_up(rows * 8, 16);
  offsets[3] = off;  if (flags & 2) off += rows * Wp * 8;
  offsets[4] = off;  if (flags & 2) off += rows * Wp * 4;
  offsets[5] = off;  if (flags & 2) off += rows * Wp * 4;
  offsets[6] = off;
  offsets[7] = Kp;
  offsets[8] = Wp;
  return NAR_OK;
}

extern "C" int nar_eval_session_logs_pack(const int64_t* pred_ids, const float* pred_probs, const int64_t* cand,
                                          int64_t cand_stride, const int32_t* pos_idx, const int32_t* sess_off,
                                          const float* pop, const int64_t* negatives, const int64_t* label_next, int64_t B,
                                          int64_t K, int64_t L, int64_t num_items, int32_t flags, void* out, void* stream) {
  if (!pos_idx || !sess_off || !label_next || !out || B < 1 || K < 1 || L < 0 || num_items <= 0 || !(flags & 3) ||
      (flags & ~3) || ((flags & 1) && !negatives) ||
      ((flags & 2) && (!pred_ids || !pred_probs || !cand || !pop || cand_stride < 1)) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return NAR_ERR_INVALID;
  if (B > 0x7fffffffLL || L > 0x7fffffffLL || K > 0x0fffffffLL) return NAR_ERR_UNSUPPORTED;
  int64_t o[9];
  const int rc = nar_eval_session_logs_layout(B, L, K, flags, o);
  if (rc != NAR_OK) return rc;
  char* base = static_cast<char*>(out);
  Args a;
  a.pred_ids = pred_ids; a.pred_probs = pred_probs; a.cand = cand; a.cand_stride = cand_stride;
  a.pos_idx = pos_idx; a.sess_off = sess_off; a.pop = pop; a.neg = negatives; a.label_next = label_next;
  a.B = (int)B; a.L = (int)L; a.K = (int)K; a.W = (int)K + 1; a.Kp = (int)o[7]; a.Wp = (int)o[8]; a.V = num_items;
  a.hdr = reinterpret_cast<int*>(base);
  a.counts = reinterpret_cast<int*>(base + o[0]);
  a.o_neg = (flags & 1) ? reinterpret_cast<int64_t*>(base + o[1]) : nullptr;
  const bool rec = flags & 2;
  a.o_labels = rec ? reinterpret_cast<int64_t*>(base + o[2]) : nullptr;
  a.o_ids = rec ? reinterpret_cast<int64_t*>(base + o[3]) : nullptr;
  a.o_probs = rec ? reinterpret_cast<float*>(base + o[4]) : nullptr;
  a.o_pops = rec ? reinterpret_cast<float*>(base + o[5]) : nullptr;
  const unsigned grid = (unsigned)(L > 0 ? (L + ROWS - 1) / ROWS : 1);
  nar_eval_session_logs_pack_kernel<<<grid, THREADS, 0, as_stream(stream)>>>(a);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
