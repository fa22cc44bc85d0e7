// Feature-row assembly for the NAR hot path: the embedding gather (HBM-bound kernel the
// north_star names), its backward (gamma/beta grads + IndexedSlices scatter-add), and the
// recency / novelty normalisation statistics.
//
// Reference: nar_model.py:921-994 get_item_features, :730-773 get_features, :887-907
// scale_center_features, :996-1039 normalisation, :1055-1089 recency, :1134-1193 novelty.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>

namespace nar {
namespace feat {

constexpr float MS_PER_DAY = 1000.0f * 60.0f * 60.0f * 24.0f;

// nar_model.py:1055-1060 (int64 -> float32 BEFORE the subtraction) + log_1p :28-34
__device__ __forceinline__ float recency_raw(int64_t ts_ref, int64_t created, float inv_log_base) {
  // explicit _rn intrinsics: no FMA contraction, so that the value a row gets is bit-identical to the value
  // the statistics kernel saw (with degenerate variance, 1 ulp of difference is amplified by 1/1e-12)
  const float days = fmaxf(__fdiv_rn(__fsub_rn(__ll2float_rn(ts_ref), __ll2float_rn(created)), MS_PER_DAY), 0.f);
  return __fmul_rn(logf(__fadd_rn(days, 1.0f)), inv_log_base);
}
__device__ __forceinline__ float novelty_raw(float pop_norm, float inv_log_base) {
  return -__fmul_rn(logf(pop_norm), inv_log_base);
}
// normalize_values + min_max_normalization (:1011-1039, :996-1009); st = {mean, std, zmin, zmax}
__device__ __forceinline__ float normalize(float x, const float* st) {
  const float z = __fdiv_rn(__fsub_rn(x, st[0]), st[1]);
  const float scaled = __fdiv_rn(__fadd_rn(__fsub_rn(z, st[2]), 1e-24f), fmaxf(__fsub_rn(st[3], st[2]), 2e-24f));
  return __fsub_rn(__fmul_rn(scaled, 2.0f), 1.0f);
}

// statistics group of a row: 0 clicked (input) rows, 1 positives, 2 negatives.  n_cand > 0: candidate rows come in
// groups of n_cand, positive first; n_cand == 0: rows [n_input, n_input + n_positive) are the positives
__device__ __forceinline__ int row_group(int64_t r, int64_t n_input, int64_t n_cand, int64_t n_positive = 0) {
  if (r < n_input) return 0;
  if (n_cand <= 0) return r < n_input + n_positive ? 1 : 2;
  return ((r - n_input) % n_cand) == 0 ? 1 : 2;
}

// raw (un-scaled) value of column (c - seg.col) of segment `sg` for one row
__device__ __forceinline__ float seg_value(const nar_feature_plan& P, const nar_segment& sg, int j, int64_t pos,
                                           int64_t item, int64_t ts_ref, const float* st) {
  switch (sg.kind) {
    case NAR_SEG_CTX_OHE: { const int64_t id = P.ctx_int[sg.src][pos]; return id == j ? 1.f : 0.f; }
    case NAR_SEG_CTX_EMBED: {
      int64_t id = P.ctx_int[sg.src][pos]; id = id < 0 ? 0 : (id >= sg.card ? sg.card - 1 : id);
      return sg.table[id * sg.ld + j];
    }
    case NAR_SEG_CTX_NUM: return P.ctx_float[sg.src][pos];
    case NAR_SEG_CTX_ZERO: return 0.f;
    case NAR_SEG_META_OHE: { const int64_t id = P.meta[sg.src][item]; return id == j ? 1.f : 0.f; }
    case NAR_SEG_META_EMBED: {
      int64_t id = P.meta[sg.src][item]; id = id < 0 ? 0 : (id >= sg.card ? sg.card - 1 : id);
      return sg.table[id * sg.ld + j];
    }
    case NAR_SEG_META_NUM: return (float)P.meta[sg.src][item];
    case NAR_SEG_ACR:
    case NAR_SEG_ITEM_EMB: return sg.table[item * sg.ld + j];
    case NAR_SEG_RECENCY:
      return normalize(recency_raw(ts_ref, P.created_at_ts[item], 1.0f / logf(P.log_base_recency)), st);
    case NAR_SEG_NOVELTY:
      return normalize(novelty_raw(P.pop_norm[item], 1.0f / logf(P.log_base_novelty)), st + 4);
  }
  return 0.f;
}

// ------------------------------------------------------------------ forward gather
// ONE launch, two kinds of CTA, no shared memory, no prologue (a plain row gather of the same bytes runs at HBM
// speed because thousands of short independent warps are in flight - this kernel keeps that shape):
//  * "wide" CTAs: one warp per output row moves the wide table rows (ACR, item embedding): ids -> 128-bit
//    loads -> fma with gamma / beta -> 128-bit streaming stores.  That is ~87 % of the bytes.
//  * "narrow" CTAs: one warp per (chunk of 8 rows, group of 32 columns) writes the narrow columns (one-hot, small
//    embeddings, numerics, recency, novelty, padding), one lane per column.  Branch-free: the per-column descriptors (source lane,
//    kind, table offset / one-hot index, cardinality, stride) come from a device table owned by the context
//    (rebuilt by a one-CTA kernel only when the static part of the plan changes) and live in registers across
//    the rows; the scalars a row needs (context ids / floats at its position, metadata of its item) are
//    fetched by ONE lane each - for all 8 rows back to back, one memory round trip per chunk - finished to a
//    32-bit word and handed to the column lanes with shuffles; lanes 0-7 / 8-15 compute the normalised recency /
//    novelty of the 8 rows in one instruction stream.
//  History (profiles/gather_features_r1*.txt): v1 was bound by the serial instruction stream of each warp
//  (~1200 instructions per row: per-column switch statements, IEEE divisions + logf + a 64-bit modulo executed by
//  one lane while 31 idled); splitting showed the narrow columns - 13 % of the bytes - took 2/3 of the time.
constexpr int GATHER_WARPS = 8;
constexpr int GATHER_CHUNK = 8;
constexpr int GATHER_MAX_NARROW = 512;
constexpr int GATHER_MAX_TAIL = 8;
constexpr int LANE_CTX_INT = 0, LANE_CTX_FLOAT = 12, LANE_META = 20, LANE_RECENCY = 28, LANE_NOVELTY = 29;
enum { CK_ZERO = 0, CK_OHE = 1, CK_VALUE = 2, CK_EMBED = 3, CK_PAD = 4, CK_NONE = 0xff };
enum { SM_NONE = 0, SM_ID_AT_POS = 1, SM_FLOAT_AT_POS = 2, SM_ID_AT_ITEM = 3, SM_NUM_AT_ITEM = 4 };

// device table: d[i] = {col | kind << 16 | src_lane << 24, a, card - 1, ld}; a = one-hot index (CK_OHE) or the
// offset in floats of table[0][j] from GatherArgs::ebase (CK_EMBED)
struct GatherDesc {
  int4 d[GATHER_MAX_NARROW];
  int n_narrow;
  int pad_[15];
};
static_assert(sizeof(GatherDesc) <= NAR_GATHER_DESC_BYTES, "context scratch too small");

struct GatherArgs {
  const void* src[32];            // scalar source of lane l (phase A), or NULL
  unsigned char mode[32];         // SM_*
  const float* wtab[2];           // wide segments (ACR, item embedding): 16-byte aligned body
  int wcol[2], wld[2], wnvec[2];
  int ntail;                      // columns of the wide segments that cannot move as 128-bit vectors
  short tail_col[GATHER_MAX_TAIL]; unsigned char tail_seg[GATHER_MAX_TAIL]; short tail_j[GATHER_MAX_TAIL];
  const float* ebase;             // lowest address of the small embedding tables
  const float* gamma; const float* beta; const float* stats;
  const int64_t* created_at_ts; const float* pop_norm;
  float log_base_recency, log_base_novelty;
  int row_ld, n_narrow_blocks, period, n_col_groups;   // n_col_groups = ceil(narrow columns / 32)
  int n_positive;                 // n_cand == 0 layout: rows [n_input, n_input + n_positive) are positives
  int n_full, ctx_col0;           // rows >= n_full carry item features only: their columns >= ctx_col0 are written as 0
};

__global__ void __launch_bounds__(128)
gather_setup_kernel(const __grid_constant__ nar_feature_plan P, int n_narrow_plain, const float* ebase,
                    GatherDesc* __restrict__ D) {
  const int tid = threadIdx.x;
  if (tid == 0) D->n_narrow = n_narrow_plain;
  for (int i = tid; i < n_narrow_plain; i += blockDim.x) {
    int c = i, q = 0;
    while (q < P.n_narrow - 1 && c >= P.narrow_end[q] - P.narrow_begin[q]) { c -= P.narrow_end[q] - P.narrow_begin[q]; ++q; }
    c += P.narrow_begin[q];
    const int si = P.col_seg[c];
    int kind = CK_PAD, src_lane = 0, a = 0, cm1 = 0, ld = 0;      // padding columns are written as 0
    if (si != 255) {
      kind = CK_ZERO;
      const nar_segment& g = P.seg[si];
      const int j = c - g.col;
      switch (g.kind) {
        case NAR_SEG_CTX_OHE: kind = CK_OHE; src_lane = LANE_CTX_INT + g.src; a = j; break;
        case NAR_SEG_META_OHE: kind = CK_OHE; src_lane = LANE_META + g.src; a = j; break;
        case NAR_SEG_CTX_EMBED: kind = CK_EMBED; src_lane = LANE_CTX_INT + g.src; a = (int)(g.table + j - ebase); cm1 = g.card - 1; ld = g.ld; break;
        case NAR_SEG_META_EMBED: kind = CK_EMBED; src_lane = LANE_META + g.src; a = (int)(g.table + j - ebase); cm1 = g.card - 1; ld = g.ld; break;
        case NAR_SEG_CTX_NUM: kind = CK_VALUE; src_lane = LANE_CTX_FLOAT + g.src; break;
        case NAR_SEG_META_NUM: kind = CK_VALUE; src_lane = LANE_META + g.src; break;
        case NAR_SEG_RECENCY: kind = CK_VALUE; src_lane = LANE_RECENCY; break;
        case NAR_SEG_NOVELTY: kind = CK_VALUE; src_lane = LANE_NOVELTY; break;
        default: break;   // CTX_ZERO: raw 0 -> beta
      }
    }
    D->d[i] = make_int4(c | (kind << 16) | (src_lane << 24), a, cm1, ld);
  }
}

__device__ __forceinline__ int clamp_id32(long long v) {
  return v < -1 ? -1 : (v > 0x7fffffffLL ? 0x7fffffff : (int)v);
}
__device__ __forceinline__ void ld_b64(const void* p, unsigned& lo, unsigned& hi) {
  asm volatile("ld.global.nc.v2.u32 {%0, %1}, [%2];" : "=r"(lo), "=r"(hi) : "l"(p));
}
__device__ __forceinline__ void ld_b32(const void* p, unsigned& lo) {
  asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(lo) : "l"(p));
}

// raw (un-scaled) value of a narrow column, branch-free: z / a / cm1 / ld from the descriptor, val = the
// scalar of the column's source lane
__device__ __forceinline__ float narrow_raw(int z, int a, int cm1, int ld, const float* __restrict__ ebase, int val) {
  const int kind = (z >> 16) & 0xff;
  const int idx = max(0, min(val, cm1));
  float re = 0.f;
  if (kind == CK_EMBED) re = __ldg(ebase + (a + idx * ld));
  const float r1 = (kind == CK_OHE && val == a) ? 1.f : re;
  return kind == CK_VALUE ? __int_as_float(val) : r1;
}

template <int WU>                                  // 128-bit vectors of wide table data per lane and row
__global__ void __launch_bounds__(GATHER_WARPS * 32, (WU <= 4 ? 5 : 3))
gather_features_kernel(const __grid_constant__ GatherArgs A, const GatherDesc* __restrict__ D,
                       const int32_t* __restrict__ row_pos, const int64_t* __restrict__ row_item,
                       int n_rows, int n_input, int n_cand,
                       const int64_t* __restrict__ event_ts, const int64_t* __restrict__ max_ts,
                       float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  // narrow and wide CTAs are interleaved in launch order (period P): the narrow ones are latency bound, the wide
  // ones HBM bound, so they should be resident together
  const int b = (int)blockIdx.x, P = A.period, nbP = A.n_narrow_blocks * P;
  const bool is_narrow = b < nbP && (b % P) == 0;
  if (!is_narrow) {
    // ================================================================ wide CTA: one warp per row
    const int wblock = b < nbP ? b - b / P - 1 : b - A.n_narrow_blocks;
    const int r = wblock * GATHER_WARPS + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    const long long item = row_item[r];
    const int nv0 = A.wnvec[0], nvt = nv0 + A.wnvec[1];
    float* orowf = out + (int64_t)r * A.row_ld;
    float4* orow = reinterpret_cast<float4*>(orowf);
    const float* r0 = A.wtab[0] + item * (int64_t)A.wld[0];
    const float* r1 = A.wtab[1] + item * (int64_t)A.wld[1];
    const float4* t0 = reinterpret_cast<const float4*>(r0);
    const float4* t1 = reinterpret_cast<const float4*>(r1) - nv0;
    const int c0 = A.wcol[0] >> 2, c1 = (A.wcol[1] >> 2) - nv0;
    float4 wv[WU];
#pragma unroll
    for (int u = 0; u < WU; ++u) {
      const int v = u * 32 + lane;
      if (v < nvt) wv[u] = __ldg((v >= nv0 ? t1 : t0) + v);
    }
    float tv = 0.f;
    if (lane < A.ntail) tv = __ldg((A.tail_seg[lane] ? r1 : r0) + A.tail_j[lane]);
#pragma unroll
    for (int u = 0; u < WU; ++u) {
      const int v = u * 32 + lane;
      if (v < nvt) {
        const int c4 = (v >= nv0 ? c1 : c0) + v;
        const float4 g = __ldg(reinterpret_cast<const float4*>(A.gamma) + c4), b = __ldg(reinterpret_cast<const float4*>(A.beta) + c4);
        float4 x = wv[u];
        x.x = x.x * g.x + b.x; x.y = x.y * g.y + b.y; x.z = x.z * g.z + b.z; x.w = x.w * g.w + b.w;
        __stcs(orow + c4, x);                       // streaming store: the row is consumed once by the GEMM's TMA
      }
    }
    if (lane < A.ntail) { const int c = A.tail_col[lane]; orowf[c] = tv * __ldg(A.gamma + c) + __ldg(A.beta + c); }
    return;
  }
  // ================================================================== narrow CTA: one warp per (chunk of 8 rows, 32 columns)
  constexpr int CH = GATHER_CHUNK;
  const int w = (b / P) * GATHER_WARPS + (threadIdx.x >> 5);
  const int chunk = w / A.n_col_groups, n = w - chunk * A.n_col_groups;
  const int base = chunk * CH;
  if (base >= n_rows) return;
  const int rows_here = min(CH, n_rows - base);
  // this lane's column: descriptor, gamma, beta
  const int i = n * 32 + lane;
  int nd_z = CK_NONE << 16, nd_a = 0, nd_c = 0, nd_l = 0;
  float nd_g = 0.f, nd_b = 0.f;
  if (i < D->n_narrow) {
    const int4 d = __ldg(&D->d[i]);
    nd_z = d.x; nd_a = d.y; nd_c = d.z; nd_l = d.w;
    if (((d.x >> 16) & 0xff) != CK_PAD) { nd_g = __ldg(A.gamma + (d.x & 0xffff)); nd_b = __ldg(A.beta + (d.x & 0xffff)); }
  }
  const int kind = (nd_z >> 16) & 0xff;
  const bool uses_src = kind == CK_OHE || kind == CK_VALUE || kind == CK_EMBED;
  // which scalar sources do the 32 columns of this warp need?
  const unsigned need = __reduce_or_sync(0xffffffffu, uses_src ? (1u << ((unsigned)nd_z >> 24)) : 0u);
  const int my_mode = ((need >> lane) & 1u) ? A.mode[lane] : SM_NONE;
  const char* my_src = static_cast<const char*>(A.src[lane]);
  int c_pos = 0; long long c_item = 0; float c_norm = 0.f;
  if ((lane & 7) < rows_here) {
    const int rr = base + (lane & 7);
    c_pos = row_pos[rr]; c_item = row_item[rr];
  }
  // ---- the scalars of all rows, one lane per source, all loads in flight together
  unsigned lo[CH], hi[CH];
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const int pos = __shfl_sync(0xffffffffu, c_pos, k);
    const long long item = __shfl_sync(0xffffffffu, c_item, k);
    lo[k] = 0; hi[k] = 0;
    if (k < rows_here) {
      if (my_mode == SM_FLOAT_AT_POS) ld_b32(my_src + 4 * (int64_t)pos, lo[k]);
      else if (my_mode == SM_ID_AT_POS) ld_b64(my_src + 8 * (int64_t)pos, lo[k], hi[k]);
      else if (my_mode >= SM_ID_AT_ITEM) ld_b64(my_src + 8 * item, lo[k], hi[k]);
    }
  }
  // ---- normalised recency (lanes 0-7) / novelty (lanes 8-15) of the chunk's rows, if a column here needs them
  const int role = lane >> 3;
  if ((lane & 7) < rows_here && role < 2 && ((need >> (LANE_RECENCY + role)) & 1u)) {
    const int rr = base + (lane & 7);
    float x, scale;
    if (role == 0) {
      const int64_t ts_ref = (rr < n_input) ? event_ts[c_pos] : max_ts[0];
      // nar_model.py:1055-1060: int64 -> float32 BEFORE the subtraction; _rn intrinsics, see recency_raw()
      const float days = fmaxf(__fdiv_rn(__fsub_rn(__ll2float_rn(ts_ref), __ll2float_rn(A.created_at_ts[c_item])), MS_PER_DAY), 0.f);
      x = __fadd_rn(days, 1.0f);
      scale = 1.0f / logf(A.log_base_recency);
    } else {
      x = A.pop_norm[c_item];
      scale = -(1.0f / logf(A.log_base_novelty));
    }
    const float raw = __fmul_rn(logf(x), scale);               // == recency_raw / novelty_raw bit for bit
    const int g = rr < n_input ? 0 : (n_cand <= 0 ? (rr < n_input + A.n_positive ? 1 : 2)
                                                  : (((unsigned)(rr - n_input) % (unsigned)n_cand) == 0 ? 1 : 2));
    c_norm = normalize(raw, A.stats + 8 * g + 4 * role);
  }
  const int src_lane = (unsigned)nd_z >> 24;
  float* ocol = out + (int64_t)base * A.row_ld + (nd_z & 0xffff);
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    if (k < rows_here) {
      const float nrm = __shfl_sync(0xffffffffu, c_norm, (lane == LANE_NOVELTY ? 8 : 0) + k);
      // finish the scalar (branch-free): int64 -> clamped int32 id / float, one 32-bit word to shuffle
      const long long a64 = (long long)(((unsigned long long)hi[k] << 32) | lo[k]);
      const int as_id = clamp_id32(a64);
      const int as_num = __float_as_int((float)a64);
      int mine = my_mode == SM_NONE ? __float_as_int(nrm) : as_id;     // lanes LANE_RECENCY / LANE_NOVELTY: SM_NONE
      mine = my_mode == SM_FLOAT_AT_POS ? (int)lo[k] : mine;
      mine = my_mode == SM_NUM_AT_ITEM ? as_num : mine;
      const int val = __shfl_sync(0xffffffffu, mine, src_lane);
      const float raw = narrow_raw(nd_z, nd_a, nd_c, nd_l, A.ebase, val);
      const bool item_only = (base + k >= A.n_full) && ((nd_z & 0xffff) >= A.ctx_col0);    // no context on this row
      if (kind != CK_NONE) ocol[(int64_t)k * A.row_ld] = item_only ? 0.f : raw * nd_g + nd_b;
    }
  }
}

// ------------------------------------------------------------------ backward
// thread per column, CTA per block of rows: d_beta[c] += sum dX ; d_gamma[c] += sum dX*raw ;
// trainable embeddings: grad[id, j] += dX*gamma (scatter-add of the IndexedSlices gradient)
constexpr int BWD_ROWS = 32;
constexpr int BWD_THREADS = 256;

__global__ void __launch_bounds__(BWD_THREADS)
gather_features_bwd_kernel(const __grid_constant__ nar_feature_plan P, const int32_t* __restrict__ row_pos,
                           const int64_t* __restrict__ row_item, int64_t n_rows, int64_t n_input, int64_t n_cand,
                           int64_t n_positive, int64_t n_full, int ctx_col0, int rpb /* rows per CTA, <= BWD_ROWS */,
                           const int64_t* __restrict__ event_ts, const int64_t* __restrict__ max_ts,
                           const float* __restrict__ d_out, float* __restrict__ d_gamma, float* __restrict__ d_beta) {
  __shared__ int64_t s_pos[BWD_ROWS], s_item[BWD_ROWS], s_ts[BWD_ROWS];
  __shared__ int s_grp[BWD_ROWS];
  const int64_t r0 = (int64_t)blockIdx.x * rpb;
  const int nr = (int)min((int64_t)rpb, n_rows - r0);
  if (threadIdx.x < nr) {
    const int64_t r = r0 + threadIdx.x;
    const int64_t pos = row_pos[r];
    s_pos[threadIdx.x] = pos;
    s_item[threadIdx.x] = row_item[r];
    s_ts[threadIdx.x] = (r < n_input) ? event_ts[pos] : max_ts[0];
    s_grp[threadIdx.x] = row_group(r, n_input, n_cand, n_positive);
  }
  __syncthreads();
  // rows >= n_full carry item features only: their context columns (>= ctx_col0) hold no gradient
  const int nr_ctx = (int)max((int64_t)0, min((int64_t)nr, n_full - r0));
  for (int c = threadIdx.x; c < P.row_ld; c += BWD_THREADS) {
    const int si = P.col_seg[c];
    if (si == 255) continue;
    const int nr = c >= ctx_col0 ? nr_ctx : (int)min((int64_t)rpb, n_rows - r0);
    const nar_segment& sg = P.seg[si];
    const int j = c - sg.col;
    const float gam = P.gamma[c];
    float acc_b = 0.f, acc_g = 0.f;
    // 4 rows per trip: the 8 loads (dX, re-gathered raw value) are issued before the first atomic - the compiler may
    // not move loads across the atomics itself (they could alias the tables)
    for (int i0 = 0; i0 < nr; i0 += 4) {
      float d[4], raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u;
        d[u] = 0.f; raw[u] = 0.f;
        if (i < nr) {
          d[u] = __ldg(d_out + (r0 + i) * (int64_t)P.row_ld + c);
          raw[u] = seg_value(P, sg, j, s_pos[i], s_item[i], s_ts[i], P.stats + 8 * s_grp[i]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u;
        acc_b += d[u];
        acc_g += d[u] * raw[u];
        if (sg.grad != nullptr && i < nr) {
          int64_t id;
          if (sg.kind == NAR_SEG_ITEM_EMB) id = s_item[i];
          else if (sg.kind == NAR_SEG_CTX_EMBED) id = P.ctx_int[sg.src][s_pos[i]];
          else id = P.meta[sg.src][s_item[i]];
          if (sg.kind != NAR_SEG_ITEM_EMB) id = id < 0 ? 0 : (id >= sg.card ? sg.card - 1 : id);
          atomicAdd(sg.grad + id * (int64_t)sg.ld + j, d[u] * gam);
        }
      }
    }
    atomicAdd(d_beta + c, acc_b);
    atomicAdd(d_gamma + c, acc_g);
  }
}

// ------------------------------------------------------------------ statistics
// single CTA.  Pass A: the first n_norm nonzero buffer entries (order kept).  If the buffer is
// empty: each row group uses its own non-padded rows (first batch only).
constexpr int STATS_THREADS = 1024;

struct Acc { float sum, mn, mx; float cnt; };

__device__ float block_reduce(float v, int op, float* sh) {   // op 0 sum, 1 min, 2 max
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = op == 0 ? warp_sum(v) : (op == 1 ? warp_min(v) : warp_max(v));
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    float x = (lane < (int)(blockDim.x >> 5)) ? sh[lane] : (op == 0 ? 0.f : (op == 1 ? INFINITY : -INFINITY));
    x = op == 0 ? warp_sum(x) : (op == 1 ? warp_min(x) : warp_max(x));
    if (lane == 0) sh[32] = x;
  }
  __syncthreads();
  return sh[32];
}

__global__ void __launch_bounds__(STATS_THREADS)
feature_stats_kernel(const int64_t* __restrict__ buffer, int64_t buf_len, int64_t n_norm,
                     const int64_t* __restrict__ created, const float* __restrict__ pop_norm,
                     const int64_t* __restrict__ max_ts_p, float log_base_rec, float log_base_nov,
                     const int32_t* __restrict__ row_pos, const int64_t* __restrict__ row_item, int64_t n_rows,
                     int64_t n_input, int64_t n_cand, const int64_t* __restrict__ event_ts, float* __restrict__ stats) {
  __shared__ float sh[40];
  __shared__ int s_cnt[STATS_THREADS];
  __shared__ int s_total;
  const int t = threadIdx.x;
  const float ilr = 1.0f / logf(log_base_rec), iln = 1.0f / logf(log_base_nov);
  const int64_t max_ts = max_ts_p[0];
  // contiguous chunk per thread so that ranks follow buffer order
  const int64_t chunk = (buf_len + STATS_THREADS - 1) / STATS_THREADS;
  const int64_t lo = min(buf_len, (int64_t)t * chunk), hi = min(buf_len, lo + chunk);
  int c = 0;
  for (int64_t i = lo; i < hi; ++i) c += buffer[i] != 0;
  s_cnt[t] = c;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int i = 0; i < STATS_THREADS; ++i) { const int x = s_cnt[i]; s_cnt[i] = run; run += x; }
    s_total = run;
  }
  __syncthreads();
  const int total = s_total;
  if (total > 0) {
    const int64_t n_use = min((int64_t)total, n_norm);
    // pass 1: sums
    float sr = 0.f, sn = 0.f, mnr = INFINITY, mxr = -INFINITY, mnn = INFINITY, mxn = -INFINITY;
    int rank = s_cnt[t];
    for (int64_t i = lo; i < hi; ++i) {
      const int64_t id = buffer[i];
      if (id == 0) continue;
      if (rank < n_use) {
        const float a = recency_raw(max_ts, created[id], ilr), b = novelty_raw(pop_norm[id], iln);
        sr += a; sn += b; mnr = fminf(mnr, a); mxr = fmaxf(mxr, a); mnn = fminf(mnn, b); mxn = fmaxf(mxn, b);
      }
      ++rank;
    }
    const float inv_n = 1.0f / (float)n_use;
    const float mean_r = block_reduce(sr, 0, sh) * inv_n;
    const float mean_n = block_reduce(sn, 0, sh) * inv_n;
    const float min_r = block_reduce(mnr, 1, sh), max_r = block_reduce(mxr, 2, sh);
    const float min_n = block_reduce(mnn, 1, sh), max_n = block_reduce(mxn, 2, sh);
    float vr = 0.f, vn = 0.f;
    rank = s_cnt[t];
    for (int64_t i = lo; i < hi; ++i) {
      const int64_t id = buffer[i];
      if (id == 0) continue;
      if (rank < n_use) {
        const float a = recency_raw(max_ts, created[id], ilr) - mean_r, b = novelty_raw(pop_norm[id], iln) - mean_n;
        vr += a * a; vn += b * b;
      }
      ++rank;
    }
    const float var_r = block_reduce(vr, 0, sh) * inv_n, var_n = block_reduce(vn, 0, sh) * inv_n;
    if (t == 0) {
      const float sd_r = sqrtf(var_r + 1e-24f), sd_n = sqrtf(var_n + 1e-24f);
      for (int g = 0; g < 3; ++g) {
        float* s = stats + 8 * g;
        s[0] = mean_r; s[1] = sd_r; s[2] = (min_r - mean_r) / sd_r; s[3] = (max_r - mean_r) / sd_r;
        s[4] = mean_n; s[5] = sd_n; s[6] = (min_n - mean_n) / sd_n; s[7] = (max_n - mean_n) / sd_n;
      }
    }
    return;
  }
  // ---- empty buffer: statistics of each row group over its own non-padded rows
  for (int g = 0; g < 3; ++g) {
    float sr = 0.f, sn = 0.f, mnr = INFINITY, mxr = -INFINITY, mnn = INFINITY, mxn = -INFINITY, cnt = 0.f;
    for (int64_t r = t; r < n_rows; r += STATS_THREADS) {
      if (row_group(r, n_input, n_cand) != g) continue;
      const int64_t id = row_item[r];
      if (id == 0) continue;
      const int64_t ts = (r < n_input) ? event_ts[row_pos[r]] : max_ts;
      const float a = recency_raw(ts, created[id], ilr), b = novelty_raw(pop_norm[id], iln);
      sr += a; sn += b; mnr = fminf(mnr, a); mxr = fmaxf(mxr, a); mnn = fminf(mnn, b); mxn = fmaxf(mxn, b); cnt += 1.f;
    }
    const float n = block_reduce(cnt, 0, sh);
    const float inv_n = n > 0.f ? 1.0f / n : 0.f;
    const float mean_r = block_reduce(sr, 0, sh) * inv_n, mean_n = block_reduce(sn, 0, sh) * inv_n;
    const float min_r = block_reduce(mnr, 1, sh), max_r = block_reduce(mxr, 2, sh);
    const float min_n = block_reduce(mnn, 1, sh), max_n = block_reduce(mxn, 2, sh);
    float vr = 0.f, vn = 0.f;
    for (int64_t r = t; r < n_rows; r += STATS_THREADS) {
      if (row_group(r, n_input, n_cand) != g) continue;
      const int64_t id = row_item[r];
      if (id == 0) continue;
      const int64_t ts = (r < n_input) ? event_ts[row_pos[r]] : max_ts;
      const float a = recency_raw(ts, created[id], ilr) - mean_r, b = novelty_raw(pop_norm[id], iln) - mean_n;
      vr += a * a; vn += b * b;
    }
    const float var_r = block_reduce(vr, 0, sh) * inv_n, var_n = block_reduce(vn, 0, sh) * inv_n;
    if (t == 0) {
      const float sd_r = sqrtf(var_r + 1e-24f), sd_n = sqrtf(var_n + 1e-24f);
      float* s = stats + 8 * g;
      s[0] = mean_r; s[1] = sd_r; s[2] = (min_r - mean_r) / sd_r; s[3] = (max_r - mean_r) / sd_r;
      s[4] = mean_n; s[5] = sd_n; s[6] = (min_n - mean_n) / sd_n; s[7] = (max_n - mean_n) / sd_n;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ plain row gather / scatter-add
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ table, int64_t n_table_rows, int64_t ld, int width,
                   const int64_t* __restrict__ ids, int64_t n, float* __restrict__ out, int64_t ld_out) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= n) return;
  int64_t id = ids[r];
  id = id < 0 ? 0 : (id >= n_table_rows ? n_table_rows - 1 : id);
  const float* src = table + id * ld;
  float* dst = out + r * ld_out;
  const bool vec = ((ld & 3) == 0) && ((ld_out & 3) == 0) && ((reinterpret_cast<uintptr_t>(table) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  int j0 = 0;
  if (vec) {
    const int nv = width >> 2;
    for (int j = lane; j < nv; j += 32) reinterpret_cast<float4*>(dst)[j] = __ldg(reinterpret_cast<const float4*>(src) + j);
    j0 = nv << 2;
  }
  for (int j = j0 + lane; j < width; j += 32) dst[j] = __ldg(src + j);
}

__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(float* __restrict__ table, int64_t n_table_rows, int64_t ld, int width,
                        const int64_t* __restrict__ ids, int64_t n, const float* __restrict__ src, int64_t ld_src) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= n) return;
  int64_t id = ids[r];
  if (id < 0 || id >= n_table_rows) return;
  for (int j = lane; j < width; j += 32) atomicAdd(table + id * ld + j, src[r * ld_src + j]);
}

__global__ void __launch_bounds__(256)
build_rows_kernel(const int32_t* __restrict__ pos_idx, int64_t L, const int64_t* __restrict__ item_clicked,
                  const int64_t* __restrict__ label_next, const int64_t* __restrict__ negatives, int64_t K,
                  int32_t* __restrict__ row_pos, int64_t* __restrict__ row_item) {
  const int64_t n_cand = K + 1;
  const int64_t total = L * (n_cand + 1);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = i / (n_cand + 1), j = i - l * (n_cand + 1);     // j = 0 input, 1 positive, 2.. negatives
    const int32_t pos = pos_idx[l];
    int64_t r, item;
    if (j == 0) { r = l; item = item_clicked[pos]; }
    else if (j == 1) { r = L + l * n_cand; item = label_next[pos]; }
    else { r = L + l * n_cand + (j - 1); item = negatives[(int64_t)pos * K + (j - 2)]; }
    row_pos[r] = pos;
    row_item[r] = item;
  }
}

// Base rows of the per-unique-id CAR layer 1 (engine.cu): [0,L) clicked items, [L,2L) positives, then one row per
// entry of the step's unique-negative table (U = table capacity + 1: unused entries and the last "padding negative"
// slot hold item 0; their context columns are written as 0).
__global__ void __launch_bounds__(256)
build_base_rows_kernel(const int32_t* __restrict__ pos_idx, int64_t L, const int64_t* __restrict__ item_clicked,
                       const int64_t* __restrict__ label_next, const int64_t* __restrict__ uitems,
                       const int32_t* __restrict__ n_unique_p, int64_t U, int32_t* __restrict__ base_pos,
                       int64_t* __restrict__ base_item) {
  const int64_t n_base = 2 * L + U;
  const int n_unique = n_unique_p[0];
  const int32_t pos0 = pos_idx[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_base; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t pos; int64_t item;
    if (i < L) { pos = pos_idx[i]; item = item_clicked[pos]; }
    else if (i < 2 * L) { pos = pos_idx[i - L]; item = label_next[pos]; }
    else { const int64_t u = i - 2 * L; pos = pos0; item = u < n_unique ? uitems[u] : 0; }
    base_pos[i] = pos; base_item[i] = item;
  }
}

}  // namespace feat
}  // namespace nar

extern "C" int nar_build_base_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* label_next_item,
                                   const int64_t* unique_items, const int32_t* n_unique, int64_t U, const int32_t* neg_uidx,
                                   int64_t K, int32_t* base_pos, int64_t* base_item, void* stream) {
  if (!pos_idx || !item_clicked || !label_next_item || !unique_items || !n_unique || !neg_uidx || !base_pos || !base_item)
    return NAR_ERR_INVALID;
  if (K <= 0 || U <= 0) return NAR_ERR_INVALID;
  if (L <= 0) return NAR_OK;
  const int64_t total = 2 * L + U;
  int64_t g = (total + 255) / 256; if (g > NAR_GRID_SMS * 8) g = NAR_GRID_SMS * 8;
  nar::feat::build_base_rows_kernel<<<(unsigned)g, 256, 0, as_stream(stream)>>>(pos_idx, L, item_clicked, label_next_item,
                                                                              unique_items, n_unique, U, base_pos, base_item);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_build_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* label_next_item,
                              const int64_t* negatives, int64_t K, int32_t* row_pos, int64_t* row_item, void* stream) {
  if (!pos_idx || !item_clicked || !label_next_item || !negatives || !row_pos || !row_item || K < 0) return NAR_ERR_INVALID;
  if (L <= 0) return NAR_OK;
  const int64_t total = L * (K + 2);
  int64_t g = (total + 255) / 256; if (g > NAR_GRID_SMS * 8) g = NAR_GRID_SMS * 8;
  nar::feat::build_rows_kernel<<<(unsigned)g, 256, 0, as_stream(stream)>>>(pos_idx, L, item_clicked, label_next_item, negatives, K, row_pos, row_item);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_gather_features(nar_ctx* ctx, const nar_feature_plan* plan, const int32_t* row_pos,
                                   const int64_t* row_item, const nar_row_layout* rows,
                                   const int64_t* event_timestamp, const int64_t* max_ts, float* out, void* stream) {
  if (!ctx || !plan || !row_pos || !row_item || !out || !max_ts || !rows) return NAR_ERR_INVALID;
  const int64_t n_rows = rows->n_rows, n_input = rows->n_input, n_cand = rows->n_cand;
  if (n_cand < 0 || n_input < 0 || rows->n_positive < 0) return NAR_ERR_INVALID;
  if (plan->n_segments > NAR_MAX_SEGMENTS) return NAR_ERR_INVALID;
  if (n_rows <= 0) return NAR_OK;
  if (!ctx || !ctx->gather_desc) return NAR_ERR_INVALID;
  // lane budget of the scalar prefetch (phase A): <= 12 context ids, <= 8 context floats, <= 8 metadata arrays
  int n_ci = 0, n_cf = 0, n_me = 0, n_wide = 0, n_narrow_cols = 0, n_tail = 0, n_vec = 0;
  unsigned meta_num_mask = 0;
  nar::feat::GatherArgs A;
  memset(&A, 0, sizeof(A));
  const float* e_lo = nullptr; const float* e_hi = nullptr;     // address range of the small embedding tables
  for (int i = 0; i < plan->n_segments; ++i) {
    const nar_segment& g = plan->seg[i];
    if (g.kind == NAR_SEG_CTX_OHE || g.kind == NAR_SEG_CTX_EMBED) n_ci = g.src + 1 > n_ci ? g.src + 1 : n_ci;
    if (g.kind == NAR_SEG_CTX_NUM) n_cf = g.src + 1 > n_cf ? g.src + 1 : n_cf;
    if (g.kind == NAR_SEG_META_OHE || g.kind == NAR_SEG_META_EMBED || g.kind == NAR_SEG_META_NUM) n_me = g.src + 1 > n_me ? g.src + 1 : n_me;
    if (g.kind == NAR_SEG_META_NUM && g.src < 32) meta_num_mask |= 1u << g.src;
    if (g.kind == NAR_SEG_ACR || g.kind == NAR_SEG_ITEM_EMB) {
      const bool vec = ((g.col & 3) == 0) && ((g.ld & 3) == 0) && ((plan->row_ld & 3) == 0);
      if (n_wide < 2) {
        A.wtab[n_wide] = g.table; A.wcol[n_wide] = g.col; A.wld[n_wide] = g.ld; A.wnvec[n_wide] = vec ? (g.width >> 2) : 0;
        for (int j = vec ? (g.width & ~3) : 0; j < g.width; ++j, ++n_tail)
          if (n_tail < nar::feat::GATHER_MAX_TAIL) { A.tail_col[n_tail] = (short)(g.col + j); A.tail_seg[n_tail] = (unsigned char)n_wide; A.tail_j[n_tail] = (short)j; }
      }
      ++n_wide;
      n_vec += vec ? (g.width >> 2) : 0;
    }
    if (g.kind == NAR_SEG_CTX_EMBED || g.kind == NAR_SEG_META_EMBED) {
      if (!e_lo || g.table < e_lo) e_lo = g.table;
      const float* end = g.table + (int64_t)g.card * g.ld;
      if (!e_hi || end > e_hi) e_hi = end;
    }
  }
  for (int q = 0; q < plan->n_narrow; ++q) n_narrow_cols += plan->narrow_end[q] - plan->narrow_begin[q];
  if (n_ci > 12 || n_cf > 8 || n_me > 8 || n_wide > 2 || plan->row_ld > NAR_MAX_COLS || plan->row_ld > 0xffff ||
      n_narrow_cols > nar::feat::GATHER_MAX_NARROW || n_tail > nar::feat::GATHER_MAX_TAIL || n_vec > 8 * 32 ||
      n_rows > 0x7fffffffLL / 2 || (e_hi - e_lo) > 0x7fffffffLL ||     // table offsets are 32-bit (one flat parameter buffer)
      (reinterpret_cast<uintptr_t>(plan->gamma) & 15) || (reinterpret_cast<uintptr_t>(plan->beta) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15)) return NAR_ERR_UNSUPPORTED;
  // descriptor table: rebuilt only when the static part of the plan changed (calls sharing a context are stream-ordered)
  {
    nar_feature_plan* key = static_cast<nar_feature_plan*>(ctx->gather_key);
    bool same = ctx->gather_key_valid && key->n_segments == plan->n_segments && key->row_ld == plan->row_ld &&
                key->n_narrow == plan->n_narrow &&
                memcmp(key->seg, plan->seg, sizeof(nar_segment) * plan->n_segments) == 0 &&
                memcmp(key->narrow_begin, plan->narrow_begin, sizeof(plan->narrow_begin)) == 0 &&
                memcmp(key->narrow_end, plan->narrow_end, sizeof(plan->narrow_end)) == 0 &&
                memcmp(key->col_seg, plan->col_seg, plan->row_ld) == 0;
    if (!same) {
      nar::feat::gather_setup_kernel<<<1, 128, 0, as_stream(stream)>>>(*plan, n_narrow_cols, e_lo,
                                                                       static_cast<nar::feat::GatherDesc*>(ctx->gather_desc));
      NAR_LAUNCH_CHECK();
      *key = *plan;
      ctx->gather_key_valid = 1;
    }
  }
  for (int l = 0; l < 32; ++l) {
    const void* p = nullptr; int mode = nar::feat::SM_NONE;
    if (l < nar::feat::LANE_CTX_FLOAT) { if (l < n_ci) { p = plan->ctx_int[l]; mode = nar::feat::SM_ID_AT_POS; } }
    else if (l < nar::feat::LANE_META) { if (l - nar::feat::LANE_CTX_FLOAT < n_cf) { p = plan->ctx_float[l - nar::feat::LANE_CTX_FLOAT]; mode = nar::feat::SM_FLOAT_AT_POS; } }
    else if (l < nar::feat::LANE_RECENCY) {
      const int m = l - nar::feat::LANE_META;
      if (m < n_me) { p = plan->meta[m]; mode = ((meta_num_mask >> m) & 1u) ? nar::feat::SM_NUM_AT_ITEM : nar::feat::SM_ID_AT_ITEM; }
    }
    A.src[l] = p; A.mode[l] = (unsigned char)(p ? mode : nar::feat::SM_NONE);
  }
  A.gamma = plan->gamma; A.beta = plan->beta; A.stats = plan->stats;
  A.created_at_ts = plan->created_at_ts; A.pop_norm = plan->pop_norm;
  A.log_base_recency = plan->log_base_recency; A.log_base_novelty = plan->log_base_novelty;
  A.row_ld = plan->row_ld;
  A.ebase = e_lo; A.ntail = n_tail;
  A.n_positive = (int)rows->n_positive;
  A.n_full = rows->n_full < n_rows ? (int)(rows->n_full < 0 ? 0 : rows->n_full) : (int)n_rows;
  A.ctx_col0 = (int)rows->ctx_col0;
  const nar::feat::GatherDesc* D = static_cast<const nar::feat::GatherDesc*>(ctx->gather_desc);
  // narrow CTAs first (longer running): one warp per (chunk of 8 rows, 32 columns); then one wide CTA per 8 rows
  const int64_t n_chunks = (n_rows + nar::feat::GATHER_CHUNK - 1) / nar::feat::GATHER_CHUNK;
  A.n_col_groups = (n_narrow_cols + 31) / 32;
  const int64_t nb = (n_chunks * A.n_col_groups + nar::feat::GATHER_WARPS - 1) / nar::feat::GATHER_WARPS;
  A.n_narrow_blocks = (int)nb;
  const int64_t wb = (n_vec > 0 || n_tail > 0) ? (n_rows + nar::feat::GATHER_WARPS - 1) / nar::feat::GATHER_WARPS : 0;
  const unsigned grid = (unsigned)(nb + wb);
  if (grid == 0) return NAR_OK;
  A.period = nb > 0 ? (int)((nb + wb) / nb) : 1;
  const int wu = (n_vec + 31) / 32;
#define NAR_GATHER_LAUNCH(WU)                                                                                     \
  nar::feat::gather_features_kernel<WU><<<grid, nar::feat::GATHER_WARPS * 32, 0, as_stream(stream)>>>(            \
      A, D, row_pos, row_item, (int)n_rows, (int)n_input, (int)n_cand, event_timestamp, max_ts, out)
  if (wu <= 1) NAR_GATHER_LAUNCH(1); else if (wu == 2) NAR_GATHER_LAUNCH(2); else if (wu == 3) NAR_GATHER_LAUNCH(3);
  else if (wu == 4) NAR_GATHER_LAUNCH(4); else if (wu <= 6) NAR_GATHER_LAUNCH(6); else NAR_GATHER_LAUNCH(8);   // up to 1024 wide floats per row
#undef NAR_GATHER_LAUNCH
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_gather_features_bwd(nar_ctx* ctx, const nar_feature_plan* plan, const int32_t* row_pos,
                                       const int64_t* row_item, const nar_row_layout* rows,
                                       const int64_t* event_timestamp, const int64_t* max_ts, const float* d_out,
                                       float* d_gamma, float* d_beta, void* stream) {
  if (!ctx || !plan || !row_pos || !row_item || !d_out || !d_gamma || !d_beta || !rows) return NAR_ERR_INVALID;
  const int64_t n_rows = rows->n_rows, n_input = rows->n_input, n_cand = rows->n_cand;
  if (n_rows <= 0) return NAR_OK;
  const int64_t n_full = rows->n_full < n_rows ? (rows->n_full < 0 ? 0 : rows->n_full) : n_rows;
  // rows per CTA: 32 for long row lists; fewer when that would leave most SMs idle (the per-unique-id base rows of a
  // step are ~2 K rows: 32 rows per CTA = 61 CTAs measured 65 us, latency bound)
  int rpb = (int)(n_rows / (4 * (int64_t)ctx->sm_count));
  rpb = rpb < 4 ? 4 : (rpb > nar::feat::BWD_ROWS ? nar::feat::BWD_ROWS : rpb);
  const unsigned grid = (unsigned)((n_rows + rpb - 1) / rpb);
  nar::feat::gather_features_bwd_kernel<<<grid, nar::feat::BWD_THREADS, 0, as_stream(stream)>>>(
      *plan, row_pos, row_item, n_rows, n_input, n_cand, rows->n_positive, n_full, (int)rows->ctx_col0, rpb, event_timestamp, max_ts,
      d_out, d_gamma, d_beta);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_feature_stats(nar_ctx* ctx, const int64_t* buffer, int64_t buf_len, int64_t n_norm,
                                 const int64_t* created_at_ts, const float* pop_norm, const int64_t* max_ts,
                                 float log_base_recency, float log_base_novelty, const int32_t* row_pos,
                                 const int64_t* row_item, int64_t n_rows, int64_t n_input, int64_t n_cand,
                                 const int64_t* event_timestamp, float* stats, void* stream) {
  if (!ctx || !buffer || !created_at_ts || !pop_norm || !max_ts || !stats) return NAR_ERR_INVALID;
  nar::feat::feature_stats_kernel<<<1, nar::feat::STATS_THREADS, 0, as_stream(stream)>>>(
      buffer, buf_len, n_norm, created_at_ts, pop_norm, max_ts, log_base_recency, log_base_novelty, row_pos,
      row_item, n_rows, n_input, n_cand, event_timestamp, stats);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_gather_rows_f32(const float* table, int64_t n_table_rows, int64_t ld, int width,
                                   const int64_t* ids, int64_t n, float* out, int64_t ld_out, void* stream) {
  if (!table || !ids || !out) return NAR_ERR_INVALID;
  if (n <= 0) return NAR_OK;
  nar::feat::gather_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, as_stream(stream)>>>(table, n_table_rows, ld, width, ids, n, out, ld_out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_scatter_add_rows_f32(float* table, int64_t n_table_rows, int64_t ld, int width,
                                        const int64_t* ids, int64_t n, const float* src, int64_t ld_src, void* stream) {
  if (!table || !ids || !src) return NAR_ERR_INVALID;
  if (n <= 0) return NAR_OK;
  nar::feat::scatter_add_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, as_stream(stream)>>>(table, n_table_rows, ld, width, ids, n, src, ld_src);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
