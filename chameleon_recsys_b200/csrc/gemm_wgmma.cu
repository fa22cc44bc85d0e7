// TMA-fed wgmma GEMM (sm_90a) with fused epilogues for the NAR dense layers.
//
//   D[M,N] = epilogue( sum_k A(m,k) * B(n,k) )
//
// Replaces every tf.layers.Dense of the reference graph (nar_model.py:375-473) and the UGRNN
// input projection (:1317); forward, dgrad and wgrad all go through this one kernel by
// choosing operand majors (no transposed copies of activations are ever made):
//   fwd   Y  = X  * W        A = X  (K-major)   B = W   (MN-major: W is [in,out]) or W^T (K-major)
//   dgrad dX = dY * W^T      A = dY (K-major)   B = W   (K-major)
//   wgrad dW = X^T * dY      A = X  (MN-major)  B = dY  (MN-major), split-K + red.add
//
// CTA = 256 threads = two warpgroups, one 128 x 128 output tile, k-tiles of 32 (32 fp32 = one 128-byte swizzle row);
// two CTAs per SM unless B needs separate 3xTF32 split tiles (see Cfg), else one:
//   thread 0     keeps STAGES - 1 k-tiles of A and B ahead of the one being multiplied (cp.async.bulk.tensor.2d,
//                128-byte swizzle, one mbarrier per stage) and refills a stage as soon as its MMAs are done;
//   warpgroup w  multiplies rows [64w, 64w + 64) of the tile with wgmma.m64n128: A from registers, B from shared
//                memory.  A is read from the swizzled TMA tile straight into the register fragment whatever its major,
//                and that is also where 3xTF32 splits it.  wgmma reads 32-bit B operands only K-major, so a B tile that
//                arrives MN-major (the forward weights W [in,out], the wgrad dY) is first transposed in shared memory
//                by all 256 threads: in place for single-pass TF32, into separate tiles for 3xTF32, where the same
//                pass writes B's lo part.
//   epilogue     accumulators -> shared memory -> row-contiguous bias / activation / activation-derivative and
//                st.global.v4, or red.global.add.v4 for split-K.
//
// 3xTF32: hi = x with the low 13 mantissa bits cleared, lo = x - hi; D += Alo*Bhi + Ahi*Blo + Ahi*Bhi restores ~fp32
// accuracy (the reference is fp32 end to end and logits are divided by temperature 0.1 before exp).
//   MODE 0: single pass.   MODE 1: 3x, B_lo computed in-kernel.   MODE 2: 3x, B_lo read from HBM (nar_adam_tf keeps it).
//   MODE 4: bf16x3 - the same error compensation with bf16 pieces on the bf16 tensor path, which runs at twice the tf32
//           rate: x = hi + lo with hi = bf16(x), lo = bf16(x - hi) (16 mantissa bits kept).  A: fp32 K-major tile by
//           TMA, split in registers.  B: a pre-split, TRANSPOSED bf16 plane maintained next to the weights
//           (nar_pack_bf16x3): row n holds, per block of 32 k, the 32 hi values followed by the 32 lo values = one
//           128-byte swizzle row, so ONE K-major TMA box brings both halves and no transpose pass is needed.
// The scorer's product PD = Ec * PR[position] (nar_model.py:478, :493) never reaches HBM: its Dense layer's forward and
// weight gradient scale A by PR where the fragment is built (EXT_SCALE_*), and its dgrad derives dEc and dPR in an
// epilogue over position-aligned M tiles (EXT_PROD_BWD), optionally with the column sums of dEc (the gradient of the
// bias of the layer that produced Ec).
#include "common.cuh"
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

namespace nar {
namespace gemm {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 32;                       // 32 fp32 = 128 B = one 128-byte swizzle span
constexpr int TILE_BYTES = 128 * BK * 4;     // one 128 x 32 fp32 operand tile (= one 128 x 64 bf16 plane tile)
constexpr int NUM_THREADS = 256;
constexpr int EPI_LD = BN + 4;               // floats per staged accumulator row (16-byte aligned rows)

// Extensions of the plain GEMM (template parameter EXT of the kernel; 0 = none):
//   EXT_SCALE_SMEM  A scale (nar_gemm_epilogue.a_scale), its slice for the k-tile staged by TMA with the stage: a K-major
//                   A needs the scale rows of the tile's row groups (at most SC_ROWS_K) x 32 k, an MN-major A those of
//                   the k-tile's k groups (at most SC_ROWS_MN) x 128 m; SC_BYTES per stage either way
//   EXT_SCALE_GMEM  A scale read from global memory at the fragment: any group size (those whose slices do not fit)
//   EXT_PROD_BWD    scorer-product backward epilogue (nar_gemm_epilogue.pred, .d_bias): position-aligned M tiles
//   EXT_CAR_BWD     CAR layer-1 backward epilogue (nar_gemm_epilogue.car_*): the gradients of PP / PC / PI, no D
//                   (TF32 or 3xTF32 with B split in-kernel, K-major operands)
//   EXT_TRANS_D     D written transposed, D[n * ldd + m] (nar_gemm_tf32_dt): a weight gradient computed as
//                   dW^T = dY^T * X, A = dY MN-major and B = X^T K-major, lands in dW [in, out] with no prep pass on B
constexpr int EXT_SCALE_SMEM = 1, EXT_SCALE_GMEM = 2, EXT_PROD_BWD = 3, EXT_CAR_BWD = 4, EXT_TRANS_D = 5;
constexpr int SC_ROWS_K = 32, SC_ROWS_MN = 8;
constexpr int SC_BYTES = 4096;
static_assert(SC_ROWS_K * BK * 4 == SC_BYTES && SC_ROWS_MN * BM * 4 == SC_BYTES, "a_scale slice per stage");

template <int MODE, bool B_MN, int SC = 0> struct Cfg {                // SC: bytes of a_scale slice per stage
  static constexpr bool SPLIT3 = MODE == 1 || MODE == 2;
  static constexpr bool BLO = MODE == 2;
  static constexpr bool PREP = B_MN || SPLIT3;                        // B goes through the transpose / split pass
  // MODE 0 transposes an MN-major B within its own stage (prep_b); only the 3xTF32 split writes separate prep tiles
  static constexpr bool PREP_TILES = SPLIT3;
  static constexpr int STAGE_BYTES = TILE_BYTES * (BLO ? 3 : 2);      // A | B [| B_lo]
  // Without prep tiles two CTAs share an SM (3 stages = 96 KB each, <= 128 registers per thread), so that one CTA's
  // epilogue runs under the other's main loop; with them, there is room for one CTA.
  static constexpr int CTAS_PER_SM = PREP_TILES ? 1 : 2;
  static constexpr int STAGES = (BLO || !PREP_TILES) ? 3 : 4;
  static constexpr int PREP_TILE_BYTES = PREP_TILES ? TILE_BYTES * 2 : 0;   // K-major B_hi | B_lo
  static constexpr int PREP_BYTES = 2 * PREP_TILE_BYTES;             // double-buffered: k-tile kt uses buffer kt & 1
  static constexpr int SC_OFF = STAGES * STAGE_BYTES + PREP_BYTES;    // [STAGES] a_scale slices
  static constexpr int BAR_OFF = SC_OFF + STAGES * SC;
  static constexpr int SMEM_BYTES = BAR_OFF + 64 + 1024;              // + barriers + alignment slack
  static_assert(STAGES * STAGE_BYTES >= BM * EPI_LD * 4, "the epilogue stages the accumulators in the operand ring");
  static_assert(SMEM_BYTES <= 227 * 1024, "227 KB of shared memory per block");
  static_assert(CTAS_PER_SM * (SMEM_BYTES + 1024) <= 228 * 1024, "228 KB of shared memory per SM (1 KB reserved per block)");
};

struct Params {
  int64_t M, N, K;
  float* D; int64_t ldd;
  const float* bias;
  const float* aux; int64_t ld_aux;
  int act, dact, accumulate;
  int k_tiles_per_split;
  int n_tiles;                 // blockIdx.x = m_blk * n_tiles + n_blk (N fastest: CTAs sharing an A tile run together)
  // A scale (EXT_SCALE_*): A's storage is [a_rows, a_cols]; storage row i uses scale row i / group
  const float* a_scale; int64_t ld_a_scale, a_rows, a_cols; uint32_t group;
  // EXT_PROD_BWD: M tile m_blk = positions [m_blk * pos_per_tile, ...), `group` rows each, n_pos positions in all;
  // d_bias (optional): += the column sums of D
  const float* pred; float* d_pred; float* d_bias; int64_t ld_pred, n_pos; int pos_per_tile;
  // EXT_CAR_BWD: row r = slot r % (car_k + 1) of position r / (car_k + 1); [L | L | U, ld_car] pre-activation parts and
  // their gradients
  const float *car_pp, *car_pc, *car_pi; const int32_t *car_pos_idx, *car_neg_uidx;
  float *car_dpp, *car_dpc, *car_dpi; int64_t ld_car; int car_k;
};

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
  // bounded spin: a protocol bug traps (launch error) instead of hanging the GPU
  for (uint32_t it = 0; it < (1u << 26); ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    if (ok) return;
  }
  __trap();
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// waits until at most N committed groups of this warpgroup's MMAs are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] += A[64 x 8] (registers, tf32) * B[128 x 8] (shared memory, K-major)
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}
// D[64 x 128] += A[64 x 16] (registers, bf16 pairs) * B[128 x 16] (shared memory, K-major)
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}

// wgmma shared-memory descriptor: [0,14) start>>4, [16,30) LBO>>4 (unused for swizzled K-major), [32,46) SBO>>4,
// [62,64) layout (1 = 128-byte swizzle).  K-major tile of 128-byte rows, 8-row atoms 1024 B apart; stepping k within
// the row adds the byte offset to the start address (tiles are 1024-byte aligned, so the swizzle phase is right).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ uint32_t tf32_hi_bits(uint32_t x) { return x & 0xFFFFE000u; }

// x -> (bf16(x), bf16(x - bf16(x))) for two consecutive k values, each pair packed low = even k
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Byte offset of element (mn, k) in a 128 x 32 fp32 operand tile as TMA wrote it with the 128-byte swizzle:
//   K-major:  one box of 128 rows x 128 B, 16-byte chunk c of row r at chunk c ^ (r & 7)
//   MN-major: four boxes of 32 k-rows x 32 MN (4096 B each), chunk c of k-row k at chunk c ^ (k & 7)
template <bool MN_MAJOR>
__device__ __forceinline__ uint32_t tile_off(int mn, int k) {
  return MN_MAJOR ? (uint32_t)((mn >> 5) * 4096 + k * 128 + ((((mn >> 2) & 7) ^ (k & 7)) << 4) + (mn & 3) * 4)
                  : (uint32_t)(mn * 128 + (((k >> 2) ^ (mn & 7)) << 4) + (k & 3) * 4);
}

// B tile of the current stage -> K-major swizzled B_hi [| B_lo] tiles that wgmma reads.  MODE 0 passes hi_out == b and
// transposes in place.
template <bool B_MN, int MODE>
__device__ __forceinline__ void prep_b(const uint8_t* b, const uint8_t* blo, uint8_t* hi_out, uint8_t* lo_out, int tid) {
  constexpr bool SPLIT3 = MODE == 1 || MODE == 2;
  if (B_MN) {
    // thread = a block of 4 n x 4 k: four 16-byte reads along n (one per k), four 16-byte writes along k (one per n);
    // both sides are 8 distinct 16-byte chunks per 8 lanes, i.e. free of bank conflicts.  Box `box` (n in
    // [32 box, 32 box + 32)) is the same 4096 bytes in both layouts and only warps 2 box and 2 box + 1 touch it.
    const int c = tid & 7, kq = (tid >> 3) & 7, box = tid >> 6;
    // k = 4 kq + i and n = 32 box + 4 c + q have (k & 7) = 4 (kq & 1) ^ i and (n & 7) = 4 (c & 1) ^ q, so each side is
    // one base offset with i (q) XORed into the chunk and added to the row: two live registers instead of eight
    const uint32_t rd = (uint32_t)(box * 4096 + kq * 512 + ((c ^ ((kq & 1) << 2)) << 4));
    const uint32_t wr = (uint32_t)(box * 4096 + c * 512 + ((kq ^ ((c & 1) << 2)) << 4));
    float v[4][4], l[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t off = (rd ^ (i << 4)) + i * 128;
      const float4 x = *reinterpret_cast<const float4*>(b + off);
      v[i][0] = x.x; v[i][1] = x.y; v[i][2] = x.z; v[i][3] = x.w;
      if (MODE == 2) {
        const float4 y = *reinterpret_cast<const float4*>(blo + off);
        l[i][0] = y.x; l[i][1] = y.y; l[i][2] = y.z; l[i][3] = y.w;
      }
    }
    // in place: the box's two warps have read all of it before either overwrites it.  Warpgroup w (boxes 2w, 2w + 1)
    // meets at named barrier 1 + w; immediate ids, so that ptxas reserves 3 barriers rather than all 16, and a per-box
    // barrier (a 4-way branch) costs spills at 128 registers.
    if (!SPLIT3) {
      if (tid < 128) asm volatile("bar.sync 1, 128;" ::: "memory");
      else asm volatile("bar.sync 2, 128;" ::: "memory");
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t off = (wr ^ (q << 4)) + q * 128;
      float4 h = make_float4(v[0][q], v[1][q], v[2][q], v[3][q]);
      if (SPLIT3) {
        const float4 x = h;
        h.x = __uint_as_float(tf32_hi_bits(__float_as_uint(x.x))); h.y = __uint_as_float(tf32_hi_bits(__float_as_uint(x.y)));
        h.z = __uint_as_float(tf32_hi_bits(__float_as_uint(x.z))); h.w = __uint_as_float(tf32_hi_bits(__float_as_uint(x.w)));
        const float4 lo = MODE == 2 ? make_float4(l[0][q], l[1][q], l[2][q], l[3][q])
                                    : make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
        *reinterpret_cast<float4*>(lo_out + off) = lo;
      }
      *reinterpret_cast<float4*>(hi_out + off) = h;
    }
  } else {
    // K-major already: same layout, element-wise split
#pragma unroll
    for (int i = 0; i < TILE_BYTES / 16 / NUM_THREADS; ++i) {
      const uint32_t off = (uint32_t)((tid + i * NUM_THREADS) * 16);
      const float4 x = *reinterpret_cast<const float4*>(b + off);
      float4 h;
      h.x = __uint_as_float(tf32_hi_bits(__float_as_uint(x.x))); h.y = __uint_as_float(tf32_hi_bits(__float_as_uint(x.y)));
      h.z = __uint_as_float(tf32_hi_bits(__float_as_uint(x.z))); h.w = __uint_as_float(tf32_hi_bits(__float_as_uint(x.w)));
      const float4 lo = MODE == 2 ? *reinterpret_cast<const float4*>(blo + off)
                                  : make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
      *reinterpret_cast<float4*>(hi_out + off) = h;
      *reinterpret_cast<float4*>(lo_out + off) = lo;
    }
  }
}

// Epilogue element work for 4 consecutive columns of one row: bias / activation / activation-derivative / store.
__device__ __forceinline__ void epilogue_store4(const Params& p, float4 v, int64_t row, int64_t col, const float4& a) {
  float* d = p.D + row * p.ldd + col;
  if (col + 4 <= p.N) {
    if (p.bias) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col));
      v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    }
    if (p.act) { v.x = apply_act(v.x, p.act); v.y = apply_act(v.y, p.act); v.z = apply_act(v.z, p.act); v.w = apply_act(v.w, p.act); }
    if (p.dact) {        // `a` = aux[row, col..col+3], loaded by the caller
      v.x *= act_grad_from_output(a.x, p.dact); v.y *= act_grad_from_output(a.y, p.dact);
      v.z *= act_grad_from_output(a.z, p.dact); v.w *= act_grad_from_output(a.w, p.dact);
    }
    if (p.accumulate) atomicAdd(reinterpret_cast<float4*>(d), v);        // red.global.add.v4.f32
    else *reinterpret_cast<float4*>(d) = v;
  } else {
    const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (col + j < p.N) {
        float x = e[j];
        if (p.bias) x += p.bias[col + j];
        x = apply_act(x, p.act);
        if (p.dact) x *= act_grad_from_output(p.aux[row * p.ld_aux + col + j], p.dact);
        if (p.accumulate) atomicAdd(d + j, x); else d[j] = x;
      }
    }
  }
}

// A scale of the element A's storage holds at (row i, column j), read from global memory (EXT_SCALE_GMEM); 0 outside A,
// where TMA has filled the tile with zeros
// (A's storage rows fit in 31 bits when it is scaled)
__device__ __forceinline__ float scale_gmem(const Params& p, int i, int j) {
  return (i < p.a_rows && j < p.a_cols) ? __ldg(p.a_scale + (int64_t)((uint32_t)i / p.group) * p.ld_a_scale + j) : 0.f;
}
// EXT_SCALE_GMEM: the stage's A tile scaled in place, one 16-byte chunk (4 elements along the storage row) at a time, before
// its fragments are read; the same single multiply as EXT_SCALE_SMEM applies in registers
template <bool A_MN>
__device__ __forceinline__ void scale_tile_gmem(uint8_t* sa, const Params& p, int m0, int k_elem, int tid) {
#pragma unroll 1
  for (int c = tid; c < TILE_BYTES / 16; c += NUM_THREADS) {
    int row, col;                     // storage position of the chunk's first element (see tile_off)
    if (A_MN) { const int kr = (c >> 3) & 31; row = k_elem + kr; col = m0 + (c >> 8) * 32 + (((c & 7) ^ (kr & 7)) << 2); }
    else { const int r = c >> 3; row = m0 + r; col = k_elem + (((c & 7) ^ (r & 7)) << 2); }
    float4* x = reinterpret_cast<float4*>(sa + c * 16);
    float4 v = *x;
    v.x = __fmul_rn(v.x, scale_gmem(p, row, col)); v.y = __fmul_rn(v.y, scale_gmem(p, row, col + 1));
    v.z = __fmul_rn(v.z, scale_gmem(p, row, col + 2)); v.w = __fmul_rn(v.w, scale_gmem(p, row, col + 3));
    *x = v;
  }
}
__device__ __forceinline__ float2 ld_shared_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// four consecutive floats of a row, `nc` of them valid (zeros past them): one 16-byte load when the row is aligned
__device__ __forceinline__ float4 load4(const float* q, int nc, bool v4) {
  if (v4 && nc == 4) return *reinterpret_cast<const float4*>(q);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (nc > 0) v.x = q[0];
  if (nc > 1) v.y = q[1];
  if (nc > 2) v.z = q[2];
  if (nc > 3) v.w = q[3];
  return v;
}
// (a float4 store next to the scalar stores of a partial group is split into four by the compiler)
__device__ __forceinline__ void st_global_v4(float* q, const float4& v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(q), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// EXT_PROD_BWD epilogue: `stage` holds v = dL/d(prod) of the tile's rows.  EC_ROWS rows of Ec fit behind it in the
// operand ring, so the tile is processed in chunks of whole positions (or, for a position longer than EC_ROWS, in
// chunks of one position's rows), each in two phases:
//   elementwise  thread = (row, 4 columns), all rows of the chunk in flight at once: dEc = v * pr * act'(Ec) with
//                16-byte loads and stores, Ec copied into shared memory, and dEc added to the thread's column sums;
//   chain        thread = (position, column): d_pred = fmaf(v, Ec, d_pred) over the position's rows in row order from
//                shared memory - the same chain as nar_mul_pred_bwd's (carried across chunks in `chain`).
// d_bias: the eight warps' column sums (each over its rows in order) added in a fixed tree, one red.add per column.
template <int EC_ROWS>
__device__ __forceinline__ void prod_bwd_epilogue(const Params& p, float* stage, int m_blk, int n_blk, int tid) {
  constexpr int RQ = (EC_ROWS + 7) / 8;                       // rows per thread and chunk
  static_assert(EC_ROWS >= 8, "the eight warps' column sums reuse the Ec rows");
  const int g = (int)p.group;
  const int64_t pos0 = (int64_t)m_blk * p.pos_per_tile, row0 = pos0 * g;
  const int n_pos = (int)min((int64_t)p.pos_per_tile, p.n_pos - pos0);
  const int warp = tid >> 5, c4 = (tid & 31) * 4;
  const int64_t col = (int64_t)n_blk * BN + c4;
  const int nc = (int)min((int64_t)4, p.N - col);             // valid columns of the thread's group (<= 0: none)
  const bool aux_v4 = ((reinterpret_cast<uintptr_t>(p.aux) | (uintptr_t)p.ld_aux * 4) & 15) == 0;
  const bool pred_v4 = ((reinterpret_cast<uintptr_t>(p.pred) | (uintptr_t)p.ld_pred * 4) & 15) == 0;
  float* ec = stage + BM * EPI_LD;                            // [EC_ROWS, BN]: Ec of the chunk's rows
  const int pc = g <= EC_ROWS ? EC_ROWS / g : 1;              // positions per chunk
  float4 bsum = make_float4(0.f, 0.f, 0.f, 0.f);
  float chain = 0.f;
  for (int pb = 0; pb < n_pos; pb += pc) {
    const int np = min(pc, n_pos - pb), pr_end = (pb + np) * g;
    for (int r0 = pb * g; r0 < pr_end; r0 += EC_ROWS) {       // chunk: tile rows [r0, r1)
      const int r1 = min(r0 + EC_ROWS, pr_end);
      if (nc > 0) {
        float4 ev[RQ], pv[RQ];
#pragma unroll
        for (int q = 0; q < RQ; ++q) {
          const int r = r0 + warp + 8 * q;
          if (r < r1) {
            ev[q] = load4(p.aux + (row0 + r) * p.ld_aux + col, nc, aux_v4);
            pv[q] = load4(p.pred + (pos0 + r / g) * p.ld_pred + col, nc, pred_v4);
          }
        }
#pragma unroll
        for (int q = 0; q < RQ; ++q) {
          const int r = r0 + warp + 8 * q;
          if (r < r1) {
            const float4 x = *reinterpret_cast<const float4*>(stage + r * EPI_LD + c4);
            const float4 e = ev[q], pr = pv[q];
            const float4 d = make_float4(x.x * pr.x * act_grad_from_output(e.x, p.dact), x.y * pr.y * act_grad_from_output(e.y, p.dact),
                                         x.z * pr.z * act_grad_from_output(e.z, p.dact), x.w * pr.w * act_grad_from_output(e.w, p.dact));
            float* dst = p.D + (row0 + r) * p.ldd + col;
            if (nc == 4) {
              st_global_v4(dst, d);
            } else {
              dst[0] = d.x;
              if (nc > 1) dst[1] = d.y;
              if (nc > 2) dst[2] = d.z;
            }
            *reinterpret_cast<float4*>(ec + (r - r0) * BN + c4) = e;
            bsum.x += d.x; bsum.y += d.y; bsum.z += d.z; bsum.w += d.w;
          }
        }
      }
      __syncthreads();                // the chain reads other threads' rows of Ec
      for (int idx = tid; idx < np * BN; idx += NUM_THREADS) {
        const int pl = pb + idx / BN, c = idx % BN;
        const int64_t colc = (int64_t)n_blk * BN + c;
        if (colc >= p.N) continue;
        const int beg = max(pl * g, r0), end = min((pl + 1) * g, r1);
        float acc = beg == pl * g ? 0.f : chain;
#pragma unroll 8
        for (int r = beg; r < end; ++r) acc = fmaf(stage[r * EPI_LD + c], ec[(r - r0) * BN + c], acc);
        if (end == (pl + 1) * g) p.d_pred[(pos0 + pl) * p.ld_pred + colc] = acc;
        else chain = acc;             // only when g > EC_ROWS: one position per chunk, thread = column
      }
      __syncthreads();                // the next chunk overwrites Ec
    }
  }
  if (p.d_bias) {
    float* part = ec;                 // [8 warps, BN]
    *reinterpret_cast<float4*>(part + warp * BN + c4) = bsum;
    __syncthreads();
    if (tid < BN && (int64_t)n_blk * BN + tid < p.N) {
      const float* s = part + tid;
      const float t = ((s[0] + s[BN]) + (s[2 * BN] + s[3 * BN])) + ((s[4 * BN] + s[5 * BN]) + (s[6 * BN] + s[7 * BN]));
      atomicAdd(p.d_bias + (int64_t)n_blk * BN + tid, t);      // red.global.add.f32
    }
  }
}

// EXT_CAR_BWD row of the tile (thread tid < BM): its position l (-1 past M) and the unique-table index u of a negative
// (slot j >= 1; -1 for the positive).  Loaded before the main loop, so that the two dependent index loads complete under
// it; the epilogue reads them from shared memory (s_l / s_u).
__device__ __forceinline__ void car_bwd_row(const Params& p, int m0, int tid, int32_t& l, int32_t& u) {
  l = -1; u = -1;
  const int row = m0 + tid, n_cand = p.car_k + 1;
  if (tid >= BM || row >= p.M) return;
  l = row / n_cand;
  const int j = row - l * n_cand;
  if (j > 0) u = __ldg(p.car_neg_uidx + (int64_t)__ldg(p.car_pos_idx + l) * p.car_k + j - 1);
}

// EXT_CAR_BWD epilogue: `stage` holds v = dL/dH1 of the tile's rows, H1 = act(pre) with pre = PP[l] for the positive and
// PC[l] + PI[u] for a negative - the same fp32 add of the same operands as car_combine_kernel, so act'(pre) is bit for
// bit the factor the plain dgrad takes from H1.  g = v * act'(pre):
//   positive   dPP[l] = g (the row's only writer)
//   negative   dPI[u] += g (red.add: a popular u is drawn by many positions), and g stays in `stage` for
//   dPC[l] += the sum of the tile's negative rows of l in ascending row order, one red.add per (position, column).  With
//              1 + K <= 128 a position's rows lie in at most two M tiles, so dPC gets at most two adds onto zero and is
//              bit-reproducible (commutative); dPI is not (float atomics in launch order).
__device__ __forceinline__ void car_bwd_epilogue(const Params& p, float* stage, const int32_t* s_l, const int32_t* s_u, int m0,
                                                 int n_blk, int tid) {
  constexpr int RB = 8;               // rows per batch: their L2 gathers are all in flight before the dependent arithmetic
  const int warp = tid >> 5, c4 = (tid & 31) * 4;
  const int64_t col = (int64_t)n_blk * BN + c4;
  const int64_t ld = p.ld_car;
  if (col < p.N) {                    // N % 4 == 0 (host checks)
#pragma unroll 1
    for (int it0 = 0; it0 < BM / 8; it0 += RB) {
      float4 a[RB], b[RB];
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        const int rl = (it0 + q) * 8 + warp;
        const int l = s_l[rl], u = s_u[rl];
        if (l < 0) continue;
        if (u < 0) {
          a[q] = __ldg(reinterpret_cast<const float4*>(p.car_pp + l * ld + col));
        } else {
          a[q] = __ldg(reinterpret_cast<const float4*>(p.car_pi + u * ld + col));
          b[q] = __ldg(reinterpret_cast<const float4*>(p.car_pc + l * ld + col));
        }
      }
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        const int rl = (it0 + q) * 8 + warp;
        const int l = s_l[rl], u = s_u[rl];
        if (l < 0) continue;
        const float4 pre = u < 0 ? a[q] : make_float4(a[q].x + b[q].x, a[q].y + b[q].y, a[q].z + b[q].z, a[q].w + b[q].w);
        float4* sv = reinterpret_cast<float4*>(stage + rl * EPI_LD + c4);
        float4 g = *sv;
        g.x *= act_grad_from_output(apply_act(pre.x, p.dact), p.dact);
        g.y *= act_grad_from_output(apply_act(pre.y, p.dact), p.dact);
        g.z *= act_grad_from_output(apply_act(pre.z, p.dact), p.dact);
        g.w *= act_grad_from_output(apply_act(pre.w, p.dact), p.dact);
        if (u < 0) {
          *reinterpret_cast<float4*>(p.car_dpp + l * ld + col) = g;
        } else {
          atomicAdd(reinterpret_cast<float4*>(p.car_dpi + u * ld + col), g);     // red.global.add.v4.f32
          *sv = g;
        }
      }
    }
  }
  __syncthreads();                    // the per-position sums read other warps' rows of `stage`
  const int n_cand = p.car_k + 1;
  const int last = (int)min((int64_t)m0 + BM, p.M) - 1, l0 = m0 / n_cand;
  const int n_pos = last / n_cand - l0 + 1;
  for (int idx = tid; idx < n_pos * BN; idx += NUM_THREADS) {
    const int c = idx % BN, l = l0 + idx / BN;
    const int64_t colc = (int64_t)n_blk * BN + c;
    const int r_beg = max(l * n_cand + 1, m0), r_end = min((l + 1) * n_cand, last + 1);
    if (colc >= p.N || r_beg >= r_end) continue;
    const float* v = stage + (r_beg - m0) * EPI_LD + c;
    float acc = v[0];
#pragma unroll 8
    for (int r = 1; r < r_end - r_beg; ++r) acc += v[r * EPI_LD];
    atomicAdd(p.car_dpc + l * ld + colc, acc);
  }
}

// TMA for one 128 x 32 fp32 operand tile at MN coordinate mn0, K element k_elem
template <bool MN_MAJOR>
__device__ __forceinline__ void load_operand(uint32_t dst, const CUtensorMap* map, uint64_t* bar, int mn0, int k_elem) {
  if (!MN_MAJOR) {
    tma_load_2d(dst, map, bar, k_elem, mn0);                       // one box: 128 rows x 128 B
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) tma_load_2d(dst + i * 4096, map, bar, mn0 + i * 32, k_elem);   // boxes of 32 MN x 32 k
  }
}

// ---------------------------------------------------------------- kernel
// tmap_x: B_lo (MODE 2) or the a_scale slices (EXT_SCALE_SMEM)
template <bool A_MN, bool B_MN, int MODE, int EXT>
__global__ void __launch_bounds__(NUM_THREADS, (Cfg<MODE, B_MN>::CTAS_PER_SM))
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_x, const Params p) {
  constexpr bool SC_SMEM = EXT == EXT_SCALE_SMEM, SC_GMEM = EXT == EXT_SCALE_GMEM, SCALE = SC_SMEM || SC_GMEM;
  constexpr bool PROD_BWD = EXT == EXT_PROD_BWD, CAR_BWD = EXT == EXT_CAR_BWD, TRANS_D = EXT == EXT_TRANS_D;
  using C = Cfg<MODE, B_MN, SC_SMEM ? SC_BYTES : 0>;
  constexpr bool BF16 = MODE == 4;
  static_assert(!BF16 || !B_MN, "bf16x3: A fp32 of either major, B the transposed (K-major) bf16 plane");
  static_assert(!SCALE || (BF16 && !A_MN) || (MODE == 0 && A_MN && B_MN), "A scale: bf16x3 (K-major A), or single-pass TF32 weight gradient");
  static_assert(!TRANS_D || ((MODE == 0 || MODE == 1) && A_MN && !B_MN), "transposed D: TF32 / 3xTF32, A MN-major, B K-major");
  static_assert(!PROD_BWD || (MODE == 0 && !A_MN && !B_MN), "product backward: single-pass TF32, K-major operands");
  static_assert(!CAR_BWD || ((MODE == 0 || MODE == 1) && !A_MN && !B_MN), "CAR backward: TF32 / 3xTF32, K-major operands");
  static_assert(!CAR_BWD || C::STAGES * C::STAGE_BYTES >= (BM * EPI_LD + 2 * BM) * 4, "CAR backward: row slots behind the staged rows");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* prep = smem + C::STAGES * C::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);     // [STAGES] TMA landed

  const int tid = threadIdx.x;
  const int n_blk = (int)(blockIdx.x % p.n_tiles), m_blk = (int)(blockIdx.x / p.n_tiles);
  const int k_tiles_total = (int)((p.K + BK - 1) / BK);
  const int kt0 = blockIdx.y * p.k_tiles_per_split;
  const int num_kt = min(kt0 + p.k_tiles_per_split, k_tiles_total) - kt0;
  // first row of the M tile: position-aligned tiles hold pos_per_tile whole positions of `group` rows
  const int m0 = PROD_BWD ? m_blk * p.pos_per_tile * (int)p.group : m_blk * BM;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (C::BLO || SC_SMEM) tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < C::STAGES; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncthreads();

  auto issue = [&](int kt) {          // thread 0: k-tile kt -> stage kt % STAGES
    const int s = kt % C::STAGES;
    uint64_t* bar = &full[s];
    mbar_expect_tx(bar, C::STAGE_BYTES + (SC_SMEM ? SC_BYTES : 0));
    const uint32_t a_dst = smem_u32(smem + s * C::STAGE_BYTES);
    const uint32_t b_dst = a_dst + TILE_BYTES;
    const int k_elem = (kt0 + kt) * BK;
    load_operand<A_MN>(a_dst, &tmap_a, bar, m0, k_elem);
    if (BF16) {
      tma_load_2d(b_dst, &tmap_b, bar, (kt0 + kt) * 64, n_blk * BN);    // 128 n-rows x (32 hi | 32 lo) bf16
    } else {
      load_operand<B_MN>(b_dst, &tmap_b, bar, n_blk * BN, k_elem);
      if (C::BLO) load_operand<B_MN>(b_dst + TILE_BYTES, &tmap_x, bar, n_blk * BN, k_elem);
    }
    if (SC_SMEM) {                    // scale rows from the first group the tile's A rows (K-major) / k-rows (MN-major) touch
      const uint32_t sc_dst = smem_u32(smem + C::SC_OFF + s * SC_BYTES);
      if (A_MN) tma_load_2d(sc_dst, &tmap_x, bar, m0, (int)((uint32_t)k_elem / p.group));
      else tma_load_2d(sc_dst, &tmap_x, bar, k_elem, (int)((uint32_t)m0 / p.group));
    }
  };
  // k-tile kt goes to stage kt % STAGES; the stage of kt - 1 is refilled (with kt - 1 + STAGES) during k-tile kt, once
  // the MMAs of kt - 1 are done, so STAGES - 1 k-tiles are ahead of the one being multiplied
  if (tid == 0)
    for (int kt = 0; kt < C::STAGES - 1 && kt < num_kt; ++kt) issue(kt);
  int32_t car_l = -1, car_u = -1;
  if (CAR_BWD) car_bwd_row(p, m0, tid, car_l, car_u);

  // wgmma fragments: warp w (of 8) owns tile rows [16w, 16w + 16); lane = 4 g + t.  A: rows 16w + g (+8), k t (+4)
  // for tf32, k 2t (+8) for bf16 pairs.  D: rows 16w + g (+8), columns 8j + 2t (+1).
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int r0 = warp * 16 + g;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  // A fragments, double-buffered: the MMAs of a k-tile read theirs asynchronously, so k-tile kt writes buffer kt & 1,
  // whose last readers (the MMAs of kt - 2) are complete after the wait_group 1 of kt - 1
  uint32_t a[2][4][4], alo[2][4][4];      // tf32: hi (or the single-pass value) | lo (3xTF32)
  uint32_t ahi16[2][2][4], alo16[2][2][4];  // bf16x3: A_hi | A_lo pairs
  // tf32 A fragment q of k-step j is at a_off[q] + 1024 j (MN-major: 8 k-rows on) or a_off[q] ^ 32 j (K-major: the
  // 16-byte chunk index (2 j + q / 2) ^ (row & 7) is chunk (q / 2) ^ (row & 7) with 2 j XORed in).  bf16x3 with an
  // MN-major A: a_off[2 h + e] is element (r0 + 8 h, 2 t + e), and k + 8 i has the same k & 7, so element
  // (r0 + 8 h, 2 t + e + 8 i) is 1024 i bytes on
  uint32_t a_off[4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
    a_off[q] = BF16 ? tile_off<true>(r0 + (q >> 1) * 8, 2 * t + (q & 1)) : tile_off<A_MN>(r0 + (q & 1) * 8, t + (q >> 1) * 4);
  const uint32_t sc0 = smem_u32(smem + C::SC_OFF);           // a_scale slice of stage 0 (shared address)

  // One k-tile; BUF = kt & 1 is a compile-time constant (the loop below is unrolled by two) so that the fragments stay
  // in registers.  The MMAs of kt are left in flight while the next k-tile waits for its TMA and stages its operands.
  auto k_tile = [&](const int kt, auto buf_tag) {
    constexpr int BUF = decltype(buf_tag)::value;
    const int s = kt % C::STAGES;
    const int k_elem = (kt0 + kt) * BK;
    const uint32_t sc_s = (uint32_t)s * SC_BYTES;              // this k-tile's a_scale slice (EXT_SCALE_SMEM)
    mbar_wait(&full[s], (uint32_t)(kt / C::STAGES) & 1u);
    const uint8_t* sa = smem + s * C::STAGE_BYTES;
    if (SC_GMEM) {
      scale_tile_gmem<A_MN>(smem + s * C::STAGE_BYTES, p, m0, k_elem, tid);
      __syncthreads();                // fragments read elements other threads scaled
    }
    uint8_t* sb = smem + s * C::STAGE_BYTES + TILE_BYTES;
    // the prep tiles, or (MODE 0) B's own stage: the MMAs of kt - 1, still in flight, read another stage
    uint8_t* pb = C::PREP_TILES ? prep + BUF * C::PREP_TILE_BYTES : sb;
    if (C::PREP) {
      prep_b<B_MN, MODE>(sb, sb + TILE_BYTES, pb, pb + TILE_BYTES, tid);
      fence_proxy_async_smem();       // generic-proxy writes -> wgmma (async proxy) reads
      __syncthreads();                // both warpgroups read the whole prep tile
    }
    const uint32_t b_hi = smem_u32(pb);
    const uint32_t b_lo = b_hi + TILE_BYTES;        // 3x: the prep B_lo tile
    if (BF16) {
      // K-major A scale: rows r0 and r0 + 8 read slice row (their group minus the tile's first group), columns 2t (+1)
      // + 8 i of it.  Recomputed per k-tile: a value kept across the k-loop does not fit in the 128 registers.
      uint32_t sc_r[2] = {0u, 0u};
      if (SC_SMEM)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          sc_r[h] = sc0 + sc_s + ((uint32_t)(m0 + r0 + 8 * h) / p.group - (uint32_t)m0 / p.group) * (BK * 4) + 8 * t;
      uint32_t (&ahi)[2][4] = ahi16[BUF];
      uint32_t (&al)[2][4] = alo16[BUF];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = r0 + (q & 1) * 8, k = 16 * j + 2 * t + (q >> 1) * 8;
          // MN-major A: the pair (k, k + 1) is two 32-bit loads from adjacent k-rows.  Each load is free of bank
          // conflicts: k * 128 B is whole bank rows, so the bank is 4 ((r >> 2) & 7 ^ k & 7) + (r & 3).  Over a warp
          // (r = 16 w + g (+ 8), g = 0..7; k & 7 = 2 t (+ 1), t = 0..3) the chunk (r >> 2 & 7) ^ (k & 7) takes 8 distinct
          // values - bit 0 from g >> 2, bits 1-2 from t - and r & 3 = g & 3 picks the word: 32 lanes, 32 banks.
          float2 x;
          if (A_MN) {
            const uint32_t kk = (16 * j + (q >> 1) * 8) * 128;
            x.x = *reinterpret_cast<const float*>(sa + a_off[(q & 1) * 2] + kk);
            x.y = *reinterpret_cast<const float*>(sa + a_off[(q & 1) * 2 + 1] + kk);
          } else {
            x = *reinterpret_cast<const float2*>(sa + tile_off<false>(r, k));
          }
          if (SC_SMEM) {        // __fmul_rn: the product is rounded on its own, never contracted into the split
            const float2 f = ld_shared_f2(sc_r[q & 1] + (16 * j + (q >> 1) * 8) * 4);
            x.x = __fmul_rn(x.x, f.x); x.y = __fmul_rn(x.y, f.y);
          }
          split_bf16x2(x.x, x.y, ahi[j][q], al[j][q]);
        }
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 2; ++j) {        // two k = 16 steps per 32-k tile: 32 B of the hi half, then of the lo half
        wgmma_bf16(acc, al[j], make_desc(b_hi + 32 * j));           // A_lo * B_hi
        wgmma_bf16(acc, ahi[j], make_desc(b_hi + 64 + 32 * j));     // A_hi * B_lo
        wgmma_bf16(acc, ahi[j], make_desc(b_hi + 32 * j));          // A_hi * B_hi
      }
    } else {
      uint32_t (&ah)[4][4] = a[BUF];
      uint32_t (&al)[4][4] = alo[BUF];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          ah[j][q] = *reinterpret_cast<const uint32_t*>(sa + (A_MN ? a_off[q] + 1024 * j : a_off[q] ^ (32 * j)));
      if (SC_SMEM) {            // MN-major A (the weight gradient): element (m, k) is stored at row k, column m
        const uint32_t g0 = (uint32_t)k_elem / p.group;
#pragma unroll
        for (int h = 0; h < 8; ++h) {                        // k = t + 4 h: fragments q >> 1 = h & 1 of k-step j = h >> 1
          const int k = t + 4 * h;
          const int sr = (int)((uint32_t)(k_elem + k) / p.group - g0);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int m = r0 + 8 * i;
            const float f = ld_shared_f32(sc0 + sc_s + (sr * BM + m) * 4);
            uint32_t& x = ah[h >> 1][(h & 1) * 2 + i];
            x = __float_as_uint(__fmul_rn(__uint_as_float(x), f));
          }
        }
      }
      if (C::SPLIT3) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint32_t h = tf32_hi_bits(ah[j][q]);
            al[j][q] = __float_as_uint(__uint_as_float(ah[j][q]) - __uint_as_float(h));
            ah[j][q] = h;
          }
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {      // small terms first
          wgmma_tf32(acc, al[j], make_desc(b_hi + 32 * j));
          wgmma_tf32(acc, ah[j], make_desc(b_lo + 32 * j));
          wgmma_tf32(acc, ah[j], make_desc(b_hi + 32 * j));
        }
      } else {
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_tf32(acc, ah[j], make_desc(b_hi + 32 * j));
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                  // this warpgroup's MMAs of kt - 1 are done
    __syncthreads();                  // ... and the other's: stage (kt - 1) % STAGES and prep buffer (kt - 1) & 1 are free
    if (tid == 0 && kt + C::STAGES - 1 < num_kt) issue(kt + C::STAGES - 1);
  };
  if (SCALE) {                        // (the same loop without a counter kept past it: the scale leaves no register for it)
    for (int kt = 0; kt < num_kt; kt += 2) {
      k_tile(kt, std::integral_constant<int, 0>());
      if (kt + 1 < num_kt) k_tile(kt + 1, std::integral_constant<int, 1>());
    }
  } else {
    int kt = 0;
    for (; kt + 1 < num_kt; kt += 2) {
      k_tile(kt, std::integral_constant<int, 0>());
      k_tile(kt + 1, std::integral_constant<int, 1>());
    }
    if (kt < num_kt) k_tile(kt, std::integral_constant<int, 0>());
  }
  wgmma_wait<0>();
  fence_acc(acc);
  __syncthreads();                    // the other warpgroup's last MMAs may still read B from the operand ring

  // ===== epilogue: the accumulators go through shared memory (the operand ring is idle now) so that each warp then
  // handles 128 contiguous bytes of one row of D / aux per instruction
  float* stage = reinterpret_cast<float*>(smem);
  int32_t* s_l = reinterpret_cast<int32_t*>(stage + BM * EPI_LD);      // EXT_CAR_BWD: [BM] positions | [BM] slots
  int32_t* s_u = s_l + BM;
  if (CAR_BWD && tid < BM) { s_l[tid] = car_l; s_u[tid] = car_u; }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = 8 * j + 2 * t;
    if (TRANS_D) {   // stage row = tile column: 4 (2 t + i) + g + const over a warp, 32 banks per scalar store
      stage[c * EPI_LD + r0] = acc[4 * j]; stage[(c + 1) * EPI_LD + r0] = acc[4 * j + 1];
      stage[c * EPI_LD + r0 + 8] = acc[4 * j + 2]; stage[(c + 1) * EPI_LD + r0 + 8] = acc[4 * j + 3];
    } else {
      *reinterpret_cast<float2*>(stage + r0 * EPI_LD + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stage + (r0 + 8) * EPI_LD + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  __syncthreads();
  if (PROD_BWD) {                     // Ec rows of a chunk in the rest of the operand ring (60 at 3 stages of 32 KB)
    prod_bwd_epilogue<(C::STAGES * C::STAGE_BYTES - BM * EPI_LD * 4) / (BN * 4)>(p, stage, m_blk, n_blk, tid);
    return;
  }
  if (CAR_BWD) {
    car_bwd_epilogue(p, stage, s_l, s_u, m0, n_blk, tid);
    return;
  }
  if (TRANS_D) {                      // D row = tile column n, D columns = tile rows m: 128 contiguous bytes per warp
    const int64_t col = (int64_t)m0 + lane * 4;
    if (col >= p.M) return;
    for (int it = 0; it < BN / 8; ++it) {
      const int nl = it * 8 + warp;
      const int64_t row = (int64_t)n_blk * BN + nl;
      if (row >= p.N) break;
      const float4 v = *reinterpret_cast<const float4*>(stage + nl * EPI_LD + lane * 4);
      float* d = p.D + row * p.ldd + col;
      if (col + 4 <= p.M) {
        if (p.accumulate) atomicAdd(reinterpret_cast<float4*>(d), v);      // red.global.add.v4.f32
        else *reinterpret_cast<float4*>(d) = v;
      } else {
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 3; ++j)
          if (col + j < p.M) { if (p.accumulate) atomicAdd(d + j, e[j]); else d[j] = e[j]; }
      }
    }
    return;
  }
  const int c4 = lane * 4;
  const int64_t col = (int64_t)n_blk * BN + c4;
  if (col >= p.N) return;
  for (int it = 0; it < BM / 8; ++it) {
    const int rl = it * 8 + warp;
    const int64_t row = (int64_t)m0 + rl;
    if (row >= p.M) break;
    const float4 v = *reinterpret_cast<const float4*>(stage + rl * EPI_LD + c4);
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.dact && col + 4 <= p.N) av = *reinterpret_cast<const float4*>(p.aux + row * p.ld_aux + col);
    epilogue_store4(p, v, row, col, av);
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// operand with logical shape [mn, k]; kmajor: ptr[mn*ld + k] else ptr[k*ld + mn].  Out-of-range boxes read zeros.
static int make_operand_map(const nar_ctx* ctx, CUtensorMap* map, const float* ptr, int64_t mn, int64_t k, int64_t ld, bool kmajor) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0 || (ld & 3) != 0 || ld <= 0) return NAR_ERR_INVALID;
  cuuint64_t dims[2]; cuuint64_t strides[1]; cuuint32_t box[2]; cuuint32_t estr[2] = {1, 1};
  if (kmajor) { dims[0] = (cuuint64_t)k; dims[1] = (cuuint64_t)mn; box[0] = BK; box[1] = 128; }
  else        { dims[0] = (cuuint64_t)mn; dims[1] = (cuuint64_t)k; box[0] = 32; box[1] = BK; }
  strides[0] = (cuuint64_t)ld * 4;
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled)(
      map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? NAR_OK : NAR_ERR_INVALID;
}

// the pre-split bf16 weight plane of MODE 4: [n_rows, ld] bf16, K-major, 64 elements (128 B) of it per 32-k tile
static int make_bf16_plane_map(const nar_ctx* ctx, CUtensorMap* map, const void* ptr, int64_t n_rows, int64_t k_tiles, int64_t ld) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0 || (ld & 7) != 0 || ld < k_tiles * 64) return NAR_ERR_INVALID;
  cuuint64_t dims[2] = {(cuuint64_t)(k_tiles * 64), (cuuint64_t)n_rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled)(
      map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? NAR_OK : NAR_ERR_INVALID;
}

// nar_pack_bf16x3: W [K, N] fp32 (row stride ldw) -> plane [N, ld_out] bf16 (see MODE 4).  32 x 32 tiles through shared
// memory: reads coalesced along n, writes 64 contiguous bytes (32 hi or 32 lo values of one n) per half warp.
struct PackDesc { const float* W; uint16_t* out; int K, N, ldw, ld_out; };
constexpr int MAX_PACK = 32;
constexpr int PACK_MAX_BLOCKS = 2 * 132;     // grid-stride; two blocks per SM of an H100 SXM

__global__ void __launch_bounds__(256)
pack_bf16x3_kernel(const PackDesc* __restrict__ descs) {
  __shared__ float tile[32][33];
  const PackDesc d = descs[blockIdx.y];
  const int kb_n = (d.K + 31) / 32, nb_n = (d.N + 31) / 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
  for (int t = blockIdx.x; t < kb_n * nb_n; t += gridDim.x) {
    const int kb = t / nb_n, nb = t - kb * nb_n;
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int k = kb * 32 + i, n = nb * 32 + tx;
      tile[i][tx] = (k < d.K && n < d.N) ? d.W[(int64_t)k * d.ldw + n] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {                             // i = n within the tile, tx = k within the block
      const int n = nb * 32 + i;
      if (n < d.N) {
        const float x = tile[tx][i];
        const __nv_bfloat16 h = __float2bfloat16_rn(x);
        const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
        uint16_t* o = d.out + (int64_t)n * d.ld_out + kb * 64 + tx;
        o[0] = *reinterpret_cast<const uint16_t*>(&h);
        o[32] = *reinterpret_cast<const uint16_t*>(&l);
      }
    }
  }
}

// a_scale slices for EXT_SCALE_SMEM: scale [n_groups, cols] (row stride ld), boxes of SC_ROWS_K groups x 32 columns (K-major
// A) or SC_ROWS_MN groups x 128 columns (MN-major A), unswizzled.  Out-of-range groups / columns read zeros.
static int make_scale_map(const nar_ctx* ctx, CUtensorMap* map, const float* ptr, int64_t n_groups, int64_t cols, int64_t ld, bool a_mn) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)n_groups};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {a_mn ? (cuuint32_t)BM : (cuuint32_t)BK, a_mn ? (cuuint32_t)SC_ROWS_MN : (cuuint32_t)SC_ROWS_K};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled)(
      map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? NAR_OK : NAR_ERR_INVALID;
}

template <bool A_MN, bool B_MN, int MODE, int EXT = 0>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tbl, const Params& p, dim3 grid, cudaStream_t st) {
  auto kern = gemm_kernel<A_MN, B_MN, MODE, EXT>;
  constexpr int smem = Cfg<MODE, B_MN, EXT == EXT_SCALE_SMEM ? SC_BYTES : 0>::SMEM_BYTES;
  static bool attr_set = false;     // per instantiation
  if (!attr_set) {
    NAR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // all of the SM's unified L1 / shared memory as shared memory, so that CTAS_PER_SM blocks fit side by side
    NAR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    attr_set = true;
  }
  kern<<<grid, NUM_THREADS, smem, st>>>(ta, tb, tbl, p);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

template <int MODE>
static int ctas_per_sm(bool b_mn) { return b_mn ? Cfg<MODE, true>::CTAS_PER_SM : Cfg<MODE, false>::CTAS_PER_SM; }

}  // namespace gemm
}  // namespace nar

extern "C" int nar_pack_bf16x3(const float* const* W, void* const* out, const int32_t* K, const int32_t* N, const int32_t* ldw,
                               const int32_t* ld_out, int n, void* descs_dev, void* stream) {
  using namespace nar::gemm;
  if (!W || !out || !K || !N || !ldw || !ld_out || !descs_dev || n <= 0 || n > MAX_PACK) return NAR_ERR_INVALID;
  PackDesc h[MAX_PACK];
  int max_tiles = 1;
  for (int i = 0; i < n; ++i) {
    if (!W[i] || !out[i] || K[i] <= 0 || N[i] <= 0 || ld_out[i] < (K[i] + 31) / 32 * 64) return NAR_ERR_INVALID;
    h[i].W = W[i]; h[i].out = static_cast<uint16_t*>(out[i]); h[i].K = K[i]; h[i].N = N[i]; h[i].ldw = ldw[i]; h[i].ld_out = ld_out[i];
    const int t = ((K[i] + 31) / 32) * ((N[i] + 31) / 32);
    max_tiles = t > max_tiles ? t : max_tiles;
  }
  // the descriptor table is written once per distinct set (callers keep it; stream-ordered copy from a pageable buffer
  // would be a sync, so it goes through a kernel-argument-sized async memcpy only when it changed)
  static PackDesc last[MAX_PACK]; static int last_n = 0; static void* last_dev = nullptr;
  if (last_dev != descs_dev || last_n != n || memcmp(last, h, sizeof(PackDesc) * n) != 0) {
    NAR_CHECK_CUDA(cudaMemcpy(descs_dev, h, sizeof(PackDesc) * n, cudaMemcpyHostToDevice));
    memcpy(last, h, sizeof(PackDesc) * n); last_n = n; last_dev = descs_dev;
  }
  dim3 grid((unsigned)(max_tiles > PACK_MAX_BLOCKS ? PACK_MAX_BLOCKS : max_tiles), (unsigned)n);
  pack_bf16x3_kernel<<<grid, 256, 0, as_stream(stream)>>>(static_cast<const PackDesc*>(descs_dev));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

namespace nar {
namespace gemm {

// nar_gemm_tf32, and with trans_d D written transposed (nar_gemm_tf32_dt)
static int gemm(nar_ctx* ctx, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda, int a_kmajor, const float* B,
                int64_t ldb, int b_kmajor, float* D, int64_t ldd, const nar_gemm_epilogue* epi, void* stream, bool trans_d) {
  if (!ctx || !ctx->encode_tiled) return NAR_ERR_NO_DEVICE;
  if (!A || !epi || (!B && epi->precision != 4)) return NAR_ERR_INVALID;
  const bool car_bwd = epi->car_pp != nullptr;       // writes the CAR layer-1 gradients instead of D
  if (car_bwd ? D != nullptr : !D) return NAR_ERR_INVALID;
  if (M <= 0 || N <= 0 || K <= 0) return NAR_OK;     // empty problem: nothing to do
  if ((ldd & 3) != 0 || (reinterpret_cast<uintptr_t>(D) & 15u) != 0) return NAR_ERR_INVALID;
  if (epi->bias && (reinterpret_cast<uintptr_t>(epi->bias) & 15u) != 0) return NAR_ERR_INVALID;
  if (epi->dact && !car_bwd && (!epi->aux || (epi->ld_aux & 3) != 0 || (reinterpret_cast<uintptr_t>(epi->aux) & 15u) != 0)) return NAR_ERR_INVALID;
  if (epi->precision != 1 && epi->precision != 3 && epi->precision != 4) return NAR_ERR_INVALID;
  auto is_act = [](int32_t a) { return a == NAR_ACT_NONE || a == NAR_ACT_LEAKY_RELU || a == NAR_ACT_TANH; };
  if (!is_act(epi->act) || !is_act(epi->dact)) return NAR_ERR_INVALID;
  // every split-K CTA runs the epilogue on its own partial sum: a bias or an activation would apply once per split
  if (epi->split_k > 1 && (epi->bias || epi->act)) return NAR_ERR_INVALID;
  const bool bf16 = epi->precision == 4;
  if (bf16 && (!epi->b_bf16 || epi->accumulate || epi->split_k > 1)) return NAR_ERR_INVALID;
  const bool blo = epi->precision == 3 && epi->b_lo != nullptr;
  const int mode = bf16 ? 4 : (epi->precision == 1 ? 0 : (blo ? 2 : 1));
  const bool scale = epi->a_scale != nullptr, prod_bwd = epi->pred != nullptr;
  const int64_t a_rows = a_kmajor ? M : K, a_cols = a_kmajor ? K : M;       // A's storage
  // transposed D: TF32 / 3xTF32 splitting B in-kernel, A MN-major, B K-major, a plain (or accumulated) product
  if (trans_d && ((mode != 0 && mode != 1) || a_kmajor || !b_kmajor || epi->bias || epi->act || epi->dact || epi->aux || scale ||
                  prod_bwd || car_bwd)) return NAR_ERR_INVALID;
  if (scale) {
    // implemented: bf16x3 (K-major A), and single-pass TF32 with both operands MN-major (the weight gradient)
    if (!((mode == 4 && a_kmajor) || (mode == 0 && !a_kmajor && !b_kmajor)) || prod_bwd) return NAR_ERR_INVALID;
    if (epi->a_scale_group < 1 || a_rows > 0x7fffffffLL || a_cols > 0x7fffffffLL || epi->a_scale_group > a_rows ||
        epi->ld_a_scale < a_cols || (epi->ld_a_scale & 3) != 0 ||
        (reinterpret_cast<uintptr_t>(epi->a_scale) & 15u) != 0) return NAR_ERR_INVALID;
  } else if (epi->a_scale_group != 0 || epi->ld_a_scale != 0) {
    return NAR_ERR_INVALID;
  }
  if (prod_bwd) {
    const int64_t g = epi->pred_group;
    if (mode != 0 || !a_kmajor || !b_kmajor || epi->accumulate || epi->split_k > 1 || epi->bias || epi->act) return NAR_ERR_INVALID;
    if (g < 1 || g > BM || M % g != 0 || !epi->d_pred || !epi->aux || epi->ld_aux < N || epi->ld_pred < N) return NAR_ERR_INVALID;
  } else if (epi->d_pred || epi->pred_group != 0 || epi->ld_pred != 0 || epi->d_bias) {
    return NAR_ERR_INVALID;
  }
  if (car_bwd) {
    const int64_t kk = epi->car_k, ld = epi->ld_car;
    auto al16 = [](const void* q) { return q && (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
    if ((mode != 0 && mode != 1) || !a_kmajor || !b_kmajor || epi->accumulate || epi->split_k > 1 || epi->bias || epi->act ||
        epi->aux || scale || prod_bwd) return NAR_ERR_INVALID;
    // row, position and table indices in 32 bits
    if (kk < 1 || kk > 0x7fffffffLL - 1 || M > 0x7fffffffLL - BM || M % (kk + 1) != 0 || (N & 3) != 0 || ld < N || (ld & 3) != 0)
      return NAR_ERR_INVALID;
    if (!al16(epi->car_pp) || !al16(epi->car_pc) || !al16(epi->car_pi) || !al16(epi->car_dpp) || !al16(epi->car_dpc) ||
        !al16(epi->car_dpi) || !epi->car_pos_idx || !epi->car_neg_uidx) return NAR_ERR_INVALID;
  } else if (epi->car_pc || epi->car_pi || epi->car_pos_idx || epi->car_neg_uidx || epi->car_dpp || epi->car_dpc || epi->car_dpi ||
             epi->ld_car != 0 || epi->car_k != 0) {
    return NAR_ERR_INVALID;
  }
  // position-aligned M tiles: pos_per_tile whole positions of pred_group rows each (the rest of the 128 rows unused)
  const int64_t pos_per_tile = prod_bwd ? BM / epi->pred_group : 0, n_pos = prod_bwd ? M / epi->pred_group : 0;
  const int64_t n_tiles = (N + BN - 1) / BN, m_tiles = prod_bwd ? (n_pos + pos_per_tile - 1) / pos_per_tile : (M + BM - 1) / BM;
  if (n_tiles * m_tiles > 0x7fffffffLL) return NAR_ERR_UNSUPPORTED;
  const int k_tiles = (int)((K + BK - 1) / BK);
  const bool amn = !a_kmajor, bmn = !b_kmajor;
  int split = epi->split_k;
  if (split <= 0) {          // auto, for accumulate: as many CTAs as fit in one wave of the SMs' resident slots
    split = 1;               // (a CTA past a whole wave would run alone in a second one), at least 8 k-tiles per split;
    if (epi->accumulate && !epi->bias && !epi->act) {    // one split when the epilogue adds a bias or applies act
      const int per_sm = mode == 0 ? ctas_per_sm<0>(bmn) : (mode == 1 ? ctas_per_sm<1>(bmn) : ctas_per_sm<2>(bmn));
      const int64_t fit = (int64_t)per_sm * ctx->sm_count / (n_tiles * m_tiles);
      const int64_t cap = k_tiles / 8 > 1 ? k_tiles / 8 : 1;
      split = (int)(fit < cap ? fit : cap);
      if (split < 1) split = 1;
    }
  }
  if (split > k_tiles) split = k_tiles;
  if (split > 1 && !epi->accumulate) return NAR_ERR_INVALID;
  int per = (k_tiles + split - 1) / split;
  split = (k_tiles + per - 1) / per;          // no empty splits
  CUtensorMap ta, tb;
  int rc = make_operand_map(ctx, &ta, A, M, K, lda, a_kmajor != 0);
  if (rc) return rc;
  if (bf16) rc = make_bf16_plane_map(ctx, &tb, epi->b_bf16, N, k_tiles, epi->ld_bf16);
  else rc = make_operand_map(ctx, &tb, B, N, K, ldb, b_kmajor != 0);
  if (rc) return rc;
  CUtensorMap tbl = tb;
  if (blo) {
    rc = make_operand_map(ctx, &tbl, epi->b_lo, N, K, ldb, b_kmajor != 0);
    if (rc) return rc;
  }
  Params p;
  p.M = M; p.N = N; p.K = K; p.D = D; p.ldd = ldd; p.bias = epi->bias; p.aux = epi->aux; p.ld_aux = epi->ld_aux;
  p.act = epi->act; p.dact = epi->dact; p.accumulate = epi->accumulate; p.k_tiles_per_split = per;
  p.n_tiles = (int)n_tiles;
  p.a_scale = epi->a_scale; p.ld_a_scale = epi->ld_a_scale; p.a_rows = a_rows; p.a_cols = a_cols;
  p.group = (uint32_t)(scale ? epi->a_scale_group : (prod_bwd ? epi->pred_group : 1));
  p.pred = epi->pred; p.d_pred = epi->d_pred; p.d_bias = epi->d_bias; p.ld_pred = epi->ld_pred; p.n_pos = n_pos; p.pos_per_tile = (int)pos_per_tile;
  p.car_pp = epi->car_pp; p.car_pc = epi->car_pc; p.car_pi = epi->car_pi; p.car_pos_idx = epi->car_pos_idx;
  p.car_neg_uidx = epi->car_neg_uidx; p.car_dpp = epi->car_dpp; p.car_dpc = epi->car_dpc; p.car_dpi = epi->car_dpi;
  p.ld_car = epi->ld_car; p.car_k = (int)epi->car_k;
  dim3 grid((unsigned)(n_tiles * m_tiles), (unsigned)split, 1);
  cudaStream_t st = as_stream(stream);
  if (scale) {
    // the staged slice holds the groups one tile's rows (K-major A: 128) or one k-tile's rows (MN-major A: 32) touch
    const int64_t span = (a_kmajor ? BM - 1 : BK - 1) / epi->a_scale_group + 2;
    if (span <= (a_kmajor ? SC_ROWS_K : SC_ROWS_MN)) {
      rc = make_scale_map(ctx, &tbl, epi->a_scale, (a_rows + epi->a_scale_group - 1) / epi->a_scale_group, a_cols, epi->ld_a_scale,
                          !a_kmajor);
      if (rc) return rc;
      if (mode == 4) return launch<false, false, 4, EXT_SCALE_SMEM>(ta, tb, tbl, p, grid, st);
      return launch<true, true, 0, EXT_SCALE_SMEM>(ta, tb, tbl, p, grid, st);
    }
    if (mode == 4) return launch<false, false, 4, EXT_SCALE_GMEM>(ta, tb, tbl, p, grid, st);
    return launch<true, true, 0, EXT_SCALE_GMEM>(ta, tb, tbl, p, grid, st);
  }
  if (prod_bwd) return launch<false, false, 0, EXT_PROD_BWD>(ta, tb, tbl, p, grid, st);
  if (car_bwd) {                      // the engine's backward precision: single-pass TF32, or 3xTF32 splitting B in-kernel
    if (mode == 0) return launch<false, false, 0, EXT_CAR_BWD>(ta, tb, tbl, p, grid, st);
    return launch<false, false, 1, EXT_CAR_BWD>(ta, tb, tbl, p, grid, st);
  }
  if (trans_d) {
    if (mode == 0) return launch<true, false, 0, EXT_TRANS_D>(ta, tb, tbl, p, grid, st);
    return launch<true, false, 1, EXT_TRANS_D>(ta, tb, tbl, p, grid, st);
  }
  if (mode == 4) return amn ? launch<true, false, 4>(ta, tb, tbl, p, grid, st) : launch<false, false, 4>(ta, tb, tbl, p, grid, st);
#define NAR_GEMM_CASE(a, b) \
  if (amn == a && bmn == b) { \
    if (mode == 0) return launch<a, b, 0>(ta, tb, tbl, p, grid, st); \
    if (mode == 1) return launch<a, b, 1>(ta, tb, tbl, p, grid, st); \
    return launch<a, b, 2>(ta, tb, tbl, p, grid, st); \
  }
  NAR_GEMM_CASE(false, false) NAR_GEMM_CASE(false, true) NAR_GEMM_CASE(true, false) NAR_GEMM_CASE(true, true)
#undef NAR_GEMM_CASE
  return NAR_ERR_INVALID;
}

}  // namespace gemm
}  // namespace nar

extern "C" int nar_gemm_tf32(nar_ctx* ctx, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda, int a_kmajor,
                             const float* B, int64_t ldb, int b_kmajor, float* D, int64_t ldd,
                             const nar_gemm_epilogue* epi, void* stream) {
  return nar::gemm::gemm(ctx, M, N, K, A, lda, a_kmajor, B, ldb, b_kmajor, D, ldd, epi, stream, false);
}

extern "C" int nar_gemm_tf32_dt(nar_ctx* ctx, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda, int a_kmajor,
                                const float* B, int64_t ldb, int b_kmajor, float* D, int64_t ldd,
                                const nar_gemm_epilogue* epi, void* stream) {
  return nar::gemm::gemm(ctx, M, N, K, A, lda, a_kmajor, B, ldb, b_kmajor, D, ldd, epi, stream, true);
}
