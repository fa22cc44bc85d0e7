// Context + small HBM-bound helpers: TF-flavoured Adam, column sums (bias grads), l2 loss,
// transpose (Wh^T for BPTT), activation backward.
#include "common.cuh"
#include <stdlib.h>

namespace nar {
namespace misc {

__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// tf.train.AdamOptimizer (nar_model.py:708-722): lr_t = lr*sqrt(1-b2^t)/(1-b1^t) computed on the host
// in double; w -= lr_t * m / (sqrt(v) + eps).  Elements [0, reg_end) carry an l2_regularizer:
// their gradient gets + reg_l2 * w (d/dw of reg_l2 * sum(w^2)/2).
__global__ void __launch_bounds__(256)
adam_tf_kernel(float4* __restrict__ w, const float4* __restrict__ g, float4* __restrict__ m, float4* __restrict__ v,
               int64_t n4, int64_t reg_end4, float reg_l2, float lr_t, float b1, float b2, float eps, float4* __restrict__ wlo) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 wi = w[i], gi = g[i], mi = m[i], vi = v[i];
    const float r = i < reg_end4 ? reg_l2 : 0.f;
#define NAR_ADAM1(c)                                              \
    { const float gg = fmaf(r, wi.c, gi.c);                       \
      mi.c = b1 * mi.c + (1.f - b1) * gg;                         \
      vi.c = b2 * vi.c + (1.f - b2) * gg * gg;                    \
      wi.c -= lr_t * mi.c / (sqrtf(vi.c) + eps); }
    NAR_ADAM1(x) NAR_ADAM1(y) NAR_ADAM1(z) NAR_ADAM1(w)
#undef NAR_ADAM1
    w[i] = wi; m[i] = mi; v[i] = vi;
    if (wlo) wlo[i] = make_float4(tf32_lo(wi.x), tf32_lo(wi.y), tf32_lo(wi.z), tf32_lo(wi.w));
  }
}

__global__ void __launch_bounds__(256)
tf32_lo_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ lo) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) lo[i] = tf32_lo(x[i]);
}

// out[c] += sum_r x[r,c] ; CTA = 256 columns x 64-row slab
__global__ void __launch_bounds__(256)
colsum_add_kernel(const float* __restrict__ x, int64_t rows, int64_t cols, int64_t ld, float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * 64, r1 = min(rows, r0 + 64);
  if (c >= cols) return;
  // 8 independent partial sums: 8 loads in flight per thread instead of a load -> add chain
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int64_t r = r0;
  for (; r + 8 <= r1; r += 8) {
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] += __ldg(x + (r + u) * ld + c);
  }
  for (; r < r1; ++r) a[0] += __ldg(x + r * ld + c);
  atomicAdd(out + c, ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7])));
}

__global__ void __launch_bounds__(256)
l2_loss_add_kernel(const float* __restrict__ x, int64_t n, float scale, float* __restrict__ out) {
  __shared__ float sh[8];
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    acc = fmaf(v, v, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += sh[i];
    atomicAdd(out, scale * 0.5f * t);
  }
}

__global__ void __launch_bounds__(256)
act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, int64_t n, int act, float* __restrict__ dx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dx[i] = dy[i] * act_grad_from_output(y[i], act);
}

__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ src, int64_t rows, int64_t cols, int64_t ld_src, float* __restrict__ dst, int64_t ld_dst) {
  __shared__ float tile[32][33];
  const int64_t c0 = (int64_t)blockIdx.x * 32, r0 = (int64_t)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = r0 + i, c = c0 + tx;
    tile[i][tx] = (r < rows && c < cols) ? src[r * ld_src + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int64_t c = c0 + i, r = r0 + tx;       // dst[c, r]
    if (c < cols && r < rows) dst[c * ld_dst + r] = tile[tx][i];
  }
}

// dropout with counter-based masks (spec: oracle/dropout_ref.py): one Philox4x32-10 block per 4 consecutive columns
__global__ void __launch_bounds__(256)
dropout_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t rows, int cols4, int64_t ld,
                    const int32_t* __restrict__ row_pos, int64_t n_input, int64_t n_cand, int64_t K, int tensor_id,
                    float inv_keep, unsigned long long thr, uint32_t k0, uint32_t k1, uint32_t step) {
  const int64_t total = rows * cols4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols4; const int cb = (int)(i - r * cols4);
    unsigned long long key = (unsigned long long)(long long)row_pos[r];
    int tid = tensor_id;
    if (tensor_id == 0) {
      if (r < n_input) tid = 1;
      else { const int64_t j = (r - n_input) % n_cand; if (j == 0) tid = 2; else { tid = 3; key = key * (unsigned long long)K + (unsigned long long)(j - 1); } }
    }
    const Philox4 p = philox4x32_10((uint32_t)cb, (uint32_t)key, (uint32_t)((key >> 32) & 0xFFFFFFull) | ((uint32_t)tid << 24), step, k0, k1);
    const float4 v = *reinterpret_cast<const float4*>(src + r * ld + 4 * cb);
    float4 o;
    o.x = (unsigned long long)p.x < thr ? v.x * inv_keep : 0.f;
    o.y = (unsigned long long)p.y < thr ? v.y * inv_keep : 0.f;
    o.z = (unsigned long long)p.z < thr ? v.z * inv_keep : 0.f;
    o.w = (unsigned long long)p.w < thr ? v.w * inv_keep : 0.f;
    *reinterpret_cast<float4*>(dst + r * ld + 4 * cb) = o;
  }
}

// the residual session stack's layer output: out = h + res, 4 columns per thread (out may alias h or res)
__global__ void __launch_bounds__(256)
residual_add_kernel(const float* h, const float* res, int64_t rows, int cols4, int64_t ld, float* out) {
  const int64_t total = rows * cols4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols4; const int64_t o = r * ld + 4 * (i - r * cols4);
    const float4 a = *reinterpret_cast<const float4*>(h + o);
    const float4 b = *reinterpret_cast<const float4*>(res + o);
    *reinterpret_cast<float4*>(out + o) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

static unsigned grid_for(int64_t n, int per_block) {
  int64_t g = (n + per_block - 1) / per_block;
  const int64_t cap = NAR_GRID_SMS * 8;
  return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace misc
}  // namespace nar

// ------------------------------------------------------------------ context
extern "C" int nar_abi_version(void) { return NAR_ABI_VERSION; }

extern "C" int nar_abi_struct_size(int which) {
  switch (which) {
    case 0: return (int)sizeof(nar_feature_plan);
    case 1: return (int)sizeof(nar_model_cfg);
    case 2: return (int)sizeof(nar_step_io);
    case 3: return (int)sizeof(nar_row_layout);
    case 4: return (int)sizeof(nar_gemm_epilogue);
    case 5: return (int)sizeof(nar_segment);
  }
  return -1;
}

extern "C" const char* nar_status_string(int status) {
  switch (status) {
    case NAR_OK: return "ok";
    case NAR_ERR_INVALID: return "invalid argument";
    case NAR_ERR_UNSUPPORTED: return "unsupported";
    case NAR_ERR_NO_DEVICE: return "no sm_90 CUDA device / driver entry point";
    case NAR_ERR_WORKSPACE: return "workspace too small";
  }
  if (status > 0) return cudaGetErrorString((cudaError_t)status);
  return "unknown";
}

extern "C" int nar_ctx_create(int device, nar_ctx** out) {
  if (!out) return NAR_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return NAR_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  NAR_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return NAR_ERR_NO_DEVICE;         // sm_90a code only
  NAR_CHECK_CUDA(cudaSetDevice(device));
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) return NAR_ERR_NO_DEVICE;
  nar_ctx* c = new nar_ctx();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->encode_tiled = fn;
  c->gather_desc = nullptr; c->gather_key = nullptr; c->gather_key_valid = 0;
  if (cudaMalloc(&c->gather_desc, NAR_GATHER_DESC_BYTES) != cudaSuccess) { delete c; return NAR_ERR_NO_DEVICE; }
  c->gather_key = malloc(sizeof(nar_feature_plan));
  *out = c;
  return NAR_OK;
}

extern "C" int nar_ctx_destroy(nar_ctx* ctx) {
  if (ctx) { cudaFree(ctx->gather_desc); free(ctx->gather_key); }
  delete ctx;
  return NAR_OK;
}

// ------------------------------------------------------------------ helpers
extern "C" int nar_tf32_lo(const float* x, int64_t n, float* lo, void* stream) {
  if (!x || !lo) return NAR_ERR_INVALID;
  if (n <= 0) return NAR_OK;
  nar::misc::tf32_lo_kernel<<<nar::misc::grid_for(n, 1024), 256, 0, as_stream(stream)>>>(x, n, lo);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_adam_tf(float* params, const float* grads, float* m, float* v, int64_t n, int64_t reg_end, float reg_l2,
                           float lr, float beta1, float beta2, float eps, int64_t step, float* params_lo, void* stream) {
  if (!params || !grads || !m || !v || (n & 3) || (reg_end & 3) || step < 1) return NAR_ERR_INVALID;
  if (n == 0) return NAR_OK;
  const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, (double)step)) / (1.0 - pow((double)beta1, (double)step));
  nar::misc::adam_tf_kernel<<<nar::misc::grid_for(n / 4, 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<float4*>(params), reinterpret_cast<const float4*>(grads), reinterpret_cast<float4*>(m),
      reinterpret_cast<float4*>(v), n / 4, reg_end / 4, reg_l2, (float)lr_t, beta1, beta2, eps,
      reinterpret_cast<float4*>(params_lo));
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_dropout_rows(const float* src, float* dst, int64_t rows, int64_t cols, int64_t ld, const int32_t* row_pos,
                                int64_t n_input, int64_t n_cand, int64_t K, int tensor_id, float keep_prob, uint64_t seed,
                                uint32_t step, void* stream) {
  if (!src || !dst || !row_pos || (cols & 3) || (ld & 3) || tensor_id < 0 || tensor_id > 255) return NAR_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) return NAR_ERR_INVALID;   // float4 rows
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NAR_ERR_INVALID;
  if (tensor_id == 0 && (n_cand <= 0 || K != n_cand - 1)) return NAR_ERR_INVALID;
  if (rows <= 0 || cols <= 0) return NAR_OK;
  const unsigned long long thr = (unsigned long long)floor((double)keep_prob * 4294967296.0);
  nar::misc::dropout_rows_kernel<<<nar::misc::grid_for(rows * (cols / 4), 256), 256, 0, as_stream(stream)>>>(
      src, dst, rows, (int)(cols / 4), ld, row_pos, n_input, n_cand, K, tensor_id, 1.0f / keep_prob, thr, (uint32_t)seed,
      (uint32_t)(seed >> 32) ^ 0x5DEECE66u, step);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_colsum_add(const float* x, int64_t rows, int64_t cols, int64_t ld, float* out, void* stream) {
  if (!x || !out) return NAR_ERR_INVALID;
  if (rows <= 0 || cols <= 0) return NAR_OK;
  dim3 grid((unsigned)((cols + 255) / 256), (unsigned)((rows + 63) / 64));
  if (grid.y > 65535u) return NAR_ERR_UNSUPPORTED;
  nar::misc::colsum_add_kernel<<<grid, 256, 0, as_stream(stream)>>>(x, rows, cols, ld, out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_l2_loss_add(const float* x, int64_t n, float scale, float* out, void* stream) {
  if (!x || !out) return NAR_ERR_INVALID;
  if (n <= 0) return NAR_OK;
  nar::misc::l2_loss_add_kernel<<<nar::misc::grid_for(n, 1024), 256, 0, as_stream(stream)>>>(x, n, scale, out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_act_bwd(const float* dy, const float* y, int64_t n, int act, float* dx, void* stream) {
  if (!dy || !y || !dx) return NAR_ERR_INVALID;
  if (n <= 0) return NAR_OK;
  nar::misc::act_bwd_kernel<<<nar::misc::grid_for(n, 1024), 256, 0, as_stream(stream)>>>(dy, y, n, act, dx);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_residual_add(const float* h, const float* res, int64_t rows, int64_t cols, int64_t ld, float* out,
                                void* stream) {
  if (!h || !res || !out || cols < 0 || (cols & 3) || (ld & 3) || ld < cols) return NAR_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(out)) & 15u)
    return NAR_ERR_INVALID;                                                                        // float4 accesses
  if (rows <= 0 || cols == 0) return NAR_OK;
  nar::misc::residual_add_kernel<<<nar::misc::grid_for(rows * (cols / 4), 256), 256, 0, as_stream(stream)>>>(
      h, res, rows, (int)(cols / 4), ld, out);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}

extern "C" int nar_transpose_f32(const float* src, int64_t rows, int64_t cols, int64_t ld_src, float* dst, int64_t ld_dst, void* stream) {
  if (!src || !dst) return NAR_ERR_INVALID;
  if (rows <= 0 || cols <= 0) return NAR_OK;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  nar::misc::transpose_kernel<<<grid, 256, 0, as_stream(stream)>>>(src, rows, cols, ld_src, dst, ld_dst);
  NAR_LAUNCH_CHECK();
  return NAR_OK;
}
